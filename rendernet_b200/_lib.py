"""ctypes binding of librendernet_b200.so (C ABI declared in include/rendernet_b200.h).

The library is built in-tree by ``rendernet_b200/csrc/Makefile`` (``__graft_entry__.build()``).
There is NO fallback: if the shared object is missing the import fails loudly.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# RENDERNET_B200_LIB points at another build of the SAME C ABI (same-box A/B of two builds: scripts/step_time.py)
LIB_PATH = os.environ.get("RENDERNET_B200_LIB") or os.path.join(_HERE, "librendernet_b200.so")


class rn_conv_desc(C.Structure):
    _fields_ = [
        ("ndim", C.c_int), ("B", C.c_int), ("H", C.c_int), ("W", C.c_int), ("D", C.c_int),
        ("Cin", C.c_int), ("Cout", C.c_int), ("cout_pad", C.c_int), ("ntaps", C.c_int),
        ("taps", C.c_void_p), ("x", C.c_void_p), ("w_packed", C.c_void_p), ("bias", C.c_void_p),
        ("alpha", C.c_void_p), ("act", C.c_int), ("residual", C.c_void_p), ("residual_is_f32", C.c_int),
        ("out16", C.c_void_p), ("out32", C.c_void_p),
        ("o_base", C.c_longlong), ("o_b", C.c_longlong), ("o_y", C.c_longlong), ("o_x", C.c_longlong),
        ("o_z", C.c_longlong), ("fmt", C.c_int), ("force_bn", C.c_int), ("force_kps", C.c_int),
        ("max_ctas", C.c_int),
        ("x_channels", C.c_int), ("a_c_base", C.c_int), ("a_c_ntile", C.c_int), ("w_banded", C.c_int),
        ("band_cin", C.c_int), ("band_cout", C.c_int), ("band_sz", C.c_int),
        ("cluster", C.c_int), ("cta_group", C.c_int), ("ny", C.c_int), ("tile_w", C.c_int), ("msub", C.c_int),
        ("o_nsplit", C.c_int), ("o_nhi", C.c_longlong),
        ("x_plane", C.c_longlong), ("w_plane", C.c_longlong), ("o_plane", C.c_longlong),
        ("epi_groups", C.c_int), ("res_prefetch", C.c_int), ("tma_store", C.c_int),
        ("phong", C.c_void_p),
    ]


class rn_phong(C.Structure):
    _fields_ = [("light_dir", C.c_void_p), ("light_col", C.c_void_p), ("out_u8", C.c_void_p), ("ambient", C.c_float),
                ("k_diffuse", C.c_float), ("background_white", C.c_int), ("with_mask", C.c_int)]


class rn_tuning(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("cluster", "cta_group", "kps", "msub", "epilogue_groups", "res_prefetch", "tma_store", "yhalo")]


_vp, _i, _f, _ll = C.c_void_p, C.c_int, C.c_float, C.c_longlong
_tp = C.POINTER(rn_tuning)
PLAN_FIELDS = ("bn", "cluster", "cta_group", "msub", "epilogue_groups", "ny", "tile_w", "tile_h", "tile_d", "kps", "stages",
               "smem_bytes", "grid", "tiles", "epilogue_mode", "row_bytes")

# name -> (restype, argtypes); mirrors include/rendernet_b200.h one to one
SIGNATURES = {
    "rn_version": (_i, []),
    "rn_error_string": (C.c_char_p, [_i]),
    "rn_launch_count": (_ll, []),
    "rn_resample_f32": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _vp]),
    "rn_interpolate_f32": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _ll, _vp]),
    "rn_pack_conv_weights": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _vp, _i, _i, _vp]),
    "rn_cast_f32_to_16": (_i, [_vp, _vp, _ll, _ll, _i, _vp]),
    "rn_cast_16_to_f32": (_i, [_vp, _vp, _ll, _i, _vp]),
    "rn_bias_act_16": (_i, [_vp, _vp, _vp, _i, _vp, _vp, _vp, _ll, _i, _i, _vp]),
    "rn_conv_igemm": (_i, [C.POINTER(rn_conv_desc), _vp]),
    "rn_conv_plan": (_i, [C.POINTER(rn_conv_desc), C.POINTER(C.c_int), _i]),
    "rn_conv2d_same": (_i, [_vp, _vp, _vp, _vp, _i, _vp, _i, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _tp, _vp]),
    "rn_conv3d_same": (_i, [_vp, _vp, _vp, _vp, _i, _vp, _i, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _tp, _vp]),
    "rn_conv3d_banded_bytes": (_ll, [_i, _i, _i]),
    "rn_pack_conv3d_banded": (_i, [_vp, _vp, _i, _i, _i, _i, _vp]),
    "rn_expand_channels": (_i, [_vp, _vp, _i, _i, _vp]),
    "rn_conv3d_banded_same": (_i, [_vp, _vp, _vp, _vp, _i, _vp, _i, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _tp, _vp]),
    "rn_pack_conv2d_transpose_weights": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "rn_conv2d_transpose_same": (_i, [_vp, _vp, _vp, _vp, _i, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _tp, _vp]),
    "rn_pack_conv2d_transpose_s2_merged": (_i, [_vp, _vp, _i, _i, _i, _vp]),
    "rn_conv2d_transpose_s2_merged": (_i, [_vp, _vp, _vp, _vp, _i, _vp, _vp, _i, _i, _i, _i, _i, _i, _tp, _vp]),
    "rn_xfold_factor": (_i, [_i, _i]),
    "rn_pack_conv2d_transpose_xfold": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "rn_conv2d_transpose_s1_xfold": (_i, [_vp, _vp, _vp, _vp, _i, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, C.POINTER(rn_phong), _tp, _vp]),
    "rn_conv3d_direct": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "rn_resample_conv1_fused": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "rn_resample5_conv1_fused": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "rn_binvox_decode": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp]),
    "rn_fully_connected": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "rn_conv3d_small": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "rn_concat_channels_f32": (_i, [_vp, _vp, _vp, _ll, _i, _i, _vp]),
    "rn_prelu_backward_16": (_i, [_vp, _vp, _vp, _vp, _ll, _i, _i, _vp]),
    "rn_sigmoid_backward": (_i, [_vp, _vp, _vp, _ll, _i, _i, _f, _i, _vp]),
    "rn_conv3d_backward_data_direct": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _f, _i, _vp]),
    "rn_resample_backward_f32": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp]),
    "rn_resample5_backward_f32": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "rn_prelu_backward_f32": (_i, [_vp, _vp, _vp, _vp, _ll, _i, _vp]),
    "rn_fully_connected_backward_workspace": (_ll, [_i, _i, _i]),
    "rn_fully_connected_backward_data": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "rn_conv3d_f32_workspace": (_ll, [_i] * 8),
    "rn_conv3d_f32": (_i, [_vp, _vp, _vp, _vp, _vp] + [_i] * 10 + [_vp]),
    "rn_act_backward_f32": (_i, [_vp, _vp, _vp, _ll, _i, _vp]),
    "rn_phong_recon_loss_grad": (_i, [_vp, _vp, _vp, _vp, _vp, _f, _f, _i, _i, _vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "rn_conv2d_weight_grad": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "rn_bias_grad_16": (_i, [_vp, _vp, _ll, _i, _i, _vp]),
    "rn_conv_weight_grad_direct": (_i, [_vp, _vp, _vp] + [_i] * 22 + [_f, _vp]),
    "rn_prelu_alpha_grad": (_i, [_vp, _vp, _vp, _ll, _i, _i, _f, _vp]),
    "rn_fully_connected_param_grad": (_i, [_vp] * 8 + [_i, _i, _i, _vp]),
    "rn_prelu_grad_f32": (_i, [_vp] * 6 + [_ll, _i, _vp]),
    "rn_dropout_16": (_i, [_vp, _vp, _ll, _f, C.c_uint, C.c_uint, _i, _vp]),
    "rn_dropout_mask_host": (_i, [_vp, _ll, _f, C.c_uint, C.c_uint]),
    "rn_image_loss_grad": (_i, [_vp, _vp, _vp, _vp, _ll, _i, _i, _vp]),
    "rn_adam_step": (_i, [_vp, _vp, _vp, _vp, _ll, _f, _f, _f, _f, _vp]),
    "rn_phong_composite": (_i, [_vp, _vp, _vp, _f, _f, _i, _i, _vp, _vp, _i, _i, _i, _vp]),
}


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"rendernet_b200: CUDA extension not built ({LIB_PATH} missing). "
            "Run `python -c 'import __graft_entry__ as g; g.build()'` or `make -C rendernet_b200/csrc`. "
            "There is no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the .so does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    return lib


lib = _load()


class RenderNetCudaError(RuntimeError):
    pass


def check(code: int, what: str = "") -> None:
    if code != 0:
        msg = lib.rn_error_string(code).decode()
        raise RenderNetCudaError(f"{what}: rc={code} ({msg})")
