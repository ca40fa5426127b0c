"""Torch-facing wrappers of the C-ABI kernels.  PyTorch is plumbing here (device memory, streams);
all arithmetic happens in librendernet_b200.so.  Everything requires CUDA tensors; there is no
CPU path.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Optional, Sequence

import torch

from ._lib import check, lib, rn_conv_desc, rn_phong, rn_tuning

ACT_NONE, ACT_PRELU, ACT_SIGMOID = 0, 1, 2
_ACT = {None: ACT_NONE, "none": ACT_NONE, "prelu": ACT_PRELU, "sigmoid": ACT_SIGMOID}


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


class Split16:
    """Activation of the "exact" precision mode (RN_FMT_F16X2): a pair of fp16 planes stored back to back, `planes` = [2, *shape],
    plane 0 = hi = fp16(v), plane 1 = lo = fp16(v - hi) (~22 significant bits together).  Behaves like a tensor of the
    logical `shape` for the handful of things the model functions do with activations."""

    __slots__ = ("planes",)

    def __init__(self, planes: torch.Tensor):
        assert planes.dtype == torch.float16 and planes.shape[0] == 2 and planes.is_contiguous()
        self.planes = planes

    @property
    def shape(self):
        return tuple(self.planes.shape[1:])

    @property
    def dtype(self):
        return torch.float16

    @property
    def is_cuda(self):
        return self.planes.is_cuda

    @property
    def device(self):
        return self.planes.device

    def reshape(self, *shape):
        shape = shape[0] if len(shape) == 1 and isinstance(shape[0], (tuple, list)) else shape
        return Split16(self.planes.reshape(2, *shape))

    def numel(self):
        return self.planes.numel() // 2

    def data_ptr(self):
        return self.planes.data_ptr()

    def float(self) -> torch.Tensor:
        return self.planes[0].float() + self.planes[1].float()

    def get_shape(self):
        return list(self.shape)

    def realize(self):
        return self


def _cuda(t, dtype=None):
    if not isinstance(t, (torch.Tensor, Split16)) and hasattr(t, "realize"):
        t = t.realize()            # deferred conv output / deferred resampled grid
    if not t.is_cuda:
        raise RuntimeError("rendernet_b200 kernels need CUDA tensors (there is no CPU fallback)")
    if dtype is not None and t.dtype != dtype:
        raise TypeError(f"expected {dtype}, got {t.dtype}")
    if isinstance(t, Split16):
        return t
    return t if t.is_contiguous() else t.contiguous()


def fmt_of(dtype: torch.dtype) -> int:
    if dtype == torch.float16:
        return 0
    if dtype == torch.bfloat16:
        return 1
    raise TypeError(f"16-bit dtype expected, got {dtype}")


def _act_in(x, fmt: int, dtype):
    """Validate a 16-bit activation argument against the layer's format; returns the tensor whose data_ptr is passed."""
    x = _cuda(x)
    if fmt == 2:
        if not isinstance(x, Split16):
            raise TypeError("this layer was packed for the exact mode (fp16 hi/lo pairs): pass a Split16 activation")
        return x
    if isinstance(x, Split16):
        raise TypeError("fp16 hi/lo pair passed to a layer packed for single 16-bit operands")
    if x.dtype != dtype:
        raise TypeError(f"expected {dtype}, got {x.dtype}")
    return x


def _alloc16(shape, fmt: int, dtype, device):
    if fmt == 2:
        return torch.empty((2,) + tuple(shape), device=device, dtype=torch.float16)
    return torch.empty(tuple(shape), device=device, dtype=dtype)


def _wrap16(t, fmt: int):
    return Split16(t) if (fmt == 2 and t is not None) else t


def _unwrap(t):
    return t.planes if isinstance(t, Split16) else t


def _tune(tune):
    """dict of rn_tuning fields (tests / A-B runs) -> ctypes pointer, None -> NULL (library defaults)."""
    if not tune:
        return None
    t = rn_tuning()
    for k, v in tune.items():
        if not hasattr(t, k):
            raise KeyError(f"unknown tuning field {k!r}")
        setattr(t, k, int(v))
    return C.byref(t)


def round_up(v: int, m: int) -> int:
    return (v + m - 1) // m * m


# --------------------------------------------------------------------------------------- resampler
def resample(vox: torch.Tensor, minv: torch.Tensor, new_size: int, transform: bool) -> torch.Tensor:
    """vox [B,S,S,S,C] fp32, minv [B,3,4] fp32 -> [B,N,N,N,C] fp32 (rn_resample_f32)."""
    vox = _cuda(vox, torch.float32)
    minv = _cuda(minv, torch.float32)
    B, S, _, _, Cc = vox.shape
    out = torch.empty((B, new_size, new_size, new_size, Cc), device=vox.device, dtype=torch.float32)
    check(lib.rn_resample_f32(vox.data_ptr(), minv.data_ptr(), out.data_ptr(), B, Cc, S, new_size,
                              1 if transform else 0, _stream()), "rn_resample_f32")
    return out


def interpolate(vox: torch.Tensor, x: torch.Tensor, y: torch.Tensor, z: torch.Tensor) -> torch.Tensor:
    """tf_interpolate at explicit coordinates: vox [B,S,S,S,C] fp32, x/y/z [B*n] fp32 -> [B*n, C] fp32 (rn_interpolate_f32)."""
    vox = _cuda(vox, torch.float32)
    x, y, z = (_cuda(t.reshape(-1).to(device=vox.device, dtype=torch.float32)) for t in (x, y, z))
    B, S, _, _, Cc = vox.shape
    n = x.numel()
    if y.numel() != n or z.numel() != n or n % B != 0:
        raise ValueError("interpolate: x, y, z must hold the same number of points, a multiple of the batch size")
    out = torch.empty((n, Cc), device=vox.device, dtype=torch.float32)
    check(lib.rn_interpolate_f32(vox.data_ptr(), x.data_ptr(), y.data_ptr(), z.data_ptr(), out.data_ptr(), B, Cc, S, n // B,
                                 _stream()), "rn_interpolate_f32")
    return out


# --------------------------------------------------------------------------------------- packed layers
@dataclass
class PackedConv:
    """Device-resident, kernel-ready parameters of one convolution layer."""
    kind: str                      # conv2d | conv3d | conv2d_transpose
    ksize: Sequence[int]
    stride: int
    cin: int
    cout: int
    cout_pad: int
    w: torch.Tensor                # 16-bit packed filter
    bias: torch.Tensor             # fp32 [cout_pad]
    alpha: Optional[torch.Tensor]  # fp32 [cout_pad]
    dtype: torch.dtype
    fmt: int = 0                   # RN_FMT_*: 0 fp16, 1 bf16, 2 fp16 hi/lo pairs (w then holds [2][...])


def _pad_vec(v: Optional[torch.Tensor], n: int, n_pad: int, device) -> Optional[torch.Tensor]:
    if v is None:
        return None
    out = torch.zeros(n_pad, device=device, dtype=torch.float32)
    out[:n] = v.to(device=device, dtype=torch.float32).reshape(-1)
    return out


def pack_conv(kind: str, w_tf: torch.Tensor, bias: Optional[torch.Tensor], alpha: Optional[torch.Tensor],
              stride: int = 1, dtype: torch.dtype = torch.float16, device="cuda", fmt: Optional[int] = None) -> PackedConv:
    """w_tf in TF filter layout: conv2d [kh,kw,Cin,Cout]; conv3d [k,k,k,Cin,Cout];
    conv2d_transpose [kh,kw,Cout,Cin]."""
    w_tf = torch.as_tensor(w_tf, dtype=torch.float32).to(device).contiguous()
    fmt = fmt_of(dtype) if fmt is None else int(fmt)
    if kind == "conv2d_transpose":
        kh, kw, cout, cin = w_tf.shape
        ks = (kh, kw)
    elif kind == "conv2d":
        kh, kw, cin, cout = w_tf.shape
        ks = (kh, kw)
    elif kind == "conv3d":
        k0, k1, k2, cin, cout = w_tf.shape
        ks = (k0, k1, k2)
    else:
        raise ValueError(kind)
    cout_pad = round_up(cout, 16)
    ntaps = 1
    for k in ks:
        ntaps *= k
    packed = _alloc16((ntaps, cout_pad, cin), fmt, dtype, device)
    if kind == "conv2d_transpose":
        check(lib.rn_pack_conv2d_transpose_weights(w_tf.data_ptr(), packed.data_ptr(), ks[0], ks[1], cin, cout,
                                                   cout_pad, stride, fmt, _stream()), "pack transpose")
    else:
        if stride != 1:
            raise ValueError("tensor-core conv path is stride 1")
        check(lib.rn_pack_conv_weights(w_tf.data_ptr(), packed.data_ptr(), ntaps, cin, cout, cout_pad, 0, None, 0,
                                       fmt, _stream()), "pack")
    b = _pad_vec(bias if bias is not None else torch.zeros(cout), cout, cout_pad, device)
    a = _pad_vec(alpha, cout, cout_pad, device)
    return PackedConv(kind, ks, stride, cin, cout, cout_pad, packed, b, a, dtype, fmt)


def _out_buffers(shape, dtype, device, want16, want32, out16, out32, fmt: int = 0):
    if want16 and out16 is None:
        out16 = _alloc16(shape, fmt, dtype, device)
    out16 = _unwrap(out16)
    if want32 and out32 is None:
        out32 = torch.empty(shape, device=device, dtype=torch.float32)
    return out16, out32


def _residual(residual, fmt: int):
    """-> (tensor or None, residual_is_f32).  16-bit residuals must be in the layer's format."""
    if residual is None:
        return None, 0
    residual = _cuda(residual)
    if isinstance(residual, Split16):
        if fmt != 2:
            raise TypeError("fp16 hi/lo residual for a layer packed for single 16-bit operands")
        return residual.planes, 0
    if residual.dtype == torch.float32:
        return residual, 1
    if fmt == 2:
        raise TypeError("exact-mode layers take an fp32 or an fp16 hi/lo (Split16) residual")
    return residual, 0


def _ret(out16, out32, want16, want32, fmt):
    out16 = _wrap16(out16, fmt)
    return out16 if not want32 else ((out16, out32) if want16 else out32)


def conv2d(x: torch.Tensor, L: PackedConv, act: Optional[str] = None, residual: Optional[torch.Tensor] = None,
           want16: bool = True, want32: bool = False, out16=None, out32=None, alpha=None, tune=None):
    """SAME stride-1 conv2d + bias (+PReLU/sigmoid) (+residual).  x [B,H,W,Cin] 16-bit."""
    x = _act_in(x, L.fmt, L.dtype)
    B, H, W, Cin = x.shape
    assert Cin == L.cin and L.kind == "conv2d"
    out16, out32 = _out_buffers((B, H, W, L.cout), L.dtype, x.device, want16, want32, out16, out32, L.fmt)
    residual, res_f32 = _residual(residual, L.fmt)
    if residual is not None:
        assert tuple(residual.shape[-4:]) == (B, H, W, L.cout)
    a = _ACT[act]
    check(lib.rn_conv2d_same(x.data_ptr(), L.w.data_ptr(), L.bias.data_ptr(),
                             _ptr(alpha if alpha is not None else L.alpha) if a == ACT_PRELU else None, a, _ptr(residual), res_f32,
                             _ptr(out16), _ptr(out32), B, H, W, Cin, L.cout, L.cout_pad, L.ksize[0], L.ksize[1],
                             L.fmt, _tune(tune), _stream()), "rn_conv2d_same")
    return _ret(out16, out32, want16, want32, L.fmt)


def conv3d(x: torch.Tensor, L: PackedConv, act: Optional[str] = None, residual: Optional[torch.Tensor] = None,
           want16: bool = True, want32: bool = False, out16=None, out32=None, alpha=None, tune=None):
    """SAME stride-1 k^3 conv3d on the tensor pipe.  x [B,H,W,D,Cin] 16-bit."""
    x = _act_in(x, L.fmt, L.dtype)
    B, H, W, D, Cin = x.shape
    assert Cin == L.cin and L.kind == "conv3d"
    out16, out32 = _out_buffers((B, H, W, D, L.cout), L.dtype, x.device, want16, want32, out16, out32, L.fmt)
    residual, res_f32 = _residual(residual, L.fmt)
    a = _ACT[act]
    check(lib.rn_conv3d_same(x.data_ptr(), L.w.data_ptr(), L.bias.data_ptr(),
                             _ptr(alpha if alpha is not None else L.alpha) if a == ACT_PRELU else None, a, _ptr(residual), res_f32,
                             _ptr(out16), _ptr(out32), B, H, W, D, Cin, L.cout, L.cout_pad, L.ksize[0],
                             L.fmt, _tune(tune), _stream()), "rn_conv3d_same")
    return _ret(out16, out32, want16, want32, L.fmt)


class BandedConv3d:
    """Depth-folded 3^3 SAME conv3d (rn_conv3d_banded_same): kernel-ready banded filter + per-depth expanded
    bias / alpha vectors (cached per D)."""

    def __init__(self, w_tf: torch.Tensor, bias: Optional[torch.Tensor], dtype=torch.float16, device="cuda", sz: int = 1,
                 fmt: Optional[int] = None):
        w_tf = torch.as_tensor(w_tf, dtype=torch.float32).to(device).contiguous()
        assert tuple(w_tf.shape[:3]) == (3, 3, 3)
        self.cin, self.cout, self.sz = int(w_tf.shape[3]), int(w_tf.shape[4]), int(sz)
        nbytes = lib.rn_conv3d_banded_bytes(self.cin, self.cout, self.sz)
        if nbytes < 0:
            raise ValueError("banded conv3d needs Cin | 64 and Cout | 128")
        self.dtype = dtype
        self.fmt = fmt_of(dtype) if fmt is None else int(fmt)
        self.w = _alloc16((nbytes // 2,), self.fmt, dtype, device)
        check(lib.rn_pack_conv3d_banded(w_tf.data_ptr(), self.w.data_ptr(), self.cin, self.cout, self.sz, self.fmt,
                                        _stream()), "rn_pack_conv3d_banded")
        self.bias = (bias if bias is not None else torch.zeros(self.cout)).to(device=device, dtype=torch.float32)
        self._full = {}

    @staticmethod
    def eligible(cin: int, cout: int, D: int, sz: int = 1) -> bool:
        return (cin >= 8 and cout >= 8 and 64 % cin == 0 and 128 % cout == 0 and sz in (1, 2)
                and (-(-D // sz) * cout) % 128 == 0 and (D * cin) % 8 == 0)

    def expanded(self, v: torch.Tensor, D: int, tag) -> torch.Tensor:
        key = (tag, D)
        f = self._full.get(key)
        if f is None:
            v = _cuda(v.to(device=self.w.device, dtype=torch.float32))
            f = torch.empty(D * self.cout, device=self.w.device, dtype=torch.float32)
            check(lib.rn_expand_channels(v.data_ptr(), f.data_ptr(), self.cout, D, _stream()), "rn_expand_channels")
            self._full[key] = f
        return f


def conv3d_banded(x: torch.Tensor, L: BandedConv3d, act: Optional[str] = None,
                  residual: Optional[torch.Tensor] = None, alpha: Optional[torch.Tensor] = None, alpha_tag=None,
                  want16: bool = True, want32: bool = False, out16=None, out32=None, tune=None):
    """x [B,H,W,D,Cin] 16-bit -> [B,H,W,D,Cout]; alpha is the per-Cout PReLU slope (length Cout)."""
    x = _act_in(x, L.fmt, L.dtype)
    B, H, W, D, Cin = x.shape
    assert Cin == L.cin
    Do = -(-D // L.sz)
    out16, out32 = _out_buffers((B, H, W, Do, L.cout), L.dtype, x.device, want16, want32, out16, out32, L.fmt)
    residual, res_f32 = _residual(residual, L.fmt)
    a = _ACT[act]
    bias_full = L.expanded(L.bias, Do, "bias")
    alpha_full = None
    if a == ACT_PRELU:
        if alpha_tag is not None:
            alpha_full = L.expanded(alpha[:L.cout], Do, ("alpha", alpha_tag))
        else:                      # untagged alpha: never cached (a freed tensor's address can be reused)
            v = _cuda(alpha[:L.cout].to(device=x.device, dtype=torch.float32))
            alpha_full = torch.empty(Do * L.cout, device=x.device, dtype=torch.float32)
            check(lib.rn_expand_channels(v.data_ptr(), alpha_full.data_ptr(), L.cout, Do, _stream()), "rn_expand_channels")
    check(lib.rn_conv3d_banded_same(x.data_ptr(), L.w.data_ptr(), bias_full.data_ptr(), _ptr(alpha_full), a,
                                    _ptr(residual), res_f32, _ptr(out16), _ptr(out32), B, H, W, D, Cin, L.cout, L.sz,
                                    L.fmt, _tune(tune), _stream()), "rn_conv3d_banded_same")
    return _ret(out16, out32, want16, want32, L.fmt)


def conv2d_transpose(x: torch.Tensor, L: PackedConv, act: Optional[str] = None, want16: bool = True,
                     want32: bool = False, out16=None, out32=None, alpha=None, tune=None):
    """SAME transposed conv, out = in*stride.  x [B,H,W,Cin] 16-bit."""
    x = _act_in(x, L.fmt, L.dtype)
    B, H, W, Cin = x.shape
    assert Cin == L.cin and L.kind == "conv2d_transpose"
    s = L.stride
    out16, out32 = _out_buffers((B, H * s, W * s, L.cout), L.dtype, x.device, want16, want32, out16, out32, L.fmt)
    a = _ACT[act]
    check(lib.rn_conv2d_transpose_same(x.data_ptr(), L.w.data_ptr(), L.bias.data_ptr(),
                                       _ptr(alpha if alpha is not None else L.alpha) if a == ACT_PRELU else None, a, _ptr(out16), _ptr(out32),
                                       B, H, W, Cin, L.cout, L.cout_pad, L.ksize[0], L.ksize[1], s,
                                       L.fmt, _tune(tune), _stream()), "rn_conv2d_transpose_same")
    return _ret(out16, out32, want16, want32, L.fmt)


class MergedConvT2:
    """k=4 stride-2 SAME transposed conv as one launch (rn_conv2d_transpose_s2_merged)."""

    def __init__(self, w_tf: torch.Tensor, bias: Optional[torch.Tensor], dtype=torch.float16, device="cuda",
                 fmt: Optional[int] = None):
        w_tf = torch.as_tensor(w_tf, dtype=torch.float32).to(device).contiguous()
        assert tuple(w_tf.shape[:2]) == (4, 4)
        self.cout, self.cin, self.dtype = int(w_tf.shape[2]), int(w_tf.shape[3]), dtype
        self.fmt = fmt_of(dtype) if fmt is None else int(fmt)
        self.w = _alloc16((9, 4 * self.cout, self.cin), self.fmt, dtype, device)
        check(lib.rn_pack_conv2d_transpose_s2_merged(w_tf.data_ptr(), self.w.data_ptr(), self.cin, self.cout, self.fmt,
                                                     _stream()), "pack merged tconv")
        b = bias if bias is not None else torch.zeros(self.cout)
        self.bias = b.to(device=device, dtype=torch.float32).reshape(-1).repeat(4).contiguous()
        self._alpha = {}

    @staticmethod
    def eligible(cin: int, cout: int) -> bool:
        return cin % 16 == 0 and cout % 16 == 0


def conv2d_transpose_s2_merged(x: torch.Tensor, L: MergedConvT2, act: Optional[str] = None,
                               alpha: Optional[torch.Tensor] = None, alpha_tag=None, want16: bool = True,
                               want32: bool = False, out16=None, out32=None, tune=None):
    x = _act_in(x, L.fmt, L.dtype)
    B, H, W, Cin = x.shape
    assert Cin == L.cin
    out16, out32 = _out_buffers((B, 2 * H, 2 * W, L.cout), L.dtype, x.device, want16, want32, out16, out32, L.fmt)
    a = _ACT[act]
    alpha4 = None
    if a == ACT_PRELU:
        alpha4 = L._alpha.get(alpha_tag) if alpha_tag is not None else None
        if alpha4 is None:     # untagged alphas are recomputed, never cached by address
            alpha4 = alpha.to(device=x.device, dtype=torch.float32).reshape(-1)[: L.cout].repeat(4).contiguous()
            if alpha_tag is not None:
                L._alpha[alpha_tag] = alpha4
    check(lib.rn_conv2d_transpose_s2_merged(x.data_ptr(), L.w.data_ptr(), L.bias.data_ptr(), _ptr(alpha4), a, _ptr(out16),
                                            _ptr(out32), B, H, W, Cin, L.cout, L.fmt, _tune(tune), _stream()),
          "rn_conv2d_transpose_s2_merged")
    return _ret(out16, out32, want16, want32, L.fmt)


class XFoldConvT:
    """Stride-1 transposed conv with thin channels, x-folded (rn_conv2d_transpose_s1_xfold)."""

    def __init__(self, w_tf: torch.Tensor, bias: Optional[torch.Tensor], F: int, dtype=torch.float16, device="cuda",
                 fmt: Optional[int] = None):
        w_tf = torch.as_tensor(w_tf, dtype=torch.float32).to(device).contiguous()
        self.kh, self.kw, self.cout, self.cin = (int(v) for v in w_tf.shape)
        self.F, self.dtype = F, dtype
        self.fmt = fmt_of(dtype) if fmt is None else int(fmt)
        self.cout_pad = round_up(F * self.cout, 16)
        self.w = _alloc16((self.kh * 3, self.cout_pad, F * self.cin), self.fmt, dtype, device)
        check(lib.rn_pack_conv2d_transpose_xfold(w_tf.data_ptr(), self.w.data_ptr(), self.kh, self.kw, self.cin, self.cout,
                                                 F, self.cout_pad, self.fmt, _stream()), "pack xfold")
        b = bias if bias is not None else torch.zeros(self.cout)
        self.bias = self.tiled(b, device)
        self._alpha = {}

    def tiled(self, v: torch.Tensor, device) -> torch.Tensor:
        out = torch.zeros(self.cout_pad, device=device, dtype=torch.float32)
        out[: self.F * self.cout] = v.to(device=device, dtype=torch.float32).reshape(-1)[: self.cout].repeat(self.F)
        return out

    @staticmethod
    def factor(cin: int, W: int) -> int:
        return int(lib.rn_xfold_factor(cin, W))


def conv2d_transpose_xfold(x: torch.Tensor, L: XFoldConvT, act: Optional[str] = None, alpha: Optional[torch.Tensor] = None,
                           alpha_tag=None, want16: bool = True, want32: bool = False, out16=None, out32=None, tune=None,
                           phong: Optional[dict] = None):
    """phong (only with act="sigmoid", Cout = 3, want32): dict(light_dir [B,3], light_col [B,3] fp32 device tensors, ambient,
    k_diffuse, background_white=False, with_mask=True, want_u8=True) -> the Phong composite is applied in the epilogue; returns
    (shaded fp32 image, uint8 image or None)."""
    x = _act_in(x, L.fmt, L.dtype)
    B, H, W, Cin = x.shape
    assert Cin == L.cin and W % L.F == 0
    ph, u8 = None, None
    if phong is not None:
        if act != "sigmoid" or L.cout != 3 or not want32 or want16:
            raise ValueError("the fused Phong epilogue needs the sigmoid 3-channel fp32 output layer")
        ld, lc = _cuda(phong["light_dir"], torch.float32), _cuda(phong["light_col"], torch.float32)
        if ld.shape[0] == 1 and B > 1:
            ld = ld.expand(B, 3).contiguous()
        if lc.shape[0] == 1 and B > 1:
            lc = lc.expand(B, 3).contiguous()
        assert tuple(ld.shape) == (B, 3) and tuple(lc.shape) == (B, 3)
        if phong.get("want_u8", True):
            u8 = torch.empty((B, H, W, 3), device=x.device, dtype=torch.uint8)
        ph = rn_phong()
        ph.light_dir, ph.light_col, ph.out_u8 = ld.data_ptr(), lc.data_ptr(), _ptr(u8)
        ph.ambient, ph.k_diffuse = float(phong["ambient"]), float(phong["k_diffuse"])
        ph.background_white, ph.with_mask = int(bool(phong.get("background_white", False))), int(bool(phong.get("with_mask", True)))
    out16, out32 = _out_buffers((B, H, W, L.cout), L.dtype, x.device, want16, want32, out16, out32, L.fmt)
    a = _ACT[act]
    alpha_x = None
    if a == ACT_PRELU:
        alpha_x = L._alpha.get(alpha_tag) if alpha_tag is not None else None
        if alpha_x is None:    # untagged alphas are recomputed, never cached by address
            alpha_x = L.tiled(alpha, x.device)
            if alpha_tag is not None:
                L._alpha[alpha_tag] = alpha_x
    check(lib.rn_conv2d_transpose_s1_xfold(x.data_ptr(), L.w.data_ptr(), L.bias.data_ptr(), _ptr(alpha_x), a, _ptr(out16),
                                           _ptr(out32), B, H, W, Cin, L.cout, L.kh, L.kw, L.F, L.cout_pad, L.fmt,
                                           C.byref(ph) if ph is not None else None, _tune(tune), _stream()),
          "rn_conv2d_transpose_s1_xfold")
    if ph is not None:
        return out32, u8
    return _ret(out16, out32, want16, want32, L.fmt)


def conv_igemm_raw(x, w_packed, bias, taps, ndim, B, H, W, D, Cin, Cout, cout_pad, out16=None, out32=None,
                   alpha=None, act=ACT_NONE, residual=None, o=None, fmt=0, force_bn=0, force_kps=0, max_ctas=0,
                   cluster=0, cta_group=0, ny=0, tile_w=0, msub=0, epi_groups=0, res_prefetch=0, tma_store=0):
    """Direct access to rn_conv_igemm for tests / tuning.  taps: list of (dx,dy,dz).  fmt 2: x, w_packed, out16 and a
    16-bit residual are [2, ...] hi/lo plane tensors (or Split16)."""
    n = len(taps)
    arr = (C.c_int8 * (3 * n))(*[v for t in taps for v in t])
    x, w_packed, out16, residual = _unwrap(x), _unwrap(w_packed), _unwrap(out16), _unwrap(residual)
    d = rn_conv_desc()
    d.ndim, d.B, d.H, d.W, d.D = ndim, B, H, W, D
    d.Cin, d.Cout, d.cout_pad, d.ntaps = Cin, Cout, cout_pad, n
    d.taps = C.cast(arr, C.c_void_p)
    d.x, d.w_packed, d.bias, d.alpha = x.data_ptr(), w_packed.data_ptr(), bias.data_ptr(), _ptr(alpha)
    d.act = act
    d.residual = _ptr(residual)
    d.residual_is_f32 = 1 if (residual is not None and residual.dtype == torch.float32) else 0
    d.out16, d.out32 = _ptr(out16), _ptr(out32)
    if o is None:
        if ndim == 2:
            o = (0, H * W * Cout, W * Cout, Cout, 0)
        else:
            o = (0, H * W * D * Cout, W * D * Cout, D * Cout, Cout)
    d.o_base, d.o_b, d.o_y, d.o_x, d.o_z = o
    d.fmt, d.force_bn, d.force_kps, d.max_ctas = fmt, force_bn, force_kps, max_ctas
    d.cluster = cluster
    d.cta_group = cta_group
    d.ny, d.tile_w, d.msub = ny, tile_w, msub
    d.epi_groups, d.res_prefetch, d.tma_store = epi_groups, res_prefetch, tma_store
    if fmt == 2:
        d.x_plane = x.numel() // 2
        d.w_plane = w_packed.numel() // 2
        d.o_plane = (out16.numel() // 2) if out16 is not None else 0
    check(lib.rn_conv_igemm(C.byref(d), _stream()), "rn_conv_igemm")


# --------------------------------------------------------------------------------------- thin conv3d
def conv3d_direct(x: torch.Tensor, w_tf: torch.Tensor, bias: torch.Tensor, alpha: Optional[torch.Tensor],
                  stride: Sequence[int], dtype: torch.dtype = torch.float16, fmt: Optional[int] = None):
    """CUDA-core SAME conv3d + bias + PReLU for the thin first layers.  x fp32 or 16-bit
    [B,H,W,D,Cin]; w_tf fp32 [k,k,k,Cin,Cout]; returns 16-bit (a Split16 pair for fmt 2)."""
    x = _cuda(x)
    fmt = fmt_of(dtype) if fmt is None else int(fmt)
    if isinstance(x, Split16) != (fmt == 2 and x.dtype != torch.float32):
        raise TypeError("conv3d_direct: 16-bit input format does not match fmt")
    w_tf = _cuda(w_tf, torch.float32)
    bias = _cuda(bias, torch.float32)
    B, H, W, D, Cin = x.shape
    k = w_tf.shape[0]
    Cout = w_tf.shape[4]
    sy, sx, sz = stride
    Ho, Wo, Do = -(-H // sy), -(-W // sx), -(-D // sz)
    out = _alloc16((B, Ho, Wo, Do, Cout), fmt, dtype, x.device)
    check(lib.rn_conv3d_direct(x.data_ptr(), 1 if x.dtype == torch.float32 else 0, w_tf.data_ptr(),
                               bias.data_ptr(), _ptr(alpha), out.data_ptr(), B, H, W, D, Cin, Cout, k, sy, sx, sz,
                               fmt, _stream()), "rn_conv3d_direct")
    return _wrap16(out, fmt)


def resample_conv1(vox: torch.Tensor, minv: torch.Tensor, new_size: int, w_tf: torch.Tensor, bias: torch.Tensor,
                   alpha: Optional[torch.Tensor], dtype: torch.dtype = torch.float16, fmt: Optional[int] = None):
    """Fused resampler + axis transform + e_conv1 (5^3 s2, 1->8) + bias + PReLU; empty tiles skip the conv.
    vox fp32 [B,S,S,S,1], minv fp32 [B,3,4], w_tf fp32 [5,5,5,1,8] -> 16-bit [B,new/2,new/2,new/2,8]."""
    vox = _cuda(vox, torch.float32)
    minv = _cuda(minv, torch.float32)
    w_tf = _cuda(w_tf, torch.float32)
    bias = _cuda(bias, torch.float32)
    B, S = vox.shape[0], vox.shape[1]
    if tuple(vox.shape) != (B, S, S, S, 1) or tuple(w_tf.shape) != (5, 5, 5, 1, 8) or tuple(minv.shape) != (B, 3, 4):
        raise ValueError(f"resample_conv1: unsupported shapes {tuple(vox.shape)}, {tuple(w_tf.shape)}")
    No = new_size // 2
    fmt = fmt_of(dtype) if fmt is None else int(fmt)
    out = _alloc16((B, No, No, No, 8), fmt, dtype, vox.device)
    check(lib.rn_resample_conv1_fused(vox.data_ptr(), minv.data_ptr(), w_tf.data_ptr(), bias.data_ptr(), _ptr(alpha),
                                      out.data_ptr(), B, S, new_size, fmt, _stream()),
          "rn_resample_conv1_fused")
    return _wrap16(out, fmt)


def resample5_conv1(vox: torch.Tensor, tex: torch.Tensor, minv: torch.Tensor, new_size: int, w_tf: torch.Tensor,
                    bias: torch.Tensor, alpha: Optional[torch.Tensor], dtype: torch.dtype = torch.float16,
                    fmt: Optional[int] = None):
    """Texture net input chain in one kernel (rn_resample5_conv1_fused): resample geometry (C = 1) and texture volume (C = 4)
    with one pose + axis transform + concat + e_conv1 (5^3 s2, 5 -> 8) + bias + PReLU.
    vox fp32 [B,S,S,S,1], tex fp32 [B,S,S,S,4], minv fp32 [B,3,4], w_tf fp32 [5,5,5,5,8] -> 16-bit [B,new/2,new/2,new/2,8]."""
    vox, tex, minv = _cuda(vox, torch.float32), _cuda(tex, torch.float32), _cuda(minv, torch.float32)
    w_tf, bias = _cuda(w_tf, torch.float32), _cuda(bias, torch.float32)
    B, S = vox.shape[0], vox.shape[1]
    if (tuple(vox.shape) != (B, S, S, S, 1) or tuple(tex.shape) != (B, S, S, S, 4) or tuple(w_tf.shape) != (5, 5, 5, 5, 8)
            or tuple(minv.shape) != (B, 3, 4)):
        raise ValueError(f"resample5_conv1: unsupported shapes {tuple(vox.shape)}, {tuple(tex.shape)}, {tuple(w_tf.shape)}")
    No = new_size // 2
    fmt = fmt_of(dtype) if fmt is None else int(fmt)
    out = _alloc16((B, No, No, No, 8), fmt, dtype, vox.device)
    check(lib.rn_resample5_conv1_fused(vox.data_ptr(), tex.data_ptr(), minv.data_ptr(), w_tf.data_ptr(), bias.data_ptr(),
                                       _ptr(alpha), out.data_ptr(), B, S, new_size, fmt, _stream()), "rn_resample5_conv1_fused")
    return _wrap16(out, fmt)


def binvox_decode(pairs_list, dims, fix_coords: bool = True, device="cuda") -> torch.Tensor:
    """Run-length (value, count) byte pairs of n binvox payloads -> float32 [n, d0, d2, d1, 1] on the device."""
    import numpy as np
    d0, d1, d2 = (int(v) for v in dims)
    kept, starts, first = [], [], [0]
    for pairs in pairs_list:
        pairs = np.asarray(pairs, np.uint8).reshape(-1, 2)
        pairs = pairs[pairs[:, 1] != 0]                       # zero-length runs carry no voxels
        cnt = pairs[:, 1].astype(np.int64)
        if int(cnt.sum()) != d0 * d1 * d2:
            raise ValueError(f"binvox payload decodes to {int(cnt.sum())} voxels, dims say {d0 * d1 * d2}")
        kept.append(pairs)
        starts.append(np.cumsum(cnt) - cnt)
        first.append(first[-1] + pairs.shape[0])
    pairs_d = torch.from_numpy(np.ascontiguousarray(np.concatenate(kept))).to(device)
    starts_d = torch.from_numpy(np.concatenate(starts).astype(np.int32)).to(device)
    first_d = torch.tensor(first, dtype=torch.int32, device=device)
    n = len(kept)
    shape = (n, d0, d2, d1, 1) if fix_coords else (n, d0, d1, d2, 1)
    out = torch.empty(shape, device=device, dtype=torch.float32)
    check(lib.rn_binvox_decode(pairs_d.data_ptr(), starts_d.data_ptr(), first_d.data_ptr(), out.data_ptr(), n, d0, d1, d2,
                               1 if fix_coords else 0, _stream()), "rn_binvox_decode")
    return out


# --------------------------------------------------------------------------------------- misc
def cast_to_16(x: torch.Tensor, dtype: torch.dtype = torch.float16, fmt: Optional[int] = None):
    """fp32 -> 16-bit (fmt 2: fp16 hi/lo pair, returned as Split16)."""
    x = _cuda(x, torch.float32)
    fmt = fmt_of(dtype) if fmt is None else int(fmt)
    out = _alloc16(x.shape, fmt, dtype, x.device)
    check(lib.rn_cast_f32_to_16(x.data_ptr(), out.data_ptr(), x.numel(), x.numel(), fmt, _stream()), "cast")
    return _wrap16(out, fmt)


def cast_to_f32(x) -> torch.Tensor:
    x = _cuda(x)
    fmt = 2 if isinstance(x, Split16) else fmt_of(x.dtype)
    out = torch.empty(x.shape, device=x.device, dtype=torch.float32)
    check(lib.rn_cast_16_to_f32(x.data_ptr(), out.data_ptr(), x.numel(), fmt, _stream()), "cast")
    return out


def phong_composite(img: torch.Tensor, light_dir: torch.Tensor, light_col: torch.Tensor, ambient: float,
                    k_diffuse: float, background_white: bool = False, with_mask: bool = True,
                    want_u8: bool = False):
    img = _cuda(img, torch.float32)
    B, H, W, _ = img.shape
    light_dir = _cuda(light_dir.to(device=img.device, dtype=torch.float32))
    light_col = _cuda(light_col.to(device=img.device, dtype=torch.float32))
    if light_dir.shape[0] == 1 and B > 1:
        light_dir = light_dir.expand(B, 3).contiguous()
    if light_col.shape[0] == 1 and B > 1:
        light_col = light_col.expand(B, 3).contiguous()
    out = torch.empty_like(img)
    u8 = torch.empty(img.shape, device=img.device, dtype=torch.uint8) if want_u8 else None
    check(lib.rn_phong_composite(img.data_ptr(), light_dir.data_ptr(), light_col.data_ptr(), float(ambient),
                                 float(k_diffuse), 1 if background_white else 0, 1 if with_mask else 0,
                                 out.data_ptr(), _ptr(u8), B, H, W, _stream()), "rn_phong_composite")
    return (out, u8) if want_u8 else out


def bias_act(x, bias: Optional[torch.Tensor], alpha: Optional[torch.Tensor], act: Optional[str],
             residual=None, want32: bool = False, fmt: int = 0):
    """y = act(x + bias[c]) + residual on a 16-bit channel-last tensor (rn_bias_act_16).  An fp32 `x` is first cast to
    the 16-bit format `fmt`; a Split16 `x` selects fmt 2."""
    x = _cuda(x)
    if isinstance(x, Split16):
        fmt = 2
    elif x.dtype == torch.float32:
        x = cast_to_16(x, fmt=fmt)
    else:
        fmt = fmt_of(x.dtype)
    C_ = x.shape[-1]
    a = _ACT[act]
    dev = x.device
    if bias is not None:
        bias = _cuda(bias.to(device=dev, dtype=torch.float32))
    if alpha is not None:
        alpha = _cuda(alpha.to(device=dev, dtype=torch.float32))
    if residual is not None:
        residual = _cuda(residual)
        if isinstance(residual, Split16) != (fmt == 2) or (fmt != 2 and residual.dtype != x.dtype):
            residual = cast_to_16(residual.float() if not isinstance(residual, torch.Tensor) or residual.dtype != torch.float32
                                  else residual, fmt=fmt)
    out16 = None if want32 else _alloc16(x.shape, fmt, torch.float16 if fmt != 1 else torch.bfloat16, dev)
    out32 = torch.empty(x.shape, device=dev, dtype=torch.float32) if want32 else None
    check(lib.rn_bias_act_16(x.data_ptr(), _ptr(bias), _ptr(alpha), a, _ptr(residual), _ptr(out16), _ptr(out32),
                             x.numel(), C_, fmt, _stream()), "rn_bias_act_16")
    return out32 if want32 else _wrap16(out16, fmt)


# --------------------------------------------------------------------------------------- texture decoder (config 4)
def fully_connected(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor], alpha: Optional[torch.Tensor],
                    want32: bool = True, dtype: torch.dtype = torch.float16, fmt: Optional[int] = None):
    """y = prelu(x @ w + bias; alpha).  x [B,K] fp32, w [K,N] fp32 (TF layout) -> [B,N] fp32, or 16-bit in the format
    `fmt` or else `dtype` picks (fmt 2: fp16 hi/lo pair, returned as Split16)."""
    x = _cuda(x, torch.float32)
    w = _cuda(w, torch.float32)
    B, K = x.shape
    N = w.shape[1]
    fmt = fmt_of(dtype) if fmt is None else int(fmt)
    out = (torch.empty((B, N), device=x.device, dtype=torch.float32) if want32
           else _alloc16((B, N), fmt, torch.bfloat16 if fmt == 1 else torch.float16, x.device))
    check(lib.rn_fully_connected(x.data_ptr(), w.data_ptr(), _ptr(bias), _ptr(alpha), None if want32 else out.data_ptr(),
                                 out.data_ptr() if want32 else None, B, K, N, fmt, _stream()),
          "rn_fully_connected")
    return out if want32 else _wrap16(out, fmt)


def conv3d_small(x, w_tf: torch.Tensor, bias: Optional[torch.Tensor], alpha: Optional[torch.Tensor],
                 stride: int, transposed: bool, want32: bool = True, dtype: torch.dtype = torch.float16,
                 fmt: Optional[int] = None):
    """Thin (<= 8 channel) conv3d / conv3d_transpose, TF SAME, + bias + PReLU.  x [B,H,W,D,Cin] fp32, 16-bit or Split16;
    w_tf fp32 [k,k,k,Cin,Cout] (forward) or [k,k,k,Cout,Cin] (transposed).  The kernel reads and writes ONE 16-bit format:
    a 16-bit x sets it (a 16-bit output then has x's format); for an fp32 x, `fmt` or else `dtype` picks the output's."""
    x = _cuda(x)
    w_tf = _cuda(w_tf, torch.float32)
    x_is_f32 = isinstance(x, torch.Tensor) and x.dtype == torch.float32
    if not x_is_f32:
        fx = 2 if isinstance(x, Split16) else fmt_of(x.dtype)
        if fmt is not None and int(fmt) != fx:
            raise TypeError(f"conv3d_small: a 16-bit input of format {fx} gives output format {fx}, not {fmt}")
        fmt = fx
    elif fmt is None:
        fmt = fmt_of(dtype)
    B, H, W, D, Cin = x.shape
    k = w_tf.shape[0]
    Cout = w_tf.shape[3] if transposed else w_tf.shape[4]
    if transposed:
        oshape = (B, H * stride, W * stride, D * stride, Cout)
    else:
        oshape = (B, -(-H // stride), -(-W // stride), -(-D // stride), Cout)
    out = (torch.empty(oshape, device=x.device, dtype=torch.float32) if want32
           else _alloc16(oshape, fmt, torch.bfloat16 if fmt == 1 else torch.float16, x.device))
    check(lib.rn_conv3d_small(x.data_ptr(), 1 if x_is_f32 else 0, w_tf.data_ptr(), _ptr(bias),
                              _ptr(alpha), None if want32 else out.data_ptr(), out.data_ptr() if want32 else None,
                              B, H, W, D, Cin, Cout, k, stride, 1 if transposed else 0, fmt, _stream()), "rn_conv3d_small")
    return out if want32 else _wrap16(out, fmt)


ACT_ELU = 3
_ACT_F32 = {None: ACT_NONE, "none": ACT_NONE, "elu": ACT_ELU, "sigmoid": ACT_SIGMOID}


def conv3d_f32(x: torch.Tensor, w_tf: torch.Tensor, bias: Optional[torch.Tensor], stride: int, transposed: bool,
               act: Optional[str] = None) -> torch.Tensor:
    """fp32 conv3d / conv3d_transpose, cubic k = 4, TF SAME, any channel count (rn_conv3d_f32: the shape decoder's layers and
    their data gradients), + bias, then act None / "elu" / "sigmoid".  x fp32 [B,H,W,D,Cin]; w_tf fp32 [4,4,4,Cin,Cout] (forward)
    or [4,4,4,Cout,Cin] (transposed).  Reproducible bit for bit."""
    x, w_tf = _cuda(x, torch.float32), _cuda(w_tf, torch.float32)
    if act not in _ACT_F32:
        raise ValueError(f"conv3d_f32: activation {act!r} is not one of {sorted(k for k in _ACT_F32 if k)}")
    B, H, W, D, Cin = (int(v) for v in x.shape)
    if tuple(w_tf.shape[:3]) != (4, 4, 4):
        raise ValueError(f"conv3d_f32: cubic k = 4 filters only, got {tuple(w_tf.shape)}")
    wc = int(w_tf.shape[4] if transposed else w_tf.shape[3])
    if wc != Cin:
        raise ValueError(f"conv3d_f32: filter {tuple(w_tf.shape)} does not take {Cin} input channels")
    Cout = int(w_tf.shape[3] if transposed else w_tf.shape[4])
    s = int(stride)
    oshape = (B, H * s, W * s, D * s, Cout) if transposed else (B, -(-H // s), -(-W // s), -(-D // s), Cout)
    tr = 1 if transposed else 0
    nwork = int(lib.rn_conv3d_f32_workspace(B, H, W, D, Cin, Cout, s, tr))
    if nwork < 0:
        check(int(nwork), "rn_conv3d_f32_workspace")
    work = torch.empty(nwork, device=x.device, dtype=torch.float32) if nwork > 0 else None
    if bias is not None:
        bias = _cuda(bias, torch.float32)
    out = torch.empty(oshape, device=x.device, dtype=torch.float32)
    check(lib.rn_conv3d_f32(x.data_ptr(), w_tf.data_ptr(), _ptr(bias), out.data_ptr(), _ptr(work), B, H, W, D, Cin, Cout, 4, s, tr,
                            _ACT_F32[act], _stream()), "rn_conv3d_f32")
    return out


def act_backward_f32(g: torch.Tensor, y: torch.Tensor, act: str) -> torch.Tensor:
    """dL/dz from dL/dy and the activation's output y, fp32 (rn_act_backward_f32): "elu" -> y < 0 ? g (y + 1) : g (TF-1 EluGrad),
    "sigmoid" -> g y (1 - y)."""
    g, y = _cuda(g, torch.float32), _cuda(y, torch.float32)
    if tuple(g.shape) != tuple(y.shape):
        raise ValueError(f"act_backward_f32: g {tuple(g.shape)} and y {tuple(y.shape)} differ")
    if act not in ("elu", "sigmoid"):
        raise ValueError(f"act_backward_f32: no derivative for {act!r}")
    out = torch.empty_like(g)
    check(lib.rn_act_backward_f32(g.data_ptr(), y.data_ptr(), out.data_ptr(), g.numel(), _ACT_F32[act], _stream()),
          "rn_act_backward_f32")
    return out


def concat_channels(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """tf.concat([a, b], axis=-1) for fp32 channel-last tensors."""
    a = _cuda(a, torch.float32)
    b = _cuda(b, torch.float32)
    assert a.shape[:-1] == b.shape[:-1]
    Ca, Cb = a.shape[-1], b.shape[-1]
    out = torch.empty(tuple(a.shape[:-1]) + (Ca + Cb,), device=a.device, dtype=torch.float32)
    check(lib.rn_concat_channels_f32(a.data_ptr(), b.data_ptr(), out.data_ptr(), a.numel() // Ca, Ca, Cb, _stream()),
          "rn_concat_channels_f32")
    return out


# --------------------------------------------------------------------------------------- backward (input gradients)
def conv2d_taps(x, w_packed, bias, taps, cout: int, cout_pad: int, fmt: int, residual=None, ny: int = 0, want32: bool = False,
                dtype: torch.dtype = torch.float16):
    """Stride-1 2-D convolution with an explicit tap list (dx, dy) over the packed filter [ntaps][cout_pad][Cin]
    (rn_conv_igemm): what the data gradients of the k = 4 convolutions need (their mirrored taps are not a TF SAME set).
    x: 16-bit [B,H,W,Cin] (Split16 for fmt 2); returns 16-bit [B,H,W,cout] (or fp32 with want32)."""
    x = _act_in(x, fmt, dtype)
    B, H, W, Cin = x.shape
    out16 = None if want32 else _alloc16((B, H, W, cout), fmt, dtype, x.device)
    out32 = torch.empty((B, H, W, cout), device=x.device, dtype=torch.float32) if want32 else None
    residual, _ = _residual(residual, fmt)
    conv_igemm_raw(x, w_packed, bias, [(int(t[0]), int(t[1]), 0) for t in taps], 2, B, H, W, 1, Cin, cout, cout_pad,
                   out16=out16, out32=out32, residual=residual, fmt=fmt, ny=ny)
    return out32 if want32 else _wrap16(out16, fmt)


def prelu_backward(g, y, alpha: torch.Tensor):
    """dL/d(pre) = g * (y > 0 ? 1 : alpha[c]) (rn_prelu_backward_16); g, y 16-bit tensors of one format, alpha fp32 [C]."""
    g, y = _cuda(g), _cuda(y)
    fmt = 2 if isinstance(g, Split16) else fmt_of(g.dtype)
    if isinstance(y, Split16) != (fmt == 2) or tuple(g.shape) != tuple(y.shape):
        raise TypeError("prelu_backward: g and y must have the same shape and 16-bit format")
    C_ = g.shape[-1]
    alpha = _cuda(alpha.to(device=g.device, dtype=torch.float32))
    assert alpha.numel() >= C_
    out = _alloc16(g.shape, fmt, torch.float16 if fmt != 1 else torch.bfloat16, g.device)
    check(lib.rn_prelu_backward_16(g.data_ptr(), y.data_ptr(), alpha.data_ptr(), out.data_ptr(), g.numel(), C_, fmt, _stream()),
          "rn_prelu_backward_16")
    return _wrap16(out, fmt)


def sigmoid_backward(g: torch.Tensor, img: torch.Tensor, c_pad: int, scale: float, fmt: int):
    """scale * g * img * (1 - img), zero padded to c_pad channels, as a 16-bit tensor [..., c_pad] (rn_sigmoid_backward)."""
    g, img = _cuda(g, torch.float32), _cuda(img, torch.float32)
    assert g.shape == img.shape
    Cc = img.shape[-1]
    shape = tuple(img.shape[:-1]) + (c_pad,)
    out = _alloc16(shape, fmt, torch.float16, img.device)
    check(lib.rn_sigmoid_backward(g.data_ptr(), img.data_ptr(), out.data_ptr(), img.numel() // Cc, Cc, c_pad, float(scale), fmt,
                                  _stream()), "rn_sigmoid_backward")
    return _wrap16(out, fmt)


def conv3d_backward_data_direct(g, w_tf: torch.Tensor, in_shape, stride: Sequence[int], want32: bool = False,
                                out_scale: float = 1.0):
    """Data gradient of a thin strided SAME conv3d: g 16-bit [B,Ho,Wo,Do,Cout], w_tf fp32 [k,k,k,Cin,Cout], in_shape =
    (B,H,W,D,Cin) of the forward input -> 16-bit (or fp32 x out_scale) gradient of that shape."""
    g = _cuda(g)
    fmt = 2 if isinstance(g, Split16) else fmt_of(g.dtype)
    w_tf = _cuda(w_tf, torch.float32)
    B, H, W, D, Cin = (int(v) for v in in_shape)
    k, Cout = int(w_tf.shape[0]), int(w_tf.shape[4])
    out16 = None if want32 else _alloc16((B, H, W, D, Cin), fmt, torch.float16, g.device)
    out32 = torch.empty((B, H, W, D, Cin), device=g.device, dtype=torch.float32) if want32 else None
    check(lib.rn_conv3d_backward_data_direct(g.data_ptr(), w_tf.data_ptr(), _ptr(out16), _ptr(out32), B, H, W, D, Cin, Cout, k,
                                             int(stride[0]), int(stride[1]), int(stride[2]), float(out_scale), fmt, _stream()),
          "rn_conv3d_backward_data_direct")
    return out32 if want32 else _wrap16(out16, fmt)


def resample_backward(vox: torch.Tensor, minv: torch.Tensor, gout: torch.Tensor, transform: bool, want_dvox: bool = True,
                      want_dminv: bool = True):
    """Backward of `resample`: gout fp32 [B,N,N,N,C] -> (dvox [B,S,S,S,C] or None, dminv [B,3,4] or None), fp32."""
    vox, minv, gout = _cuda(vox, torch.float32), _cuda(minv, torch.float32), _cuda(gout, torch.float32)
    B, S, _, _, Cc = vox.shape
    N = gout.shape[1]
    dvox = torch.zeros_like(vox) if want_dvox else None
    dminv = torch.zeros_like(minv) if want_dminv else None
    check(lib.rn_resample_backward_f32(vox.data_ptr(), minv.data_ptr(), gout.data_ptr(), _ptr(dvox), _ptr(dminv), B, Cc, S, N,
                                       1 if transform else 0, _stream()), "rn_resample_backward_f32")
    return dvox, dminv


def resample5_backward(vox: torch.Tensor, tex: torch.Tensor, minv: torch.Tensor, gout: torch.Tensor, want_dvox: bool = True,
                       want_dtex: bool = True, want_dminv: bool = True):
    """Backward of `resample5_conv1`'s input chain (rn_resample5_backward_f32): gout = dL/d(concat) fp32 [B,N,N,N,5] ->
    (dvox [B,S,S,S,1], dtex [B,S,S,S,4], dminv [B,3,4]), fp32, each None unless asked for."""
    vox, tex, minv, gout = (_cuda(t, torch.float32) for t in (vox, tex, minv, gout))
    B, S = vox.shape[0], vox.shape[1]
    N = gout.shape[1]
    if (tuple(vox.shape) != (B, S, S, S, 1) or tuple(tex.shape) != (B, S, S, S, 4) or tuple(minv.shape) != (B, 3, 4)
            or tuple(gout.shape) != (B, N, N, N, 5)):
        raise ValueError(f"resample5_backward: unsupported shapes {tuple(vox.shape)}, {tuple(tex.shape)}, {tuple(gout.shape)}")
    dvox = torch.zeros_like(vox) if want_dvox else None
    dtex = torch.zeros_like(tex) if want_dtex else None
    dminv = torch.zeros_like(minv) if want_dminv else None
    check(lib.rn_resample5_backward_f32(vox.data_ptr(), tex.data_ptr(), minv.data_ptr(), gout.data_ptr(), _ptr(dvox), _ptr(dtex),
                                        _ptr(dminv), B, S, N, _stream()), "rn_resample5_backward_f32")
    return dvox, dtex, dminv


def prelu_backward_f32(g: torch.Tensor, z: torch.Tensor, alpha: torch.Tensor) -> torch.Tensor:
    """dL/dz = g * (z > 0 ? 1 : alpha[c]) on fp32 tensors (rn_prelu_backward_f32); z is the pre-activation, alpha fp32 [C]."""
    g, z = _cuda(g, torch.float32), _cuda(z, torch.float32)
    if tuple(g.shape) != tuple(z.shape):
        raise ValueError(f"prelu_backward_f32: g {tuple(g.shape)} and z {tuple(z.shape)} differ")
    C_ = g.shape[-1]
    alpha = _cuda(alpha.to(device=g.device, dtype=torch.float32))
    if alpha.numel() < C_:
        raise ValueError(f"prelu_backward_f32: {alpha.numel()} slopes for {C_} channels")
    out = torch.empty_like(g)
    check(lib.rn_prelu_backward_f32(g.data_ptr(), z.data_ptr(), alpha.data_ptr(), out.data_ptr(), g.numel(), C_, _stream()),
          "rn_prelu_backward_f32")
    return out


def fully_connected_backward_data(g: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """dx = g @ w.T (rn_fully_connected_backward_data): g fp32 [B,N], w fp32 [K,N] (TF layout) -> fp32 [B,K], reproducible bit
    for bit (fixed-order split-N reduction)."""
    g, w = _cuda(g, torch.float32), _cuda(w, torch.float32)
    B, N = g.shape
    K = w.shape[0]
    if tuple(w.shape) != (K, N):
        raise ValueError(f"fully_connected_backward_data: w {tuple(w.shape)} does not match g {tuple(g.shape)}")
    work = torch.empty(int(lib.rn_fully_connected_backward_workspace(B, K, N)), device=g.device, dtype=torch.float32)
    dx = torch.empty((B, K), device=g.device, dtype=torch.float32)
    check(lib.rn_fully_connected_backward_data(g.data_ptr(), w.data_ptr(), work.data_ptr(), dx.data_ptr(), B, K, N, _stream()),
          "rn_fully_connected_backward_data")
    return dx


def phong_recon_loss_grad(albedo: torch.Tensor, normal: torch.Tensor, target: torch.Tensor, light_dir: torch.Tensor,
                          light_col: torch.Tensor, ambient: float = 0.0, k_diffuse: float = 1.0, black_background: bool = False,
                          with_mask: bool = True):
    """Face reconstruction objective (rn_phong_recon_loss_grad): loss[b] = mean (target - albedo * tf_phong_composite(normal,
    light_dir, light_col, ...))^2 and its gradients.  albedo, normal, target fp32 [B,H,W,3]; light_dir, light_col [B,3] (or [1,3]).
    Returns (loss fp64 [B], d_albedo, d_normal fp32 [B,H,W,3], d_light_dir fp32 [B,3])."""
    albedo, normal, target = (_cuda(t, torch.float32) for t in (albedo, normal, target))
    B, H, W, C3 = albedo.shape
    if C3 != 3 or tuple(normal.shape) != tuple(albedo.shape) or tuple(target.shape) != tuple(albedo.shape):
        raise ValueError(f"phong_recon_loss_grad: shapes {tuple(albedo.shape)}, {tuple(normal.shape)}, {tuple(target.shape)}")
    ld, lc = (_cuda(t.to(device=albedo.device, dtype=torch.float32).reshape(-1, 3).expand(B, 3).contiguous(), torch.float32)
              for t in (light_dir, light_col))
    loss = torch.zeros(B, device=albedo.device, dtype=torch.float64)
    d_albedo, d_normal = torch.empty_like(albedo), torch.empty_like(albedo)
    d_light = torch.zeros((B, 3), device=albedo.device, dtype=torch.float32)
    check(lib.rn_phong_recon_loss_grad(albedo.data_ptr(), normal.data_ptr(), target.data_ptr(), ld.data_ptr(), lc.data_ptr(),
                                       float(ambient), float(k_diffuse), 1 if black_background else 0, 1 if with_mask else 0,
                                       loss.data_ptr(), d_albedo.data_ptr(), d_normal.data_ptr(), d_light.data_ptr(), B, H, W,
                                       _stream()), "rn_phong_recon_loss_grad")
    return loss, d_albedo, d_normal, d_light


def conv2d_weight_grad(x, g, kh: int, kw: int) -> torch.Tensor:
    """dW of a stride-1 SAME conv2d on the tensor cores (rn_conv2d_weight_grad): x 16-bit [B,H,W,Cin] (layer input), g 16-bit
    [B,H,W,Cout] (gradient of the conv output), same 16-bit format -> fp32 [kh,kw,Cin,Cout] (TF filter layout)."""
    x, g = _cuda(x), _cuda(g)
    fmt = 2 if isinstance(x, Split16) else fmt_of(x.dtype)
    if isinstance(g, Split16) != (fmt == 2):
        raise TypeError("conv2d_weight_grad: x and g must share the 16-bit format")
    B, H, W, Cin = x.shape
    Cout = g.shape[-1]
    assert tuple(g.shape[:3]) == (B, H, W)
    dw = torch.empty((kh, kw, Cin, Cout), device=x.device, dtype=torch.float32)
    check(lib.rn_conv2d_weight_grad(x.data_ptr(), g.data_ptr(), dw.data_ptr(), B, H, W, Cin, Cout, kh, kw, fmt, _stream()),
          "rn_conv2d_weight_grad")
    return dw


def bias_grad(g) -> torch.Tensor:
    """db[c] = sum over pixels of a 16-bit channel-last gradient tensor (rn_bias_grad_16) -> fp32 [C]."""
    g = _cuda(g)
    fmt = 2 if isinstance(g, Split16) else fmt_of(g.dtype)
    Cc = g.shape[-1]
    db = torch.empty(Cc, device=g.device, dtype=torch.float32)
    check(lib.rn_bias_grad_16(g.data_ptr(), db.data_ptr(), g.numel() // Cc, Cc, fmt, _stream()), "rn_bias_grad_16")
    return db


# --------------------------------------------------------------------------------------------- training step (rn_train.cu)
def _fmt_any(t) -> int:
    if isinstance(t, Split16):
        return 2
    return 3 if t.dtype == torch.float32 else fmt_of(t.dtype)


def same_pad_before(n_in: int, k: int, s: int) -> int:
    """TF SAME padding in front of a dimension (tools/layer_util.py conv wrappers all use padding='SAME')."""
    n_out = -(-n_in // s)
    return max((n_out - 1) * s + k - n_in, 0) // 2


def conv_weight_grad_direct(P, Q, ksize: Sequence[int], stride: Sequence[int], pad: Sequence[int], Ca: Optional[int] = None,
                            Cb: Optional[int] = None, scale: float = 1.0) -> torch.Tensor:
    """dW[tap][a][b] = scale * sum_pos P[pos][a] * Q[pos*stride + tap - pad][b] (rn_conv_weight_grad_direct): P on the coarse
    grid, Q on the fine grid, channel-last, 4-D ([B,H,W,C]: 2-D conv) or 5-D ([B,d1,d2,d3,C]); 16-bit / Split16 / fp32 each.
    Ca / Cb: channels actually used (<= the tensors' channel pitch).  -> fp32 [*ksize, Ca, Cb]."""
    P, Q = _cuda(P), _cuda(Q)
    if len(P.shape) == 4:
        P5, Q5 = (P.shape[0], 1) + tuple(P.shape[1:]), (Q.shape[0], 1) + tuple(Q.shape[1:])
        ks, st, pd = (1,) + tuple(ksize), (1,) + tuple(stride), (0,) + tuple(pad)
    else:
        P5, Q5, ks, st, pd = tuple(P.shape), tuple(Q.shape), tuple(ksize), tuple(stride), tuple(pad)
    B, Dp, Hp, Wp, Cap = (int(v) for v in P5)
    _, Dq, Hq, Wq, Cbp = (int(v) for v in Q5)
    assert int(Q5[0]) == B
    Ca, Cb = int(Ca or Cap), int(Cb or Cbp)
    dW = torch.empty(tuple(int(k) for k in ksize) + (Ca, Cb), device=P.device, dtype=torch.float32)
    check(lib.rn_conv_weight_grad_direct(P.data_ptr(), Q.data_ptr(), dW.data_ptr(), B, Dp, Hp, Wp, Ca, Cap, Dq, Hq, Wq, Cb, Cbp,
                                         int(ks[0]), int(ks[1]), int(ks[2]), int(st[0]), int(st[1]), int(st[2]),
                                         int(pd[0]), int(pd[1]), int(pd[2]), _fmt_any(P), _fmt_any(Q), float(scale), _stream()),
          "rn_conv_weight_grad_direct")
    return dW


def prelu_alpha_grad(g, z, scale: float = 1.0) -> torch.Tensor:
    """dalpha[c] = scale * sum_{z<0} g*z over a channel-last pair of 16-bit tensors (rn_prelu_alpha_grad) -> fp32 [C]."""
    g, z = _cuda(g), _cuda(z)
    fmt = 2 if isinstance(g, Split16) else fmt_of(g.dtype)
    if isinstance(z, Split16) != (fmt == 2) or tuple(z.shape) != tuple(g.shape):
        raise TypeError("prelu_alpha_grad: g and z must share shape and 16-bit format")
    Cc = int(g.shape[-1])
    da = torch.empty(Cc, device=g.device, dtype=torch.float32)
    check(lib.rn_prelu_alpha_grad(g.data_ptr(), z.data_ptr(), da.data_ptr(), g.numel(), Cc, fmt, float(scale), _stream()),
          "rn_prelu_alpha_grad")
    return da


def fully_connected_param_grad(x: torch.Tensor, gy: torch.Tensor, z: torch.Tensor, alpha: torch.Tensor, want_gz: bool = False):
    """Parameter gradient of y = prelu(x @ w + b; alpha) (rn_fully_connected_param_grad): x fp32 [B,K], gy = dL/dy and the
    pre-activation z fp32 [B,N], alpha fp32 [N] -> (gz = dL/dz [B,N] or None, dW [K,N], db [N], dalpha [N]), fp32, reproducible
    bit for bit.  B <= 32, N % 4 == 0."""
    x, gy, z, alpha = (_cuda(t, torch.float32) for t in (x, gy, z, alpha))
    B, K = (int(v) for v in x.shape)
    N = int(gy.shape[1])
    if tuple(gy.shape) != (B, N) or tuple(z.shape) != (B, N) or alpha.numel() != N:
        raise ValueError(f"fully_connected_param_grad: x {tuple(x.shape)}, gy {tuple(gy.shape)}, z {tuple(z.shape)}, "
                         f"alpha {tuple(alpha.shape)} do not match")
    gz = torch.empty_like(gy) if want_gz else None
    dw = torch.empty((K, N), device=x.device, dtype=torch.float32)
    db = torch.empty(N, device=x.device, dtype=torch.float32)
    da = torch.empty(N, device=x.device, dtype=torch.float32)
    check(lib.rn_fully_connected_param_grad(x.data_ptr(), gy.data_ptr(), z.data_ptr(), alpha.data_ptr(), _ptr(gz), dw.data_ptr(),
                                            db.data_ptr(), da.data_ptr(), B, K, N, _stream()), "rn_fully_connected_param_grad")
    return gz, dw, db, da


def prelu_grad_f32(gy: torch.Tensor, z: torch.Tensor, alpha: torch.Tensor):
    """(gz = gy * (z > 0 ? 1 : alpha[c]), db[c] = sum gz, dalpha[c] = sum_{z<0} gy * z) of an fp32 channel-last layer with C = 4
    or 8 channels (rn_prelu_grad_f32); z is the pre-activation."""
    gy, z = _cuda(gy, torch.float32), _cuda(z, torch.float32)
    if tuple(gy.shape) != tuple(z.shape):
        raise ValueError(f"prelu_grad_f32: gy {tuple(gy.shape)} and z {tuple(z.shape)} differ")
    Cc = int(gy.shape[-1])
    alpha = _cuda(alpha.to(device=gy.device, dtype=torch.float32))
    if alpha.numel() != Cc:
        raise ValueError(f"prelu_grad_f32: {alpha.numel()} slopes for {Cc} channels")
    gz = torch.empty_like(gy)
    db = torch.empty(Cc, device=gy.device, dtype=torch.float32)
    da = torch.empty(Cc, device=gy.device, dtype=torch.float32)
    check(lib.rn_prelu_grad_f32(gy.data_ptr(), z.data_ptr(), alpha.data_ptr(), gz.data_ptr(), db.data_ptr(), da.data_ptr(),
                                gy.numel(), Cc, _stream()), "rn_prelu_grad_f32")
    return gz, db, da


def dropout(x, keep: float, seed: int, salt: int):
    """tf.nn.dropout on a 16-bit activation (rn_dropout_16): x / keep where kept, 0 elsewhere; the mask is a pure function of
    (seed, salt, element index), so calling this on the gradient with the same (seed, salt) is the backward pass."""
    x = _cuda(x)
    fmt = 2 if isinstance(x, Split16) else fmt_of(x.dtype)
    out = _alloc16(tuple(x.shape), fmt, torch.float16 if fmt == 2 else x.dtype, x.device)
    check(lib.rn_dropout_16(x.data_ptr(), out.data_ptr(), x.numel(), float(keep), int(seed) & 0xFFFFFFFF, int(salt) & 0xFFFFFFFF,
                            fmt, _stream()), "rn_dropout_16")
    return _wrap16(out, fmt)


def dropout_mask_host(n: int, keep: float, seed: int, salt: int):
    """The mask rn_dropout_16 applies, recomputed on the host (NumPy uint8 [n], 1 = kept)."""
    import numpy as np
    m = np.empty(int(n), np.uint8)
    check(lib.rn_dropout_mask_host(m.ctypes.data, int(n), float(keep), int(seed) & 0xFFFFFFFF, int(salt) & 0xFFFFFFFF),
          "rn_dropout_mask_host")
    return m


def image_loss_grad(img: torch.Tensor, target: torch.Tensor, kind: str = "mse", want_grad: bool = True):
    """Reconstruction loss of RenderNet_Shader.py:158-163 ("mse" | "bce") and dL/dimg (rn_image_loss_grad)
    -> (loss: 0-d float64 device tensor, dimg fp32 like img or None)."""
    img, target = _cuda(img, torch.float32), _cuda(target, torch.float32)
    assert tuple(img.shape) == tuple(target.shape) and img.is_contiguous() and target.is_contiguous()
    loss = torch.empty((), device=img.device, dtype=torch.float64)
    dimg = torch.empty_like(img) if want_grad else None
    check(lib.rn_image_loss_grad(img.data_ptr(), target.data_ptr(), _ptr(dimg), loss.data_ptr(), img.numel(), int(img.shape[0]),
                                 {"mse": 0, "bce": 1}[kind], _stream()), "rn_image_loss_grad")
    return loss, dimg


def adam_step(param: torch.Tensor, grad: torch.Tensor, m: torch.Tensor, v: torch.Tensor, lr_t: float, beta1: float, beta2: float,
              eps: float):
    """In-place tf.train.AdamOptimizer update of one fp32 device parameter (rn_adam_step)."""
    for t in (param, grad, m, v):
        if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()) or t.numel() != param.numel():
            raise TypeError("adam_step: contiguous fp32 CUDA tensors of one size expected")
    check(lib.rn_adam_step(param.data_ptr(), grad.data_ptr(), m.data_ptr(), v.data_ptr(), param.numel(), float(lr_t), float(beta1),
                           float(beta2), float(eps), _stream()), "rn_adam_step")
