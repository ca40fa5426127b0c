#!/usr/bin/env python
"""Generate tests/golden/*.npz by executing the REFERENCE'S OWN PYTHON SOURCE.

Needs a checkout of the reference (thunguyenphuoc/RenderNet); the tests only read the
stored fixtures:   python tests/golden/make_golden.py /path/to/RenderNet

How: TensorFlow-1 is not installable here, so `oracle/tf1_shim.py` registers a NumPy
stand-in for the ~50 TF primitives the hot path uses; the reference modules
(`tools/resampling_voxel_grid.py`, `tools/model_util.py`, `tools/layer_util.py`,
`tools/Phong_shading.py`, `tools/binvox_rw.py`, `RenderNet_demo.py`) are then imported
unmodified from that checkout, and the `RenderNet` model function is lifted out of
`RenderNet_Shader.py` with `ast` (that module trains at import time, so it cannot be
imported) and executed over the shim.  No reference source is copied into this repo.

The fixtures pin: the binvox decoder, the pose convention, the resampler (matrix,
8-tap blend, clamp rule, axis transform), the layer/scope/weight-name wiring and
data flow of the Shader network, and the NumPy Phong composite.
"""
import ast
import io
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = sys.argv[1] if __name__ == "__main__" and len(sys.argv) > 1 else os.environ.get("RENDERNET_REFERENCE", "")
sys.path.insert(0, ROOT)

from oracle import tf1_shim  # noqa: E402
from oracle import rendernet_oracle as orc  # noqa: E402  (only for seeded weight/input generation)


def _install_env():
    tf = tf1_shim.install()
    # NumPy>=1.24 removed the aliases tools/binvox_rw.py uses (np.bool :85, np.int :146)
    if not hasattr(np, "bool"):
        np.bool = bool
    if not hasattr(np, "int"):
        np.int = int
    try:
        from scipy import misc  # noqa: F401
    except Exception:
        import scipy
        m = types.ModuleType("scipy.misc")
        m.imsave = lambda *a, **k: None
        sys.modules["scipy.misc"] = m
        scipy.misc = m
    sys.path.insert(0, REF)
    return tf


def _lift_function(path, name, namespace):
    src = open(path).read()
    tree = ast.parse(src)
    for node in tree.body:
        if isinstance(node, ast.FunctionDef) and node.name == name:
            code = compile(ast.Module(body=[node], type_ignores=[]), path, "exec")
            exec(code, namespace)
            return namespace[name]
    raise KeyError(name)


def main():
    tf = _install_env()
    from tools import binvox_rw, Phong_shading, model_util, layer_util  # reference modules
    from tools import resampling_voxel_grid as rvg
    import RenderNet_demo as demo

    out = {}

    # ------------------------------------------------------------------ binvox
    bv = {}
    for nm in ("bunny", "chair", "suzanne", "table", "teapot"):
        with open(os.path.join(REF, "binvox", nm + ".binvox"), "rb") as f:
            data = binvox_rw.read_as_3d_array(f).data
        bv[nm + "_count"] = np.int64(data.sum())
        bv[nm + "_bits"] = np.packbits(data.reshape(-1))
    np.savez_compressed(os.path.join(HERE, "binvox.npz"), **bv)

    # ------------------------------------------------------------------ pose + light
    pose = demo.compute_pose_param(250.0, 60.0, 3.3)
    light = Phong_shading.generate_light_pos(60.0, 250.0)
    np.savez(os.path.join(HERE, "pose.npz"), pose_250_60_33=pose, light_60_250=light,
             pose_0_90_25=demo.compute_pose_param(0.0, 90.0, 2.5),
             pose_355_10_45=demo.compute_pose_param(355.0, 10.0, 4.5))

    # ------------------------------------------------------------------ resampler
    def ref_resample(vox, vp, size, new_size):
        vp = tf.constant(np.asarray(vp, np.float32))
        vox = tf.constant(np.asarray(vox, np.float32))
        M, S = rvg.tf_rotation_around_grid_centroid(vp)
        # tf_rotation_resampling (:616) is broken as shipped (missing positional `params`, :627-630);
        # call tf_resampling with the vestigial argument filled in.
        t = rvg.tf_resampling(vox, M, None, Scale_matrix=S, size=size, new_size=new_size)
        n = model_util.tf_transform_voxel_to_match_image(t)
        return np.asarray(M), np.asarray(S), np.asarray(t), np.asarray(n)

    with open(os.path.join(REF, "binvox", "chair.binvox"), "rb") as f:
        chair = binvox_rw.read_as_3d_array(f).data.astype(np.float32).reshape(1, 64, 64, 64, 1)
    M, S, t, n = ref_resample(chair, pose, 64, 128)
    nz = np.flatnonzero(n.reshape(-1))
    rs = dict(chair_pose=pose, chair_R=M, chair_S=S, chair_sum=np.float64(t.sum(dtype=np.float64)),
              chair_nz_idx=nz.astype(np.int32), chair_nz_val=n.reshape(-1)[nz].astype(np.float32),
              chair_count_gt=np.int64((t > 1e-6).sum()))
    rng = np.random.default_rng(7)
    vox_s = rng.random((3, 16, 16, 16, 2), dtype=np.float32)
    vp_s = np.stack([rng.uniform(0, 2 * np.pi, 3), (90 - rng.uniform(10, 170, 3)) * np.pi / 180,
                     3.3 / rng.uniform(2.5, 4.5, 3)], axis=1).astype(np.float32)
    _, _, t_s, n_s = ref_resample(vox_s, vp_s, 16, 32)
    rs.update(small_vox=vox_s, small_pose=vp_s, small_out=t_s.astype(np.float32), small_net_in=n_s.astype(np.float32))
    # axis-aligned knife-edge poses (az in {0,90,180,270} deg), binary voxels
    vox_b = (rng.random((4, 16, 16, 16, 1)) < 0.3).astype(np.float32)
    vp_b = np.stack([np.deg2rad([0.0, 90.0, 180.0, 270.0]), np.deg2rad([90 - 60.0] * 4), [1.0] * 4], axis=1).astype(np.float32)
    _, _, t_b, _ = ref_resample(vox_b, vp_b, 16, 32)
    rs.update(axis_vox=vox_b, axis_pose=vp_b, axis_out=t_b.astype(np.float32))
    np.savez_compressed(os.path.join(HERE, "resample.npz"), **rs)

    # ------------------------------------------------------------------ Shader model fn on a patch
    ns = dict(tf=tf, slim=sys.modules["tensorflow.contrib.slim"], cfg={"is_greyscale": "false"},
              keep_prob=layer_util.keep_prob, conv3d=layer_util.conv3d, prelu=layer_util.prelu,
              res_block_2d=layer_util.res_block_2d, res_block_3d=layer_util.res_block_3d,
              projection_unit=layer_util.projection_unit)
    RenderNet = _lift_function(os.path.join(REF, "RenderNet_Shader.py"), "RenderNet", ns)
    W = orc.init_shader_weights(seed=1234, alpha_range=(0.05, 0.3), gain=0.9, bias_jitter=0.02)
    patch = np.ascontiguousarray(n[:, 56:72, 56:72, :, :])           # [1,16,16,128,1] centre crop
    devnull = io.StringIO()
    stdout, sys.stdout = sys.stdout, devnull                         # layer_util prints per layer
    try:
        tf1_shim.reset(provided=W)
        img = np.asarray(RenderNet(tf.constant(patch), tf.constant(False), prob=0.75))
        used = tf1_shim.created_variables()
        tf1_shim.reset(provided=None, seed=3)
        RenderNet(tf.constant(patch[:, :4, :4]), tf.constant(False))
        fresh = tf1_shim.created_variables()
    finally:
        sys.stdout = stdout
    assert set(used) == set(W), (sorted(set(used) ^ set(W))[:10])
    names = np.array(sorted(fresh.keys()))
    shapes = np.array([";".join(map(str, fresh[k].shape)) for k in names])
    biases0 = {k: float(fresh[k].reshape(-1)[0]) for k in names if k.endswith("biases")}
    np.savez_compressed(os.path.join(HERE, "shader_patch.npz"), patch_slice=np.array([56, 72, 56, 72]),
                        weight_seed=np.int64(1234), alpha_range=np.array([0.05, 0.3]), gain=np.float64(0.9),
                        bias_jitter=np.float64(0.02), image=img.astype(np.float32),
                        var_names=names, var_shapes=shapes,
                        bias_init_names=np.array(sorted(biases0)), bias_init_vals=np.array([biases0[k] for k in sorted(biases0)]))

    # ------------------------------------------------------------------ Texture + Normal net and texture decoder
    tex_path = os.path.join(REF, "RenderNet_Texture_Face_Normal.py")
    nst = dict(tf=tf, slim=sys.modules["tensorflow.contrib.slim"], is_training=tf.constant(False),
               keep_prob=layer_util.keep_prob, conv3d=layer_util.conv3d, conv2d=layer_util.conv2d,
               conv2d_transpose=layer_util.conv2d_transpose, conv3d_transpose=layer_util.conv3d_transpose,
               fully_connected=layer_util.fully_connected, prelu=layer_util.prelu,
               res_block_2d=layer_util.res_block_2d, res_block_3d=layer_util.res_block_3d,
               projection_unit=layer_util.projection_unit)
    decoder_texture = _lift_function(tex_path, "decoder_texture", nst)
    RenderNetTex = _lift_function(tex_path, "RenderNet", nst)
    Wt = orc.init_texture_weights(seed=4321, alpha_range=(0.05, 0.3), gain=1.0, bias_jitter=0.02)
    z_in = np.random.default_rng(2).standard_normal((1, 199)).astype(np.float32)
    stdout, sys.stdout = sys.stdout, devnull
    try:
        tf1_shim.reset(provided=Wt)
        tex_dec = np.asarray(decoder_texture(tf.constant(z_in)))                       # [1,64,64,64,4]
        # graph wiring of :155-179 on the chair grid: resample both, concat on the channel axis, crop a patch
        _, _, _, tex_rot = ref_resample(tex_dec, pose, 64, 128)
        x5 = np.concatenate([n, tex_rot], axis=4)
        patch5 = np.ascontiguousarray(x5[:, 56:72, 56:72])
        img_t, nrm_t = RenderNetTex(tf.constant(patch5), prob=0.75)
        used_t = tf1_shim.created_variables()
    finally:
        sys.stdout = stdout
    assert set(used_t) == set(Wt), sorted(set(used_t) ^ set(Wt))[:10]
    np.savez_compressed(os.path.join(HERE, "texture_patch.npz"), weight_seed=np.int64(4321), alpha_range=np.array([0.05, 0.3]),
                        gain=np.float64(1.0), bias_jitter=np.float64(0.02), z_in=z_in,
                        decoder_sub=tex_dec[:, ::4, ::4, ::4].astype(np.float32),
                        decoder_sum=np.float64(tex_dec.sum(dtype=np.float64)),
                        decoder_abs_sum=np.float64(np.abs(tex_dec).sum(dtype=np.float64)),
                        patch_slice=np.array([56, 72, 56, 72]),
                        image=np.asarray(img_t, np.float32), normal=np.asarray(nrm_t, np.float32),
                        var_names=np.array(sorted(used_t.keys())),
                        var_shapes=np.array([";".join(map(str, used_t[k].shape)) for k in sorted(used_t.keys())]))

    # ------------------------------------------------------------------ Phong composite
    rng = np.random.default_rng(11)
    nm = rng.random((2, 16, 16, 3)).astype(np.float32)
    nm[:, :4] *= 0.05                                                # dark background rows -> mask ~ 0
    l2 = np.repeat(Phong_shading.generate_light_pos(60.0, 250.0), 2, 0)
    comp = Phong_shading.np_phong_composite(nm.copy(), l2.copy(), np.array([[1., 1., 1.]] * 2), 0.1, 0.9)
    comp_w = Phong_shading.np_phong_composite(nm.copy(), l2.copy(), np.array([[1., 1., 1.]] * 2), 0.1, 0.9,
                                              background_col="White")
    u8 = np.clip(255. * comp[0], 0, 255).astype(np.uint8)           # RenderNet_demo.py:58
    np.savez_compressed(os.path.join(HERE, "phong.npz"), normal_map=nm, light=l2, composite=comp,
                        composite_white=comp_w, uint8_first=u8)
    print("golden fixtures written to", HERE)
    for f in sorted(os.listdir(HERE)):
        if f.endswith(".npz"):
            print(f"  {f}: {os.path.getsize(os.path.join(HERE, f)) / 1024:.1f} KiB")


if __name__ == "__main__":
    main()
