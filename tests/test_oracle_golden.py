"""CPU tests: the oracle (oracle/rendernet_oracle.py) against the fixtures frozen from the
reference's own Python source (tests/golden/make_golden.py), plus independent
brute-force float64 known-answer checks of the TF-1 op semantics (SURVEY Appendix A).
"""
import itertools
import os

import numpy as np
import pytest
import torch

from oracle import rendernet_oracle as orc


def _g(golden_dir, name):
    return np.load(os.path.join(golden_dir, name))


def _chair(golden_dir):
    bv = _g(golden_dir, "binvox.npz")
    return np.unpackbits(bv["chair_bits"]).reshape(64, 64, 64).astype(np.float32).reshape(1, 64, 64, 64, 1)


# ----------------------------------------------------------------------------- binvox / pose
def test_binvox_counts_match_survey(golden_dir):
    bv = _g(golden_dir, "binvox.npz")
    want = dict(bunny=57835, chair=5277, suzanne=30270, table=61087, teapot=27933)   # SURVEY §4
    for k, v in want.items():
        assert int(bv[k + "_count"]) == v
        assert int(np.unpackbits(bv[k + "_bits"]).sum()) == v


def test_binvox_reader_roundtrip(golden_dir, tmp_path):
    """Encode a known grid as `#binvox 1` RLE (in file order x,z,y) and decode it."""
    rng = np.random.default_rng(0)
    grid = rng.random((8, 8, 8)) < 0.4
    flat = np.transpose(grid, (0, 2, 1)).reshape(-1).astype(np.uint8)
    rle = bytearray()
    i = 0
    while i < flat.size:
        j = i
        while j < flat.size and flat[j] == flat[i] and j - i < 255:
            j += 1
        rle += bytes([int(flat[i]), j - i])
        i = j
    p = tmp_path / "t.binvox"
    p.write_bytes(b"#binvox 1\ndim 8 8 8\ntranslate 0 0 0\nscale 1\ndata\n" + bytes(rle))
    with open(p, "rb") as f:
        got = orc.read_binvox(f)
    assert got.dtype == bool and np.array_equal(got, grid)
    with pytest.raises(IOError):
        import io
        orc.read_binvox(io.BytesIO(b"not a binvox\n"))


def test_pose_and_light(golden_dir):
    g = _g(golden_dir, "pose.npz")
    assert np.array_equal(orc.compute_pose_param(250.0, 60.0, 3.3), g["pose_250_60_33"])
    assert np.array_equal(orc.compute_pose_param(0.0, 90.0, 2.5), g["pose_0_90_25"])
    assert np.array_equal(orc.compute_pose_param(355.0, 10.0, 4.5), g["pose_355_10_45"])
    assert np.array_equal(orc.generate_light_pos(60.0, 250.0), g["light_60_250"])


# ----------------------------------------------------------------------------- resampler
def test_resampler_chair_bit_exact(golden_dir):
    g = _g(golden_dir, "resample.npz")
    R, S = orc.rotation_around_grid_centroid(g["chair_pose"])
    assert np.array_equal(R, g["chair_R"]) and np.array_equal(S, g["chair_S"])
    t = orc.resampling(_chair(golden_dir), R, S)
    assert t.shape == (1, 128, 128, 128, 1)
    assert abs(t.sum(dtype=np.float64) - float(g["chair_sum"])) < 1e-9
    assert int((t > 1e-6).sum()) == int(g["chair_count_gt"]) == 8820               # SURVEY §8c
    n = np.ascontiguousarray(orc.transform_voxel_to_match_image(t)).reshape(-1)
    ref = np.zeros(n.size, np.float32)
    ref[g["chair_nz_idx"]] = g["chair_nz_val"]
    assert np.array_equal(n, ref)
    Minv = orc.inverse_total_matrix(R, S, 64, 128)[0]
    want = np.array([[-0.81379765, 0.46984631, 0.34202021, 32.123592],
                     [0.5, 0.86602539, 0.0, -55.425625],
                     [-0.29619819, 0.17101011, -0.93969256, 100.15237]])              # SURVEY §8c
    assert np.abs(Minv - want).max() < 2e-5


def test_resampler_small_multichannel_and_axis_aligned(golden_dir):
    g = _g(golden_dir, "resample.npz")
    o = orc.rotation_resampling(g["small_vox"], g["small_pose"], 16, 32)
    assert np.array_equal(o, g["small_out"])
    assert np.array_equal(np.ascontiguousarray(orc.transform_voxel_to_match_image(o)), g["small_net_in"])
    o = orc.rotation_resampling(g["axis_vox"], g["axis_pose"], 16, 32)
    assert np.array_equal(o, g["axis_out"])


def test_resampler_against_float64_bruteforce():
    """Independent float64 loop: closed-form inverse map p_src = RotY^T RotZ^T (p-c')/s + c,
    plain trilinear inside [0, size-1), zero outside (Appendix A.1)."""
    rng = np.random.default_rng(3)
    size, new = 8, 16
    vox = rng.random((1, size, size, size, 1))
    az, el, s = 1.1, 0.7, 1.2
    out = orc.rotation_resampling(vox.astype(np.float32), np.array([[az, el, s]], np.float32), size, new)[0, ..., 0]
    a = az - np.pi / 2
    RY = np.array([[np.cos(a), 0, -np.sin(a)], [0, 1, 0], [np.sin(a), 0, np.cos(a)]])
    RZ = np.array([[np.cos(el), np.sin(el), 0], [-np.sin(el), np.cos(el), 0], [0, 0, 1]])
    Rinv = (RZ @ RY).T
    worst = 0.0
    for i, j, k in itertools.product(range(new), repeat=3):
        p = Rinv @ (np.array([k, j, i], float) - new / 2) / s + size / 2
        x, y, z = p
        if min(p) < 0 or max(p) >= size - 1:
            if min(np.abs(p)) < 1e-4 or min(np.abs(p - (size - 1))) < 1e-4:
                continue  # knife edge
            want = 0.0
        else:
            x0, y0, z0 = int(np.floor(x)), int(np.floor(y)), int(np.floor(z))
            fx, fy, fz = x - x0, y - y0, z - z0
            want = 0.0
            for dz, dy, dx in itertools.product((0, 1), repeat=3):
                wgt = (fx if dx else 1 - fx) * (fy if dy else 1 - fy) * (fz if dz else 1 - fz)
                want += wgt * vox[0, z0 + dz, y0 + dy, x0 + dx, 0]
        worst = max(worst, abs(want - out[i, j, k]))
    assert worst < 2e-4, worst


def test_device_cell_resampler_matches_golden(golden_dir):
    """oracle/resample_cells.py, the float64 resampler the backward tests differentiate: its emulated fp32 sample coordinates
    equal np.matmul's bit for bit, and its output matches the fixtures everywhere, the knife-edge points of the axis-aligned
    poses included (inside/outside decided by one ulp).  Inside the cube only fp32-vs-float64 weight rounding separates them;
    outside, the fixtures hold the reference's clamped-corner cancellation noise where the resampler writes 0 (DESIGN §4)."""
    from oracle import resample_cells as rc
    g = _g(golden_dir, "resample.npz")
    cases = [("small_vox", "small_pose", "small_out", 16, 32, False), ("small_vox", "small_pose", "small_net_in", 16, 32, True),
             ("axis_vox", "axis_pose", "axis_out", 16, 32, False), (None, "chair_pose", None, 64, 128, True)]
    for vk, pk, ok, S, N, transform in cases:
        vox = _chair(golden_dir) if vk is None else g[vk]
        if ok is None:
            want = np.zeros(N ** 3, np.float32)
            want[g["chair_nz_idx"]] = g["chair_nz_val"]
        else:
            want = g[ok]
        want = want.reshape(vox.shape[0], N, N, N, vox.shape[-1])
        R, Sm = orc.rotation_around_grid_centroid(g[pk])
        minv = orc.inverse_total_matrix(R, Sm, S, N)
        grid = rc.output_grid(N, transform)
        c = rc.sample_coords(minv, grid)
        assert np.array_equal(c, np.matmul(minv, grid.astype(np.float32)[None]))
        inside = ((c >= 0) & (c < S - 1)).all(1).reshape(vox.shape[0], N, N, N)
        got = rc.resample(torch.from_numpy(vox.astype(np.float64)), torch.from_numpy(minv.astype(np.float64)), N, transform).numpy()
        err = np.abs(got - want).max(-1)
        assert err[inside].max() < 1e-6 and err[~inside].max() < 5e-5, (ok, err[inside].max(), err[~inside].max())
        if vk == "axis_vox":
            edge = (np.minimum(np.abs(c), np.abs(c - (S - 1))).min(1) < 1e-4).reshape(inside.shape)
            assert (edge & inside).sum() > 500 and (edge & ~inside).sum() > 500       # both sides of the border are pinned
            f64 = rc.resample(torch.from_numpy(vox.astype(np.float64)), torch.from_numpy(minv.astype(np.float64)), N, transform,
                              device_cells=False).numpy()
            assert np.abs(f64 - want).max() > 0.5              # float64 coordinates decide some knife edges the other way


def test_device_cell_coordinates_round_once():
    """The fp32 emulation of oracle/resample_cells.py rounds each fused multiply-add once, as fmaf does, also where going
    through float64 would round twice: 2^30 + (64 + 2^-24) lies just above the fp32 halfway point 2^30 + 64."""
    from fractions import Fraction
    from oracle import resample_cells as rc

    def round32(v):                                        # nearest fp32 to the exact value v, ties to the even significand
        r = np.float32(float(v))
        near = [np.nextafter(r, np.float32(-np.inf)), r, np.nextafter(r, np.float32(np.inf))]
        return min(near, key=lambda f: (abs(Fraction(float(f)) - v), int(np.array(f).view(np.uint32)) & 1))

    a, c = np.float32(16519105 * 2.0 ** -24), np.float32(2.0 ** 30)          # a * 65 = 64 + 2^-24 exactly
    for s in (1, -1):
        got = rc._fma32(np.array([s * a]), 65.0, np.array([s * c]))[0]
        assert got == round32(Fraction(float(s * a)) * 65 + Fraction(float(s * c))) == np.float32(s * (2.0 ** 30 + 128))
    rng = np.random.default_rng(0)
    a = (rng.uniform(-1, 1, 3000) * np.exp2(rng.integers(-40, 6, 3000))).astype(np.float32)
    c = (rng.uniform(-1, 1, 3000) * np.exp2(rng.integers(-5, 11, 3000))).astype(np.float32)
    b = rng.integers(0, 128, 3000).astype(np.float64)
    got = rc._fma32(a, b, c)
    want = np.array([round32(Fraction(float(x)) * int(y) + Fraction(float(z))) for x, y, z in zip(a, b, c)], np.float32)
    assert np.array_equal(got, want)


def test_axis_transform_definition():
    t = np.arange(2 * 3 * 4 * 5 * 1, dtype=np.float32).reshape(2, 3, 4, 5, 1)
    n = orc.transform_voxel_to_match_image(t)
    for p, q, r in itertools.product(range(4), range(3), range(5)):
        assert n[1, p, q, r, 0] == t[1, q, 4 - 1 - p, r, 0]                        # N[b,p,q,r]=T[b,q,P-1-p,r]


# ----------------------------------------------------------------------------- conv semantics
def _brute_conv(x, w, stride, transpose=False):
    """float64 loops from the definitions in SURVEY Appendix A.2."""
    nd = x.ndim - 2
    ins = x.shape[1:1 + nd]
    ks = w.shape[:nd]
    if not transpose:
        outs, pb = [], []
        for d in range(nd):
            o = -(-ins[d] // stride[d]); tot = max((o - 1) * stride[d] + ks[d] - ins[d], 0)
            outs.append(o); pb.append(tot // 2)
        y = np.zeros((x.shape[0], *outs, w.shape[-1]))
        for o in itertools.product(*[range(n) for n in outs]):
            for t in itertools.product(*[range(k) for k in ks]):
                src = [o[d] * stride[d] + t[d] - pb[d] for d in range(nd)]
                if all(0 <= src[d] < ins[d] for d in range(nd)):
                    y[(slice(None),) + o] += x[(slice(None),) + tuple(src)] @ w[t]
        return y
    outs = [ins[d] * stride[d] for d in range(nd)]
    pb = [max(ks[d] - stride[d], 0) // 2 for d in range(nd)]
    y = np.zeros((x.shape[0], *outs, w.shape[-2]))
    for i in itertools.product(*[range(n) for n in ins]):
        for t in itertools.product(*[range(k) for k in ks]):
            o = [i[d] * stride[d] + t[d] - pb[d] for d in range(nd)]
            if all(0 <= o[d] < outs[d] for d in range(nd)):
                y[(slice(None),) + tuple(o)] += x[(slice(None),) + i] @ w[t].T
    return y


@pytest.mark.parametrize("k,s,n", [(5, 2, 8), (3, 1, 5), (3, 2, 6), (4, 1, 5)])
def test_conv3d_same_semantics(k, s, n):
    rng = np.random.default_rng(k * 10 + s)
    x = rng.standard_normal((1, n, n, n, 2)); w = rng.standard_normal((k, k, k, 2, 3))
    got = orc.conv3d(x.astype(np.float32), w.astype(np.float32), None, (s, s, s)).numpy()
    assert np.abs(got - _brute_conv(x, w, (s, s, s))).max() < 1e-4


def test_conv3d_mixed_stride():
    rng = np.random.default_rng(5)
    x = rng.standard_normal((1, 4, 4, 8, 2)); w = rng.standard_normal((3, 3, 3, 2, 3))
    got = orc.conv3d(x.astype(np.float32), w.astype(np.float32), None, (1, 1, 2)).numpy()
    assert got.shape == (1, 4, 4, 4, 3)
    assert np.abs(got - _brute_conv(x, w, (1, 1, 2))).max() < 1e-4


@pytest.mark.parametrize("k", [1, 3, 4])
def test_conv2d_same_semantics(k):
    rng = np.random.default_rng(k)
    x = rng.standard_normal((2, 6, 7, 3)); w = rng.standard_normal((k, k, 3, 4)); b = rng.standard_normal(4)
    got = orc.conv2d(x.astype(np.float32), w.astype(np.float32), b.astype(np.float32)).numpy()
    assert np.abs(got - (_brute_conv(x, w, (1, 1)) + b)).max() < 1e-4


@pytest.mark.parametrize("s", [1, 2])
def test_conv2d_transpose_same_semantics(s):
    rng = np.random.default_rng(s)
    x = rng.standard_normal((1, 5, 6, 3)); w = rng.standard_normal((4, 4, 2, 3))
    got = orc.conv2d_transpose(x.astype(np.float32), w.astype(np.float32), None, (s, s)).numpy()
    assert got.shape == (1, 5 * s, 6 * s, 2)
    assert np.abs(got - _brute_conv(x, w, (s, s), transpose=True)).max() < 1e-4


@pytest.mark.parametrize("s", [1, 2])
def test_conv3d_transpose_same_semantics(s):
    rng = np.random.default_rng(s + 7)
    x = rng.standard_normal((1, 3, 4, 3, 2)); w = rng.standard_normal((4, 4, 4, 3, 2))
    got = orc.conv3d_transpose(x.astype(np.float32), w.astype(np.float32), None, (s, s, s)).numpy()
    assert np.abs(got - _brute_conv(x, w, (s, s, s), transpose=True)).max() < 1e-4


def test_transposed_conv_of_delta_reproduces_kernel():
    w = np.arange(4 * 4, dtype=np.float32).reshape(4, 4, 1, 1)
    x = np.zeros((1, 6, 6, 1), np.float32); x[0, 3, 3, 0] = 1
    y = orc.conv2d_transpose(x, w, None, (2, 2)).numpy()[0, :, :, 0]
    assert np.array_equal(y[5:9, 5:9], w[:, :, 0, 0])                             # o = 2*i + k - 1


def test_prelu_and_projection_reshape_order():
    x = np.array([[-2.0, 3.0, -0.5]], np.float32)
    assert np.allclose(orc.prelu(x, np.array([0.5, 0.5, 0.1], np.float32)).numpy(), [[-1.0, 3.0, -0.05]])
    B, H, W, D, C = 1, 2, 2, 3, 2
    x = np.arange(B * H * W * D * C, dtype=np.float32).reshape(B, H, W, D, C)
    eye = np.eye(D * C, dtype=np.float32).reshape(1, 1, D * C, D * C)
    y = orc.projection_unit(x, eye, np.zeros(D * C, np.float32), np.ones(D * C, np.float32)).numpy()
    for d in range(D):
        for c in range(C):
            assert y[0, 1, 0, d * C + c] == x[0, 1, 0, d, c]                       # f = d*C + c


# ----------------------------------------------------------------------------- Shader net wiring
def test_shader_variable_names_and_bias_inits(golden_dir):
    g = _g(golden_dir, "shader_patch.npz")
    specs = orc.shader_layer_specs()
    mine = {}
    for name, kind, shape, b0, alpha_scope in specs:
        mine[name + "/weights"] = shape
        nb = shape[-2] if kind == "conv2d_transpose" else shape[-1]
        mine[name + "/biases"] = (nb,)
        if alpha_scope:
            mine[alpha_scope + "/alpha"] = (nb,)
    ref = {n: tuple(int(v) for v in s.split(";")) for n, s in zip(g["var_names"].tolist(), g["var_shapes"].tolist())}
    assert mine == ref
    nparams = sum(int(np.prod(s)) for s in ref.values() if len(s) > 1)
    assert abs(nparams - 237.2e6) < 0.1e6                                        # SURVEY: 237.2 M weights
    bias0 = dict(zip(g["bias_init_names"].tolist(), g["bias_init_vals"].tolist()))
    for name, kind, shape, b0, _ in specs:
        assert abs(bias0[name + "/biases"] - b0) < 1e-9, name


def test_shader_patch_matches_reference_python(golden_dir):
    """Reference RenderNet() (RenderNet_Shader.py:32-131) executed over the TF shim vs the oracle."""
    g = _g(golden_dir, "shader_patch.npz"); r = _g(golden_dir, "resample.npz")
    n = np.ascontiguousarray(orc.transform_voxel_to_match_image(
        orc.rotation_resampling(_chair(golden_dir), r["chair_pose"])))
    a, b, c, d = g["patch_slice"]
    W = orc.init_shader_weights(seed=int(g["weight_seed"]), alpha_range=tuple(g["alpha_range"]),
                                gain=float(g["gain"]), bias_jitter=float(g["bias_jitter"]))
    img = orc.rendernet_shader(np.ascontiguousarray(n[:, a:b, c:d]), W).numpy()
    assert img.shape == g["image"].shape == (1, 64, 64, 3)
    assert np.abs(img - g["image"]).max() < 5e-6


# ----------------------------------------------------------------------------- Phong
def test_phong_composite_matches_reference(golden_dir):
    g = _g(golden_dir, "phong.npz")
    lc = np.array([[1.0, 1.0, 1.0]] * 2)
    with np.errstate(over="ignore"):
        comp = orc.np_phong_composite(g["normal_map"], g["light"], lc, 0.1, 0.9)
        comp_w = orc.np_phong_composite(g["normal_map"], g["light"], lc, 0.1, 0.9, background_col="White")
    assert np.abs(comp - g["composite"]).max() < 1e-12
    assert np.abs(comp_w - g["composite_white"]).max() < 1e-12
    assert np.array_equal(orc.to_uint8(comp[0]), g["uint8_first"])


# ----------------------------------------------------------------------------- Texture + Normal net (config 4)
def test_texture_model_matches_reference_python(golden_dir):
    """decoder_texture + RenderNet of RenderNet_Texture_Face_Normal.py:34-147 executed over the TF shim vs the oracle,
    incl. the variable names the reference creates (scope quirks of :118-127)."""
    g = _g(golden_dir, "texture_patch.npz"); r = _g(golden_dir, "resample.npz")
    W = orc.init_texture_weights(seed=int(g["weight_seed"]), alpha_range=tuple(g["alpha_range"]),
                                 gain=float(g["gain"]), bias_jitter=float(g["bias_jitter"]))
    assert sorted(W) == g["var_names"].tolist()
    shapes = {n: tuple(int(v) for v in s.split(";")) for n, s in zip(g["var_names"].tolist(), g["var_shapes"].tolist())}
    assert all(tuple(W[k].shape) == shapes[k] for k in W)
    tex = orc.decoder_texture(g["z_in"], W).numpy()
    assert np.abs(tex[:, ::4, ::4, ::4] - g["decoder_sub"]).max() < 1e-6
    assert abs(tex.sum(dtype=np.float64) - float(g["decoder_sum"])) < 1e-2 * max(1.0, float(g["decoder_abs_sum"]) * 1e-3)
    pose = r["chair_pose"]
    n = orc.transform_voxel_to_match_image(orc.rotation_resampling(_chair(golden_dir), pose))
    tr = orc.transform_voxel_to_match_image(orc.rotation_resampling(tex, pose))
    a, b, c, d = g["patch_slice"]
    x5 = np.ascontiguousarray(np.concatenate([n, tr], axis=4)[:, a:b, c:d])
    img, nrm = orc.rendernet_texture(x5, W)
    assert np.abs(img.numpy() - g["image"]).max() < 5e-6
    assert np.abs(nrm.numpy() - g["normal"]).max() < 5e-6


def test_texture_decoder_float64_matches_float32_and_reference_python(golden_dir):
    """decoder_texture(dtype=torch.float64) -- the reference tests/test_gpu_texture.py holds the CUDA decoder to -- runs the same
    SAME-padding and transposed-conv code as the fp32 oracle pinned above, in float64.  Measured (max error / max |float64|):
    vs the fp32 oracle 1.3e-6, vs the fixture's every-4th-voxel sample 1.5e-7 (the fixture is fp32); the sum over all voxels is
    2.4e-10 of the fixture's sum of |values|."""
    g = _g(golden_dir, "texture_patch.npz")
    W = orc.init_texture_weights(seed=int(g["weight_seed"]), alpha_range=tuple(g["alpha_range"]),
                                 gain=float(g["gain"]), bias_jitter=float(g["bias_jitter"]))
    t32 = orc.decoder_texture(g["z_in"], W)
    t64 = orc.decoder_texture(g["z_in"], W, dtype=torch.float64)
    assert t32.dtype == torch.float32 and t64.dtype == torch.float64 and t64.shape == t32.shape == (1, 64, 64, 64, 4)
    t64 = t64.numpy()
    scale = np.abs(t64).max()
    assert np.abs(t64 - t32.numpy()).max() < 4e-6 * scale
    assert np.abs(t64[:, ::4, ::4, ::4] - g["decoder_sub"]).max() < 5e-7 * scale
    assert abs(t64.sum() - float(g["decoder_sum"])) < 1e-9 * float(g["decoder_abs_sum"])
