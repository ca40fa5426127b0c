"""GPU parity tests: every CUDA kernel, called through the C ABI (ctypes), against the CPU oracle on the same
seeded inputs.  Tolerances (floating point, stated per test):
  * resampler / Phong (fp32 kernels): absolute 2e-4 / 1e-4;
  * tensor-core convs: operands are rounded to fp16 for BOTH sides, so the fp32-output error is pure
    accumulation-order noise (<= 1e-5 relative) and the fp16-output error is one fp16 rounding (<= 2^-10 relative).
"""
import os

import numpy as np
import pytest
import torch

from oracle import rendernet_oracle as orc

pytestmark = pytest.mark.gpu
dev = "cuda"


def _ops():
    from rendernet_b200 import ops
    return ops


def q16(a):
    return torch.from_numpy(np.asarray(a, np.float32)).half().float().numpy()


def close(got, want, rel=None, abs_=None):
    got = got.float().cpu().numpy() if isinstance(got, torch.Tensor) else np.asarray(got)
    want = want.float().cpu().numpy() if isinstance(want, torch.Tensor) else np.asarray(want)
    assert got.shape == want.shape, (got.shape, want.shape)
    err = float(np.abs(got - want).max())
    bound = abs_ if abs_ is not None else rel * max(float(np.abs(want).max()), 1e-6)
    assert err <= bound, f"max abs err {err:.3e} > {bound:.3e}"
    return err


# ----------------------------------------------------------------------------------------- resampler
def test_resample_golden_small_and_chair(golden_dir):
    ops = _ops()
    g = np.load(os.path.join(golden_dir, "resample.npz"))
    R, S = orc.rotation_around_grid_centroid(g["small_pose"])
    minv = torch.from_numpy(orc.inverse_total_matrix(R, S, 16, 32)).to(dev)
    vox = torch.from_numpy(g["small_vox"]).to(dev)
    close(ops.resample(vox, minv, 32, False), g["small_out"], abs_=2e-4)
    close(ops.resample(vox, minv, 32, True), g["small_net_in"], abs_=2e-4)
    bv = np.load(os.path.join(golden_dir, "binvox.npz"))
    chair = np.unpackbits(bv["chair_bits"]).reshape(1, 64, 64, 64, 1).astype(np.float32)
    R, S = orc.rotation_around_grid_centroid(g["chair_pose"])
    minv = torch.from_numpy(orc.inverse_total_matrix(R, S, 64, 128)).to(dev)
    out = ops.resample(torch.from_numpy(chair).to(dev), minv, 128, True)
    ref = np.zeros(128 ** 3, np.float32)
    ref[g["chair_nz_idx"]] = g["chair_nz_val"]
    close(out.reshape(-1), ref, abs_=2e-4)
    assert abs(float(out.double().sum()) - float(g["chair_sum"])) < 0.05


def test_resample_properties_full_size():
    """Size-independent properties at BASELINE's full size (B=24, 64^3 -> 128^3): linearity in the voxel values,
    range preservation, and identity pose reproducing the grid at the embedded offset."""
    ops = _ops()
    rng = np.random.default_rng(0)
    B = 24
    vox = torch.from_numpy((rng.random((B, 64, 64, 64, 1)) < 0.1).astype(np.float32)).to(dev)
    poses = np.stack([rng.uniform(0, 2 * np.pi, B), (90 - rng.uniform(10, 170, B)) * np.pi / 180,
                      3.3 / rng.uniform(2.5, 4.5, B)], axis=1).astype(np.float32)
    R, S = orc.rotation_around_grid_centroid(poses)
    minv = torch.from_numpy(orc.inverse_total_matrix(R, S, 64, 128)).to(dev)
    a = ops.resample(vox, minv, 128, True)
    assert float(a.min()) >= 0.0 and float(a.max()) <= 1.0 + 1e-6
    b = ops.resample(vox * 0.25, minv, 128, True)
    close(b, a * 0.25, abs_=1e-6)                                                     # linearity
    eye = torch.eye(4)[:3].repeat(B, 1, 1).contiguous()
    eye[:, :, 3] = -32.0                                                              # p_src = p_dst - 32
    t = ops.resample(vox, eye.to(dev), 128, False)
    assert torch.equal(t[:, 32:95, 32:95, 32:95], vox[:, :63, :63, :63])              # interior copied exactly
    assert float(t[:, :32].abs().max()) == 0.0 and float(t[:, 96:].abs().max()) == 0.0


def test_resample_axis_aligned_knife_edges(golden_dir):
    ops = _ops()
    g = np.load(os.path.join(golden_dir, "resample.npz"))
    R, S = orc.rotation_around_grid_centroid(g["axis_pose"])
    minv = orc.inverse_total_matrix(R, S, 16, 32)
    out = ops.resample(torch.from_numpy(g["axis_vox"]).to(dev), torch.from_numpy(minv).to(dev), 32, False).cpu().numpy()
    diff = np.abs(out - g["axis_out"])
    # points whose source coordinate is within 1e-4 of 0 or 15 sit on the clamp discontinuity (SURVEY A.1)
    grid = orc.voxel_meshgrid(32, 32, 32)
    pts = np.matmul(minv, grid[None])
    edge = (np.minimum(np.abs(pts), np.abs(pts - 15.0)).min(axis=1) < 1e-4).reshape(out.shape[:4])
    assert diff[~edge].max() < 2e-4
    assert edge.mean() < 0.2


# ----------------------------------------------------------------------------------------- Phong
def test_phong_matches_reference(golden_dir):
    ops = _ops()
    g = np.load(os.path.join(golden_dir, "phong.npz"))
    lc = torch.ones(2, 3)
    out, u8 = ops.phong_composite(torch.from_numpy(g["normal_map"]).to(dev), torch.from_numpy(g["light"]).float(), lc,
                                  0.1, 0.9, want_u8=True)
    close(out, g["composite"].astype(np.float32), abs_=1e-4)
    assert np.abs(u8[0].cpu().numpy().astype(int) - g["uint8_first"].astype(int)).max() <= 1
    out = ops.phong_composite(torch.from_numpy(g["normal_map"]).to(dev), torch.from_numpy(g["light"]).float(), lc,
                              0.1, 0.9, background_white=True)
    close(out, g["composite_white"].astype(np.float32), abs_=1e-4)


# ----------------------------------------------------------------------------------------- tensor-core convs
CONV2D = [  # B,H,W,Cin,Cout,k,act,res,res32
    (1, 16, 16, 64, 64, 1, None, False, False), (1, 16, 16, 128, 256, 1, None, False, False),
    (1, 16, 16, 16, 16, 1, None, False, False), (1, 16, 16, 32, 32, 1, None, False, False),
    (1, 16, 16, 256, 512, 1, "prelu", False, False), (1, 16, 16, 64, 3, 1, None, False, False),
    (1, 16, 16, 64, 24, 1, None, False, False),
    (2, 16, 16, 64, 64, 3, "prelu", False, False), (1, 16, 16, 128, 128, 3, None, True, False),
    (1, 16, 16, 128, 128, 3, None, True, True), (1, 64, 64, 64, 256, 3, "prelu", False, False),
    (1, 24, 20, 32, 64, 3, "prelu", False, False),      # ragged tiles (H, W not multiples of the M box)
    (1, 8, 8, 64, 64, 3, "sigmoid", False, False),      # M box taller than the image
    (1, 5, 7, 16, 16, 3, None, True, False),            # tiny, everything ragged
    (1, 8, 8, 1024, 1024, 3, "prelu", False, False),    # one M tile: no CTA pairing -> y-halo falls back (stage budget)
    (1, 128, 128, 32, 16, 3, "prelu", False, False), (1, 256, 256, 16, 16, 3, None, False, False),
    (1, 16, 16, 64, 128, 4, "prelu", False, False), (2, 32, 32, 128, 64, 4, None, False, False),
]


@pytest.mark.parametrize("B,H,W,Cin,Cout,k,act,with_res,res32", CONV2D)
def test_conv2d_same(B, H, W, Cin, Cout, k, act, with_res, res32):
    ops = _ops()
    rng = np.random.default_rng(Cin * 7 + Cout + k)
    x = q16(rng.standard_normal((B, H, W, Cin)))
    w = q16(rng.standard_normal((k, k, Cin, Cout)) / np.sqrt(k * k * Cin))
    b = (rng.standard_normal(Cout) * 0.1).astype(np.float32)
    a = rng.uniform(0, 0.3, Cout).astype(np.float32)
    res = q16(rng.standard_normal((B, H, W, Cout))) if with_res else None
    L = ops.pack_conv("conv2d", torch.from_numpy(w), torch.from_numpy(b), torch.from_numpy(a))
    rt = None
    if with_res:
        rt = torch.from_numpy(res).to(dev)
        rt = rt if res32 else rt.half()
    y16, y32 = ops.conv2d(torch.from_numpy(x).to(dev).half(), L, act=act, residual=rt, want16=True, want32=True)
    ref = orc.conv2d(x, w, b)
    if act == "prelu":
        ref = orc.prelu(ref, a)
    elif act == "sigmoid":
        ref = torch.sigmoid(ref)
    if with_res:
        ref = ref + torch.from_numpy(res)
    close(y32, ref, rel=2e-5)
    close(y16, ref, rel=1.2e-3)


@pytest.mark.parametrize("B,H,W,D,Cin,Cout", [(1, 8, 8, 32, 32, 32), (1, 8, 8, 32, 16, 32), (2, 4, 8, 16, 16, 16),
                                               (1, 6, 5, 32, 32, 32), (1, 16, 16, 4, 32, 32), (1, 3, 3, 3, 16, 16)])
@pytest.mark.parametrize("path", ["tma5d", "banded"])
def test_conv3d_same(B, H, W, D, Cin, Cout, path):
    ops = _ops()
    if path == "banded" and not ops.BandedConv3d.eligible(Cin, Cout, D):
        pytest.skip("shape not eligible for the depth-folded path")
    rng = np.random.default_rng(D + Cin + Cout)
    x = q16(rng.standard_normal((B, H, W, D, Cin)))
    w = q16(rng.standard_normal((3, 3, 3, Cin, Cout)) / np.sqrt(27 * Cin))
    b = (rng.standard_normal(Cout) * 0.1).astype(np.float32)
    a = rng.uniform(0, 0.3, Cout).astype(np.float32)
    res = q16(rng.standard_normal((B, H, W, D, Cout)))
    xt = torch.from_numpy(x).to(dev).half()
    rt = torch.from_numpy(res).to(dev).half()
    if path == "tma5d":
        L = ops.pack_conv("conv3d", torch.from_numpy(w), torch.from_numpy(b), torch.from_numpy(a))
        y1 = ops.conv3d(xt, L, act="prelu", want16=False, want32=True)
        y2 = ops.conv3d(xt, L, act=None, residual=rt)
    else:
        L = ops.BandedConv3d(torch.from_numpy(w), torch.from_numpy(b))
        y1 = ops.conv3d_banded(xt, L, act="prelu", alpha=torch.from_numpy(a).to(dev), want16=False, want32=True)
        y2 = ops.conv3d_banded(xt, L, act=None, residual=rt)
    close(y1, orc.prelu(orc.conv3d(x, w, b), a), rel=2e-5)
    close(y2, orc.conv3d(x, w, b) + torch.from_numpy(res), rel=1.2e-3)


@pytest.mark.parametrize("B,H,W,D,Cin,Cout", [(1, 8, 8, 64, 8, 16), (2, 4, 8, 32, 8, 16), (1, 8, 16, 16, 16, 16), (1, 5, 6, 64, 8, 16)])
def test_conv3d_banded_z_stride2(B, H, W, D, Cin, Cout):
    """e_conv2's form: 3^3 conv, stride (1,1,2), TF SAME pads (1,1)/(1,1)/(0,1), depth-folded onto the tensor pipe."""
    ops = _ops()
    assert ops.BandedConv3d.eligible(Cin, Cout, D, 2)
    rng = np.random.default_rng(D + Cin)
    x = q16(rng.standard_normal((B, H, W, D, Cin)))
    w = q16(rng.standard_normal((3, 3, 3, Cin, Cout)) / np.sqrt(27 * Cin))
    b = (rng.standard_normal(Cout) * 0.1).astype(np.float32)
    a = rng.uniform(0, 0.3, Cout).astype(np.float32)
    L = ops.BandedConv3d(torch.from_numpy(w), torch.from_numpy(b), sz=2)
    y = ops.conv3d_banded(torch.from_numpy(x).to(dev).half(), L, act="prelu", alpha=torch.from_numpy(a).to(dev),
                          want16=False, want32=True)
    ref = orc.prelu(orc.conv3d(x, w, b, (1, 1, 2)), a)
    assert tuple(y.shape) == tuple(ref.shape) == (B, H, W, D // 2, Cout)
    close(y, ref, rel=2e-5)


@pytest.mark.parametrize("B,H,W,Cin,Cout,s", [(1, 16, 16, 64, 32, 2), (1, 16, 16, 64, 64, 1), (2, 8, 8, 256, 128, 2),
                                               (1, 32, 32, 32, 16, 1), (1, 32, 32, 16, 3, 1), (1, 64, 64, 64, 32, 2),
                                               (1, 7, 9, 16, 16, 2)])
def test_conv2d_transpose_same(B, H, W, Cin, Cout, s):
    ops = _ops()
    rng = np.random.default_rng(Cin + Cout + s)
    x = q16(rng.standard_normal((B, H, W, Cin)))
    w = q16(rng.standard_normal((4, 4, Cout, Cin)) / np.sqrt(16 * Cin / (s * s)))
    b = (rng.standard_normal(Cout) * 0.1).astype(np.float32)
    a = rng.uniform(0, 0.3, Cout).astype(np.float32)
    L = ops.pack_conv("conv2d_transpose", torch.from_numpy(w), torch.from_numpy(b), torch.from_numpy(a), stride=s)
    y16, y32 = ops.conv2d_transpose(torch.from_numpy(x).to(dev).half(), L, act="prelu", want32=True)
    ref = orc.prelu(orc.conv2d_transpose(x, w, b, (s, s)), a)
    close(y32, ref, rel=2e-5)
    close(y16, ref, rel=1.2e-3)


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(1, 16, 32, 32, 16), (2, 8, 64, 16, 3), (1, 5, 8, 16, 16), (1, 32, 32, 32, 32)])
def test_conv2d_transpose_s1_xfold(B, H, W, Cin, Cout):
    """x-folded formulation of the thin stride-1 transposed convs (e_conv10 / e_conv11 shapes) vs the oracle."""
    ops = _ops()
    rng = np.random.default_rng(Cin + Cout + W)
    x = q16(rng.standard_normal((B, H, W, Cin)))
    w = q16(rng.standard_normal((4, 4, Cout, Cin)) / np.sqrt(16 * Cin))
    b = (rng.standard_normal(Cout) * 0.1).astype(np.float32)
    a = rng.uniform(0, 0.3, Cout).astype(np.float32)
    F = ops.XFoldConvT.factor(Cin, W)
    assert F == 64 // Cin
    L = ops.XFoldConvT(torch.from_numpy(w), torch.from_numpy(b), F)
    xt = torch.from_numpy(x).to(dev).half()
    y16, y32 = ops.conv2d_transpose_xfold(xt, L, act="prelu", alpha=torch.from_numpy(a).to(dev), want32=True)
    ref = orc.prelu(orc.conv2d_transpose(x, w, b, (1, 1)), a)
    close(y32, ref, rel=2e-5)
    close(y16, ref, rel=1.2e-3)
    y = ops.conv2d_transpose_xfold(xt, L, act="sigmoid", want16=False, want32=True)
    close(y, torch.sigmoid(orc.conv2d_transpose(x, w, b, (1, 1))), abs_=2e-6)


@pytest.mark.parametrize("B,H,W,Cin,Cout,tw", [(1, 16, 16, 64, 64, 0), (2, 24, 20, 128, 256, 16), (1, 8, 8, 64, 16, 8),
                                                 (1, 64, 64, 64, 128, 32), (1, 5, 9, 64, 32, 0)])
def test_conv2d_yhalo_sharing(B, H, W, Cin, Cout, tw):
    """The 3 ky taps of a 3x3 conv sharing one activation halo load (A box of BH+2 rows, operands at row offsets)
    vs the oracle, incl. ragged tiles and image borders inside the halo."""
    ops = _ops()
    rng = np.random.default_rng(H * W + Cin)
    x = q16(rng.standard_normal((B, H, W, Cin)))
    w = q16(rng.standard_normal((3, 3, Cin, Cout)) / np.sqrt(9 * Cin))
    b = (rng.standard_normal(Cout) * 0.1).astype(np.float32)
    L = ops.pack_conv("conv2d", torch.from_numpy(w), torch.from_numpy(b), None)
    taps = [(kx - 1, ky - 1, 0) for ky in range(3) for kx in range(3)]
    y = torch.empty(B, H, W, Cout, device=dev, dtype=torch.float32)
    ops.conv_igemm_raw(torch.from_numpy(x).to(dev).half(), L.w, L.bias, taps, 2, B, H, W, 1, Cin, Cout, L.cout_pad,
                       out32=y, ny=3, tile_w=tw)
    close(y, orc.conv2d(x, w, b), rel=2e-5)


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(1, 16, 16, 64, 32), (2, 8, 8, 256, 128), (1, 7, 9, 16, 16), (1, 32, 32, 128, 64)])
def test_conv2d_transpose_s2_merged(B, H, W, Cin, Cout):
    """One-launch form of the k=4 stride-2 transposed conv (N = 4*Cout, 9 taps, split output addressing) vs the oracle."""
    ops = _ops()
    rng = np.random.default_rng(Cin + Cout + H)
    x = q16(rng.standard_normal((B, H, W, Cin)))
    w = q16(rng.standard_normal((4, 4, Cout, Cin)) / np.sqrt(4 * Cin))
    b = (rng.standard_normal(Cout) * 0.1).astype(np.float32)
    a = rng.uniform(0, 0.3, Cout).astype(np.float32)
    L = ops.MergedConvT2(torch.from_numpy(w), torch.from_numpy(b))
    y16, y32 = ops.conv2d_transpose_s2_merged(torch.from_numpy(x).to(dev).half(), L, act="prelu",
                                              alpha=torch.from_numpy(a).to(dev), want32=True)
    ref = orc.prelu(orc.conv2d_transpose(x, w, b, (2, 2)), a)
    close(y32, ref, rel=2e-5)
    close(y16, ref, rel=1.2e-3)


@pytest.mark.parametrize("B,H,W,Cin,Cout,k", [(2, 16, 16, 64, 256, 3), (1, 24, 20, 64, 64, 3), (1, 5, 9, 32, 32, 3),
                                              (1, 64, 64, 128, 16, 1), (3, 32, 32, 128, 128, 4)])
def test_tma_store_epilogue_bit_identical(B, H, W, Cin, Cout, k):
    """rn_tuning.tma_store is accepted and ignored (the sm_90 kernel has one, direct-store epilogue): either setting writes
    the same result -- incl. ragged tiles, residual adds and untouched neighbours -- and it matches the oracle."""
    ops = _ops()
    rng = np.random.default_rng(B * H + Cout)
    x = torch.from_numpy(q16(rng.standard_normal((B, H, W, Cin)))).to(dev).half()
    w = torch.from_numpy(q16(rng.standard_normal((k, k, Cin, Cout)) / np.sqrt(k * k * Cin)))
    L = ops.pack_conv("conv2d", w, torch.from_numpy((rng.standard_normal(Cout) * 0.1).astype(np.float32)),
                      torch.from_numpy(rng.uniform(0, 0.3, Cout).astype(np.float32)))
    res = torch.from_numpy(q16(rng.standard_normal((B, H, W, Cout)))).to(dev).half()
    outs = []
    for on in (-1, 1):              # rn_tuning.tma_store: -1 = off, 1 = on
        y1 = ops.conv2d(x, L, act="prelu", tune=dict(tma_store=on))
        y2 = ops.conv2d(x, L, act=None, residual=res, tune=dict(tma_store=on))
        torch.cuda.synchronize()
        outs.append((y1.clone(), y2.clone()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    close(outs[1][0], orc.prelu(orc.conv2d(x.float().cpu().numpy(), w.numpy(), L.bias[:Cout].cpu().numpy()),
                                L.alpha[:Cout].cpu().numpy()), rel=1.2e-3)


def test_conv_bf16_variant():
    ops = _ops()
    rng = np.random.default_rng(3)
    x = torch.from_numpy(rng.standard_normal((1, 16, 16, 64)).astype(np.float32)).bfloat16()
    w = torch.from_numpy((rng.standard_normal((3, 3, 64, 64)) / 24).astype(np.float32)).bfloat16().float()
    L = ops.pack_conv("conv2d", w, torch.zeros(64), None, dtype=torch.bfloat16)
    y = ops.conv2d(x.to(dev), L, want16=False, want32=True)
    close(y, orc.conv2d(x.float().numpy(), w.numpy(), None), rel=2e-5)


def test_conv_linearity_and_tile_schedule_full_size():
    """BASELINE-size layer (B=24, 64x64, 1024->1024, 3x3): linearity f(2x) = 2 f(x) (exact in fp16: power of two),
    independence from the persistent-CTA count, and agreement with a cuDNN fp32 conv on a slice."""
    ops = _ops()
    torch.manual_seed(0)
    B = 24
    x = torch.randn(B, 64, 64, 1024, device=dev).half()
    w = torch.randn(3, 3, 1024, 1024, device=dev) / 96.0
    L = ops.pack_conv("conv2d", w, torch.zeros(1024), None)
    y, y32 = ops.conv2d(x, L, want32=True)
    y2_32 = ops.conv2d(x * 2, L, want16=False, want32=True)
    assert torch.equal(y2_32, y32 * 2)        # fp32 accumulators scale exactly (fp16 outputs do not: subnormals)
    # same work on 37 CTAs instead of 132: different tile->CTA assignment, identical result
    taps = [(kx - 1, ky - 1, 0) for ky in range(3) for kx in range(3)]
    y3 = torch.empty_like(y)
    ops.conv_igemm_raw(x, L.w, L.bias, taps, 2, B, 64, 64, 1, 1024, 1024, 1024, out16=y3, max_ctas=37, ny=3)
    assert torch.equal(y3, y)                 # same accumulation order (y-halo sharing on, as in conv2d), other CTA count
    ops.conv_igemm_raw(x, L.w, L.bias, taps, 2, B, 64, 64, 1, 1024, 1024, 1024, out16=y3, ny=0)
    close(y3, y, rel=2e-3)                    # tap-major order without halo sharing: same result up to fp16 rounding
    ref = torch.nn.functional.conv2d(x[:1].permute(0, 3, 1, 2).float(), w.half().float().permute(3, 2, 0, 1),
                                     padding=1).permute(0, 2, 3, 1)
    close(y[:1], ref, rel=1.5e-3)


@pytest.mark.parametrize("cluster,cta_group", [(1, 1), (2, 1), (4, 1)])
@pytest.mark.parametrize("bn", [256, 128])
def test_conv_cluster_multicast_bit_identical(cluster, cta_group, bn):
    """The weight-tile TMA multicast across a 2/4-CTA cluster may not change a single bit of the result."""
    ops = _ops()
    torch.manual_seed(1)
    B, H, W, Cin, Cout = 3, 32, 32, 128, 256                    # 24 M tiles: divisible by 4
    x = torch.randn(B, H, W, Cin, device=dev).half()
    w = torch.randn(3, 3, Cin, Cout, device=dev) / (9 * Cin) ** 0.5
    L = ops.pack_conv("conv2d", w, torch.randn(Cout) * 0.1, torch.rand(Cout) * 0.3)
    taps = [(kx - 1, ky - 1, 0) for ky in range(3) for kx in range(3)]
    ref = torch.empty(B, H, W, Cout, device=dev, dtype=torch.float16)
    ops.conv_igemm_raw(x, L.w, L.bias, taps, 2, B, H, W, 1, Cin, Cout, L.cout_pad, out16=ref, alpha=L.alpha, act=1,
                       cluster=1, cta_group=1)
    close(ref, orc.prelu(orc.conv2d(x.float().cpu().numpy(), w.half().float().cpu().numpy(), L.bias[:Cout].cpu().numpy()),
                         L.alpha[:Cout].cpu().numpy()), rel=1.2e-3)
    out = torch.empty_like(ref)
    ops.conv_igemm_raw(x, L.w, L.bias, taps, 2, B, H, W, 1, Cin, Cout, L.cout_pad, out16=out, alpha=L.alpha, act=1,
                       force_bn=bn, cluster=cluster, cta_group=cta_group)
    assert torch.equal(out, ref)


@pytest.mark.parametrize("case", ["3x3_bn128_yhalo", "1x1_bn64_ragged", "banded_res", "merged_tconv", "xfold"])
def test_conv_m_subtiles_bit_identical(case):
    """msub = 2 (two 128-row accumulators per CTA share each weight stage) must not change a bit: plain 3x3 with
    y-halo (BN = 128), a 1x1 with BN = 64 on an image whose height is not a multiple of the doubled tile
    (TMA zero fill / row clipping on the second sub-tile), the banded 3^3 conv with residual + PReLU, the merged
    stride-2 transposed conv and the x-folded thin transposed conv."""
    ops = _ops()
    torch.manual_seed(4)

    def both(fn):
        """msub 1/2 x epilogue_groups 1/2 (the latter is ignored): all four runs must agree bit for bit."""
        outs = []
        for m in (1, 2):
            for g in (1, 2):
                outs.append(fn(dict(msub=m, epilogue_groups=g)).clone())
        assert all(torch.equal(outs[0], o) for o in outs[1:])
        return outs[0]

    if case == "3x3_bn128_yhalo":
        B, H, W, Cin, Cout = 2, 48, 32, 64, 128
        x = torch.randn(B, H, W, Cin, device=dev).half()
        w = torch.randn(3, 3, Cin, Cout, device=dev) / (9 * Cin) ** 0.5
        L = ops.pack_conv("conv2d", w, torch.randn(Cout) * 0.1, torch.rand(Cout) * 0.3)
        res = torch.randn(B, H, W, Cout, device=dev).half()
        y = both(lambda t: ops.conv2d(x, L, act="prelu", residual=res, tune=t))
        want = orc.prelu(orc.conv2d(x.float().cpu().numpy(), w.half().float().cpu().numpy(), L.bias[:Cout].cpu().numpy()),
                         L.alpha[:Cout].cpu().numpy()) + res.float().cpu().numpy()
        close(y, want, rel=1.5e-3)
    elif case == "1x1_bn64_ragged":
        B, H, W, Cin, Cout = 3, 20, 24, 32, 64          # H = 20: second sub-tile of the last tile row is partly outside
        x = torch.randn(B, H, W, Cin, device=dev).half()
        w = torch.randn(1, 1, Cin, Cout, device=dev) / Cin ** 0.5
        L = ops.pack_conv("conv2d", w, torch.randn(Cout) * 0.1, None)
        y = both(lambda t: ops.conv2d(x, L, tune=t))
        close(y, orc.conv2d(x.float().cpu().numpy(), w.half().float().cpu().numpy(), L.bias[:Cout].cpu().numpy()), rel=1.5e-3)
    elif case == "banded_res":
        x = torch.randn(2, 32, 32, 32, 32, device=dev).half()
        res = torch.randn(2, 32, 32, 32, 32, device=dev).half()
        w = torch.randn(3, 3, 3, 32, 32, device=dev) / (27 * 32) ** 0.5
        Lb = ops.BandedConv3d(w, torch.randn(32) * 0.1)
        al = torch.rand(32, device=dev) * 0.3
        y = both(lambda t: ops.conv3d_banded(x, Lb, act="prelu", alpha=al, residual=res, tune=t))
        want = orc.prelu(orc.conv3d(x.float().cpu().numpy(), w.half().float().cpu().numpy(), Lb.bias.cpu().numpy(), (1, 1, 1)),
                         al.cpu().numpy()) + res.float().cpu().numpy()
        close(y, want, rel=1.5e-3)
    elif case == "merged_tconv":
        x = torch.randn(2, 32, 32, 64, device=dev).half()
        w = torch.randn(4, 4, 32, 64, device=dev) / (16 * 64) ** 0.5
        L = ops.MergedConvT2(w, torch.randn(32) * 0.1)
        al = torch.rand(32, device=dev) * 0.3
        y = both(lambda t: ops.conv2d_transpose_s2_merged(x, L, act="prelu", alpha=al, tune=t))
        want = orc.prelu(orc.conv2d_transpose(x.float().cpu().numpy(), w.half().float().cpu().numpy(),
                                              L.bias[:32].cpu().numpy(), (2, 2)), al.cpu().numpy())
        close(y, want, rel=1.5e-3)
    else:
        x = torch.randn(2, 64, 64, 32, device=dev).half()
        w = torch.randn(4, 4, 16, 32, device=dev) / (16 * 32) ** 0.5
        b = torch.randn(16) * 0.1
        L = ops.XFoldConvT(w, b, ops.XFoldConvT.factor(32, 64))
        al = torch.rand(16, device=dev) * 0.3
        y = both(lambda t: ops.conv2d_transpose_xfold(x, L, act="prelu", alpha=al, tune=t))
        want = orc.prelu(orc.conv2d_transpose(x.float().cpu().numpy(), w.half().float().cpu().numpy(), b.numpy(), (1, 1)),
                         al.cpu().numpy())
        close(y, want, rel=1.5e-3)


def test_conv_two_epilogue_groups_bit_identical():
    """rn_tuning.epilogue_groups is accepted and ignored (both consumer warpgroups always store their own rows): 1 and 2 give
    the same bits, including ragged image edges and the residual / sigmoid epilogues, and match the oracle."""
    ops = _ops()
    torch.manual_seed(9)
    for (B, H, W, Cin, Cout, k, act, use_res) in ((4, 32, 32, 256, 256, 1, "prelu", False), (3, 24, 40, 128, 512, 1, None, True),
                                                  (2, 32, 32, 64, 256, 4, "sigmoid", False), (2, 16, 48, 128, 128, 3, "prelu", True)):
        x = torch.randn(B, H, W, Cin, device=dev).half()
        w = torch.randn(k, k, Cin, Cout, device=dev) / (k * k * Cin) ** 0.5
        L = ops.pack_conv("conv2d", w, torch.randn(Cout) * 0.1, torch.rand(Cout) * 0.3)
        res = torch.randn(B, H, W, Cout, device=dev).half() if use_res else None
        outs = []
        for g in (1, 2):
            outs.append(ops.conv2d(x, L, act=act, residual=res, tune=dict(epilogue_groups=g)).clone())
        assert torch.equal(outs[0], outs[1]), (B, H, W, Cin, Cout, k, act, use_res)
        want = orc.conv2d(x.float().cpu().numpy(), w.half().float().cpu().numpy(), L.bias[:Cout].cpu().numpy())
        if act == "prelu":
            want = orc.prelu(want, L.alpha[:Cout].cpu().numpy())
        elif act == "sigmoid":
            want = 1.0 / (1.0 + np.exp(-want))
        if use_res:
            want = want + res.float().cpu().numpy()
        close(outs[1], want, rel=1.5e-3)


# ----------------------------------------------------------------------------------------- thin conv3d / misc
def test_conv3d_direct_first_layers():
    ops = _ops()
    rng = np.random.default_rng(13)
    x = rng.random((1, 16, 16, 32, 1)).astype(np.float32)
    w = (rng.standard_normal((5, 5, 5, 1, 8)) / np.sqrt(125)).astype(np.float32)
    b = (rng.standard_normal(8) * 0.1).astype(np.float32)
    a = rng.uniform(0, 0.3, 8).astype(np.float32)
    t = lambda v: torch.from_numpy(v).to(dev)
    y = ops.conv3d_direct(t(x), t(w), t(b), t(a), (2, 2, 2))
    close(y, orc.prelu(orc.conv3d(x, w, b, (2, 2, 2)), a), rel=1.2e-3)
    x = q16(rng.standard_normal((1, 8, 8, 32, 8)))
    w = (rng.standard_normal((3, 3, 3, 8, 16)) / np.sqrt(27 * 8)).astype(np.float32)
    b = (rng.standard_normal(16) * 0.1).astype(np.float32)
    a = rng.uniform(0, 0.3, 16).astype(np.float32)
    y = ops.conv3d_direct(t(x).half(), t(w), t(b), t(a), (1, 1, 2))
    close(y, orc.prelu(orc.conv3d(x, w, b, (1, 1, 2)), a), rel=1.2e-3)


def test_resample_conv1_fused_bit_identical_to_unfused_and_matches_oracle(golden_dir):
    """SURVEY 8 f-1: resampler + axis transform + e_conv1 + bias + PReLU in one kernel with empty-tile skipping must
    equal, bit for bit, rn_resample_f32(transform) followed by rn_conv3d_direct -- on the chair fixture (mostly empty
    tiles), on dense random occupancy with poses that clip the cube at the grid border (partial tiles, SAME padding
    on every face) and for a reduced grid; and it must match the CPU oracle within one fp16 rounding."""
    ops = _ops()
    from rendernet_b200.engine import RenderEngine
    rng = np.random.default_rng(21)
    w = (rng.standard_normal((5, 5, 5, 1, 8)) / np.sqrt(125)).astype(np.float32)
    b = (rng.standard_normal(8) * 0.1).astype(np.float32)
    a = rng.uniform(0.05, 0.3, 8).astype(np.float32)
    t = lambda v: torch.from_numpy(np.ascontiguousarray(v)).to(dev)
    bv = np.load(os.path.join(golden_dir, "binvox.npz"))
    chair = np.unpackbits(bv["chair_bits"]).reshape(1, 64, 64, 64, 1).astype(np.float32)
    dense = rng.random((3, 64, 64, 64, 1)).astype(np.float32)
    poses = np.array([[4.363, 0.524, 1.0], [0.3, 1.2, 1.32], [2.0, -0.4, 2.2], [5.5, 2.8, 0.74]], np.float32)
    vox = np.concatenate([chair, dense], 0)
    for new_size, v in ((128, vox), (32, vox[:, :16, :16, :16]), (16, vox[:2, :8, :8, :8])):
        size = v.shape[1]
        minv = t(RenderEngine.pose_to_matrix(poses[:v.shape[0]], size, new_size))
        for alpha in (t(a), None):
            fused = ops.resample_conv1(t(v), minv, new_size, t(w), t(b), alpha)
            grid = ops.resample(t(v), minv, new_size, True)
            unfused = ops.conv3d_direct(grid, t(w), t(b), alpha, (2, 2, 2))
            assert fused.shape == unfused.shape == (v.shape[0], new_size // 2, new_size // 2, new_size // 2, 8)
            assert torch.equal(fused, unfused), (new_size, alpha is None)
        if new_size == 32:
            want = orc.prelu(orc.conv3d(grid.cpu().numpy(), w, b, (2, 2, 2)), a)
            close(ops.resample_conv1(t(v), minv, new_size, t(w), t(b), t(a)), want, rel=1.2e-3)
    # an all-empty input exercises only the skip path: output == PReLU(bias) everywhere
    zero = torch.zeros(1, 64, 64, 64, 1, device=dev)
    y = ops.resample_conv1(zero, t(RenderEngine.pose_to_matrix(poses[:1], 64, 128)), 128, t(w), t(b), t(a))
    const = np.where(b > 0, b, a * b).astype(np.float32)
    assert torch.equal(y, torch.from_numpy(const).to(dev).half().expand_as(y))
    with pytest.raises(Exception):
        ops.resample_conv1(zero, minv[:1], 24, t(w), t(b), t(a))      # new_size % 16 != 0 is rejected (rc -2)


def _rle_bytes(grid_xyz, max_run=255, zero_runs=False):
    """Encode a bool [d0,d1,d2] grid (x, y, z) the way binvox files store it: x-z-y order, (value, count) byte pairs."""
    flat = np.transpose(grid_xyz, (0, 2, 1)).reshape(-1).astype(np.uint8)
    out = bytearray()
    i = 0
    while i < flat.size:
        j = i
        while j < flat.size and flat[j] == flat[i] and j - i < max_run:
            j += 1
        out += bytes([int(flat[i]), j - i])
        if zero_runs and (i % 7 == 0):
            out += bytes([1 - int(flat[i]), 0])           # legal zero-length run
        i = j
    return bytes(out)


def test_binvox_decode_on_device_matches_reader(golden_dir, tmp_path):
    """SURVEY 8 f-2: rn_binvox_decode (RLE payload -> float32 grid on the GPU) == tools/binvox_rw.read_as_3d_array
    (:58-93) on the reference's own fixtures (chair, teapot occupancy known-answers), batched, with short and
    zero-length runs, with and without the axis fix."""
    import io
    from rendernet_b200 import binvox_rw
    bv = np.load(os.path.join(golden_dir, "binvox.npz"))
    grids = {k: np.unpackbits(bv[k + "_bits"]).reshape(64, 64, 64).astype(bool) for k in ("chair", "teapot")}
    hdr = b"#binvox 1\ndim 64 64 64\ntranslate 0 0 0\nscale 1\ndata\n"
    files = [hdr + _rle_bytes(grids["chair"]), hdr + _rle_bytes(grids["teapot"], max_run=17),
             hdr + _rle_bytes(grids["teapot"], zero_runs=True)]
    for fix in (True, False):
        want = np.stack([binvox_rw.read_as_3d_array(io.BytesIO(f), fix_coords=fix).data for f in files])
        got = binvox_rw.read_to_device([io.BytesIO(f) for f in files], fix_coords=fix)
        assert got.dtype == torch.float32 and tuple(got.shape) == (3, 64, 64, 64, 1)
        assert np.array_equal(got.cpu().numpy()[..., 0], want.astype(np.float32))
    assert int(got[1].sum()) == 27933                                       # teapot occupancy (SURVEY 4)
    rng = np.random.default_rng(0)                                          # non-cubic dims, dense random occupancy
    g = rng.random((5, 12, 7)) < 0.5
    f = b"#binvox 1\ndim 5 12 7\ntranslate 0 0 0\nscale 1\ndata\n" + _rle_bytes(g)
    got = binvox_rw.read_to_device(io.BytesIO(f))
    want = binvox_rw.read_as_3d_array(io.BytesIO(f)).data
    assert tuple(got.shape) == (1,) + want.shape + (1,) and np.array_equal(got.cpu().numpy()[0, ..., 0], want)
    with pytest.raises(IOError):
        binvox_rw.read_to_device(io.BytesIO(hdr + _rle_bytes(grids["chair"])[:-2]))     # truncated payload


def test_bias_act_and_casts():
    ops = _ops()
    rng = np.random.default_rng(5)
    x = q16(rng.standard_normal((2, 5, 7, 24)))
    r = q16(rng.standard_normal((2, 5, 7, 24)))
    a = rng.uniform(0, 0.3, 24).astype(np.float32)
    y = ops.bias_act(torch.from_numpy(x).to(dev).half(), None, torch.from_numpy(a).to(dev), "prelu",
                     residual=torch.from_numpy(r).to(dev).half())
    close(y, orc.prelu(x, a) + torch.from_numpy(r), rel=1.2e-3)
    z = ops.cast_to_f32(ops.cast_to_16(torch.from_numpy(x).to(dev)))
    assert torch.equal(z.cpu(), torch.from_numpy(x))


def test_invalid_arguments_raise():
    ops = _ops()
    from rendernet_b200._lib import RenderNetCudaError
    x = torch.zeros(1, 8, 8, 24, device=dev, dtype=torch.float16)     # Cin not a multiple of 16
    with pytest.raises(RenderNetCudaError):
        ops.conv_igemm_raw(x, x, torch.zeros(16, device=dev), [(0, 0, 0)], 2, 1, 8, 8, 1, 24, 16, 16, out16=x)
    with pytest.raises(RuntimeError):
        ops.resample(torch.zeros(1, 4, 4, 4, 1), torch.zeros(1, 3, 4), 8, True)     # CPU tensors are rejected
