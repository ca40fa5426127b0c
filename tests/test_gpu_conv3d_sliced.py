"""The depth-sliced 3^3 32 -> 32 conv3d (rn_conv3d_sliced_same, the Shader's res1 blocks).

GPU tests hold it against float64 convolutions (exact mode at the 2e-5-of-scale bar of the banded kernel's test; the fast
mode against fp16-rounded inputs at the bars of tests/test_gpu_kernels.py::test_conv3d_same), against the banded kernel it
replaces at full size, and check that it is deterministic and independent of the batch it runs in.  The host tests check
the packed filter layout and the launch plan without a GPU.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

dev = "cuda"


def _ops():
    from rendernet_b200 import ops
    return ops


def _wide(rng, shape, scale=1.0):
    """fp32 values over several binades (LO halves down in fp16's subnormal range)."""
    return (rng.standard_normal(shape) * np.exp(rng.uniform(-6.0, 1.0, shape)) * scale).astype(np.float32)


def _conv3d_np(x, w, b):
    """SAME 3^3 conv3d in float64 NumPy: x [B,H,W,D,Ci], w [ky,kx,kz,Ci,Co] (TF) -> [B,H,W,D,Co]."""
    B, H, W, D, _ = x.shape
    xp = np.pad(x.astype(np.float64), ((0, 0), (1, 1), (1, 1), (1, 1), (0, 0)))
    y = np.zeros((B, H, W, D, w.shape[-1])) + b
    for ky in range(3):
        for kx in range(3):
            for kz in range(3):
                y += xp[:, ky:ky + H, kx:kx + W, kz:kz + D] @ w[ky, kx, kz].astype(np.float64)
    return y


def _pack_np(w):
    """NumPy mirror of rn_pack_conv3d_sliced: [tap = ky*3 + kx][r = (2 - kz)*32 + co][ci]."""
    p = np.zeros((9, 96, 32), np.float32)
    for tap in range(9):
        for zs in range(3):
            p[tap, 32 * zs:32 * zs + 32, :] = w[tap // 3, tap % 3, 2 - zs].T
    return p


def _sliced_walk_np(x, packed, b):
    """The kernel's K walk on the host: tile-local input depth jl (input depth z0 - 1 + jl) feeds tile-local output depths
    z = jl-2 .. jl (clipped to the tile) through slice zs = z - (jl - 2) of the (ky, kx) filter tile."""
    B, H, W, D, _ = x.shape
    xp = np.pad(x.astype(np.float64), ((0, 0), (1, 1), (1, 1), (1, 1), (0, 0)))
    y = np.zeros((B, H, W, D, 32)) + b
    for z0 in range(0, D, 8):
        for jl in range(10):                      # input depth z0 - 1 + jl (padded index z0 + jl)
            for z in range(max(jl - 2, 0), min(jl, 7) + 1):
                zs = z - (jl - 2)
                for tap in range(9):
                    ky, kx = divmod(tap, 3)
                    wt = packed[tap, 32 * zs:32 * zs + 32, :].astype(np.float64)   # [co, ci]
                    y[:, :, :, z0 + z] += xp[:, ky:ky + H, kx:kx + W, z0 + jl] @ wt.T
    return y


def _ref64(x, w, b, al=None, res=None):
    """float64 reference on the device: conv3d (+ PReLU) (+ residual) of the unrounded fp32 tensors."""
    xt = torch.as_tensor(x).to(dev).double().permute(0, 4, 1, 2, 3)
    y = F.conv3d(F.pad(xt, (1, 1, 1, 1, 1, 1)), torch.as_tensor(w).to(dev).double().permute(4, 3, 0, 1, 2),
                 torch.as_tensor(b).to(dev).double()).permute(0, 2, 3, 4, 1)
    if al is not None:
        a = torch.as_tensor(al).to(dev).double()
        y = torch.clamp(y, min=0) + a * torch.clamp(y, max=0)
    if res is not None:
        y = y + torch.as_tensor(res).to(dev).double()
    return y


def _err(got, want):
    got, want = got.double(), want.double()
    assert got.shape == want.shape, (got.shape, want.shape)
    return float((got - want).abs().max()), float(want.abs().max())


def _layer(rng, scale=1.0):
    w = (rng.uniform(-1, 1, (3, 3, 3, 32, 32)) * np.sqrt(6.0 / (27 * 64)) * scale).astype(np.float32)
    b = rng.uniform(-0.1, 0.1, 32).astype(np.float32)
    al = rng.uniform(0.05, 0.3, 32).astype(np.float32)
    return w, b, al


# ----------------------------------------------------------------------------------------- host (no GPU)
def test_sliced_packed_layout_walk_matches_numpy_conv():
    """The packed [9][96][32] layout walked the way the kernel walks it (ten input depths per 8-depth tile, each into the
    three output depths it feeds) is the SAME 3^3 convolution."""
    rng = np.random.default_rng(1)
    x = rng.standard_normal((1, 5, 4, 16, 32)).astype(np.float32)
    w, b, _ = _layer(rng)
    got = _sliced_walk_np(x, _pack_np(w), b)
    want = _conv3d_np(x, w, b)
    assert np.abs(got - want).max() <= 1e-12 * max(np.abs(want).max(), 1.0)


@pytest.mark.parametrize("B,H,W,D", [(24, 64, 64, 32), (24, 16, 16, 32), (24, 32, 32, 32), (1, 20, 13, 16)])
@pytest.mark.parametrize("fmt", [0, 2])
def test_sliced_plan_fits_shared_memory(B, H, W, D, fmt):
    """Resident filter + >= 3 activation stages + staging panels fit the 227 KB opt-in; one persistent CTA per SM."""
    ops = _ops()
    pl = ops.SlicedConv3d.plan(B, H, W, D, fmt)
    assert pl["filter_bytes"] == (2 if fmt == 2 else 1) * 9 * 96 * 32 * 2
    assert pl["stage_bytes"] == 64 * 2 * 8 * 10
    assert pl["stages"] >= 3 and pl["smem_bytes"] <= pl["smem_limit"] == 232448
    assert pl["smem_bytes"] >= pl["filter_bytes"] + pl["stages"] * pl["stage_bytes"]
    assert pl["tiles"] == B * -(-H // 8) * -(-W // 8) * (D // 8)
    assert pl["grid"] == min(pl["tiles"], 132)
    print(f"B={B} {H}x{W}x{D} fmt={fmt}: {pl}")


def test_sliced_eligibility():
    ops = _ops()
    assert ops.SlicedConv3d.eligible(32, 32, 32) and ops.SlicedConv3d.eligible(32, 32, 8)
    assert not ops.SlicedConv3d.eligible(16, 32, 32)           # e_conv3 keeps the banded path
    assert not ops.SlicedConv3d.eligible(16, 16, 32)           # the Texture net's res1 too
    assert not ops.SlicedConv3d.eligible(32, 32, 12) and not ops.SlicedConv3d.eligible(32, 32, 32, 2)


# ----------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
def test_sliced_pack_matches_host_mirror():
    ops = _ops()
    rng = np.random.default_rng(2)
    w, b, _ = _layer(rng)
    for fmt in (0, 2):
        L = ops.SlicedConv3d(torch.from_numpy(w), torch.from_numpy(b), device=dev, fmt=fmt)
        want = torch.from_numpy(_pack_np(w)).reshape(-1)
        if fmt == 2:
            hi = want.half()
            lo = (want - hi.float()).half()
            assert torch.equal(L.w.cpu(), torch.stack([hi, lo]))
        else:
            assert torch.equal(L.w.cpu(), want.half())


SHAPES = [(24, 64, 64, 32), (4, 16, 16, 32), (4, 32, 32, 32), (2, 20, 13, 16)]


@pytest.mark.gpu
@pytest.mark.parametrize("B,H,W,D", SHAPES)
@pytest.mark.parametrize("epi", ["prelu_hilo_res", "none_f32_res"])
def test_sliced_exact_matches_float64(B, H, W, D, epi):
    """Exact mode (fp16 hi/lo pairs) vs float64: fp32 output and stored hi/lo pair within 2e-5 of the output scale."""
    ops = _ops()
    rng = np.random.default_rng(B * 100 + H + D)
    x = _wide(rng, (B, H, W, D, 32))
    w, b, al = _layer(rng)
    res = _wide(rng, (B, H, W, D, 32))
    L = ops.SlicedConv3d(torch.from_numpy(w), torch.from_numpy(b), device=dev, fmt=2)
    xs = ops.cast_to_16(torch.from_numpy(x).to(dev), fmt=2)
    if epi == "prelu_hilo_res":
        rs = ops.cast_to_16(torch.from_numpy(res).to(dev), fmt=2)
        y16, y32 = ops.conv3d_sliced(xs, L, act="prelu", residual=rs, alpha=torch.from_numpy(al).to(dev),
                                     want16=True, want32=True)
        ref = _ref64(x, w, b, al, res)
    else:
        y16, y32 = ops.conv3d_sliced(xs, L, act=None, residual=torch.from_numpy(res).to(dev), want16=True, want32=True)
        ref = _ref64(x, w, b, None, res)
    assert isinstance(y16, ops.Split16) and tuple(y16.shape) == (B, H, W, D, 32)
    e32, s = _err(y32, ref)
    e16, _ = _err(y16.float(), ref)
    print(f"sliced exact {B}x{H}x{W}x{D} {epi}: fp32-out err {e32:.2e}, pair-out err {e16:.2e} (scale {s:.2e})")
    assert e32 <= 2e-5 * s and e16 <= 2e-5 * s


@pytest.mark.gpu
@pytest.mark.parametrize("B,H,W,D", SHAPES)
def test_sliced_fast_matches_rounded_float64(B, H, W, D):
    """Fast mode (fp16 operands) vs float64 of the fp16-rounded inputs: 2e-5 (fp32 out), 1.2e-3 (fp16 out + residual)."""
    ops = _ops()
    rng = np.random.default_rng(B + H * 10 + D)
    x = torch.from_numpy(rng.standard_normal((B, H, W, D, 32)).astype(np.float32)).half()
    w, b, al = _layer(rng)
    w = torch.from_numpy(w).half().float().numpy()
    res = torch.from_numpy(rng.standard_normal((B, H, W, D, 32)).astype(np.float32)).half()
    L = ops.SlicedConv3d(torch.from_numpy(w), torch.from_numpy(b), device=dev, fmt=0)
    xt, rt = x.to(dev), res.to(dev)
    y1 = ops.conv3d_sliced(xt, L, act="prelu", alpha=torch.from_numpy(al).to(dev), want16=False, want32=True)
    y2 = ops.conv3d_sliced(xt, L, act=None, residual=rt)
    e1, s1 = _err(y1, _ref64(x.float().numpy(), w, b, al))
    e2, s2 = _err(y2.float(), _ref64(x.float().numpy(), w, b, None, res.float().numpy()))
    print(f"sliced fast {B}x{H}x{W}x{D}: prelu fp32 err {e1:.2e} (scale {s1:.2e}), residual fp16 err {e2:.2e} (scale {s2:.2e})")
    assert e1 <= 2e-5 * s1 and e2 <= 1.2e-3 * s2


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", [2, 0])
def test_sliced_agrees_with_banded_full_size(fmt):
    """B = 24, 64 x 64 x 32: the sliced and banded kernels differ only by fp32 summation order."""
    ops = _ops()
    rng = np.random.default_rng(7 + fmt)
    x = _wide(rng, (24, 64, 64, 32, 32)) if fmt == 2 else rng.standard_normal((24, 64, 64, 32, 32)).astype(np.float32)
    w, b, al = _layer(rng)
    xs = ops.cast_to_16(torch.from_numpy(x).to(dev), fmt=fmt)
    alpha = torch.from_numpy(al).to(dev)
    Ls = ops.SlicedConv3d(torch.from_numpy(w), torch.from_numpy(b), device=dev, fmt=fmt)
    Lb = ops.BandedConv3d(torch.from_numpy(w), torch.from_numpy(b), device=dev, fmt=fmt)
    ys = ops.conv3d_sliced(xs, Ls, act="prelu", alpha=alpha, want16=False, want32=True)
    yb = ops.conv3d_banded(xs, Lb, act="prelu", alpha=alpha, want16=False, want32=True)
    e, s = _err(ys, yb)
    print(f"sliced vs banded fmt={fmt}: max diff {e:.2e} (scale {s:.2e}, {e / s:.1e} of scale)")
    assert e <= 1e-5 * s


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", [2, 0])
def test_sliced_deterministic_and_batch_invariant(fmt):
    """Two runs are bit-identical, and B = 24 equals three B = 8 slices and B = 1, bit for bit."""
    ops = _ops()
    rng = np.random.default_rng(11)
    x = _wide(rng, (24, 64, 64, 32, 32))
    w, b, al = _layer(rng)
    res = _wide(rng, (24, 64, 64, 32, 32))
    L = ops.SlicedConv3d(torch.from_numpy(w), torch.from_numpy(b), device=dev, fmt=fmt)
    xt, rt, alpha = torch.from_numpy(x).to(dev), torch.from_numpy(res).to(dev), torch.from_numpy(al).to(dev)

    def run(sl):
        xs, rs = ops.cast_to_16(xt[sl].contiguous(), fmt=fmt), ops.cast_to_16(rt[sl].contiguous(), fmt=fmt)
        y = ops.conv3d_sliced(xs, L, act="prelu", residual=rs, alpha=alpha)
        return y.planes if fmt == 2 else y

    full = run(slice(0, 24))
    assert torch.equal(full, run(slice(0, 24)))
    ax = 1 if fmt == 2 else 0
    parts = torch.cat([run(slice(8 * i, 8 * i + 8)) for i in range(3)], dim=ax)
    assert torch.equal(full, parts)
    one = run(slice(13, 14))
    assert torch.equal(full.narrow(ax, 13, 1), one)
