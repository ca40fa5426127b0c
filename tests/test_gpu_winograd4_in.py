"""The exact-mode Winograd F(4x4, 3x3) input transform (rn_winograd4_in, rn_winograd.cu) at the shapes that exercise its
streaming layout: one CTA per (image, 64-channel slice, 8-block-column width tile, band of block rows).  V against float64 at
the trunk's batch, one channel slice, C = 512, a 4 x 4 image, a ragged 20 x 36 image, a width of 296 (ten width tiles, the
last one partial) and a 20 x 20 image whose few CTAs get split into bands of two block rows, the last one short; a NaN guard
on both sides of V; and the same bits for an item whatever batch it runs in."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
dev = "cuda"
NAN16 = 0x7E00


def _ops():
    from rendernet_b200 import ops
    return ops


def _run(xs, B, H, W, C, guard=0):
    """V of the pair xs as [2, 36, B, H/4, W/4, C] fp16, written into the middle of a buffer with `guard` fp16 NaNs on each
    side; returns (V, head guard, tail guard)."""
    from rendernet_b200._lib import check, lib
    n = 2 * 36 * B * (H // 4) * (W // 4) * C
    buf = torch.full((n + 2 * guard,), NAN16, device=dev, dtype=torch.int16).view(torch.float16)
    check(lib.rn_winograd4_in(xs.planes.data_ptr(), buf[guard:].data_ptr(), B, H, W, C, None), "rn_winograd4_in")
    torch.cuda.synchronize()
    return buf[guard:guard + n].view(2, 36, B, H // 4, W // 4, C), buf[:guard], buf[guard + n:]


def _check_vs_float64(x, xs, v, items, ch):
    """V of `items` x `ch` against 1/2 B^T d B in float64 of the pair the kernel read (SAME-padded 6 x 6 patches)."""
    BT = torch.from_numpy(_ops().wino4_matrices()[0])
    B, H, W, C = x.shape
    xp = xs.planes[:, items][..., ch].cpu().double()
    d = F.pad(xp[0] + xp[1], (0, 0, 1, 1, 1, 1)).unfold(1, 6, 4).unfold(2, 6, 4)   # [n, H/4, W/4, c, 6, 6]
    ref = 0.5 * torch.einsum("ai,nhwcij,bj->abnhwc", BT, d, BT).reshape(36, len(items), H // 4, W // 4, -1)
    vv = v[:, :, items][..., ch].cpu().double()
    got = vv[0] + vv[1]
    s = float(ref.abs().max())
    err = float((got - ref).abs().max())
    assert err <= 2.0 ** -20 * s, f"V error {err / s:.2e} of scale"
    assert s <= 4.5 * float(x[items][..., ch].abs().max())


@pytest.mark.parametrize("B,H,W,C", [(1, 4, 4, 64), (2, 64, 64, 64), (1, 20, 36, 512), (3, 20, 36, 128), (2, 8, 296, 64),
                                     (6, 20, 20, 1024)])
def test_input_transform_vs_float64(B, H, W, C):
    g = torch.Generator().manual_seed(B * H * W + C)
    x = torch.randn(B, H, W, C, generator=g) * 5
    xs = _ops().cast_to_16(x.to(dev), fmt=2)
    v, head, tail = _run(xs, B, H, W, C, guard=4096)
    assert bool(torch.isnan(head).all()) and bool(torch.isnan(tail).all()), "V written outside its buffer"
    assert not bool(torch.isnan(v).any()), "part of V left unwritten"
    _check_vs_float64(x, xs, v, list(range(B)), slice(0, C))


def test_input_transform_b24_vs_float64_and_batch_independence():
    """B = 24, 64 x 64, C = 1024 (the res2 trunk): seeded items and channels (one whole slice, and channels spread over the
    other slices) against float64; then items [i0, i0 + n) run at B = n give the same bits as in the B = 24 launch."""
    B, H, W, C = 24, 64, 64, 1024
    g = torch.Generator().manual_seed(2024)
    x = (torch.rand(B, H, W, C, generator=g) * 2 - 1) * 3
    ops = _ops()
    xs = ops.cast_to_16(x.to(dev), fmt=2)
    v, head, tail = _run(xs, B, H, W, C, guard=4096)
    assert bool(torch.isnan(head).all()) and bool(torch.isnan(tail).all()), "V written outside its buffer"
    assert not bool(torch.isnan(v).any()), "part of V left unwritten"
    items = sorted(torch.randperm(B, generator=g)[:3].tolist())
    spread = torch.randperm(C, generator=g)[:64].sort().values
    _check_vs_float64(x, xs, v, items, slice(448, 512))
    _check_vs_float64(x, xs, v, items, spread)
    for n, i0 in ((8, 16), (1, 5), (3, 0)):
        vn, _, _ = _run(ops.cast_to_16(x[i0:i0 + n].to(dev), fmt=2), n, H, W, C)
        assert torch.equal(vn.view(torch.int16), v[:, :, i0:i0 + n].view(torch.int16)), f"items {i0}..{i0 + n - 1} at B = {n}"
