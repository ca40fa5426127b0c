"""The per-position GEMM of the exact-mode Winograd convolution (rn_winograd_gemm) on its own: M = V . U for all 16 positions and
every N tile against float64 (V_hi + V_lo) . (U_hi + U_lo), at the trunk's B = 24, 64 x 64 and at a ragged 18 x 34 image whose
17-wide position images leave part of every 128-row tile outside the image.  M is allocated with a NaN tail: every valid row
must hold its own value (a row stored without its mask lands on another row's offset or in the tail) and the tail must stay
untouched."""
import pytest
import torch

pytestmark = pytest.mark.gpu
dev = "cuda"
BAR = 2.5e-5     # of sum_k |v_k| |u_k|: the fp32 accumulation of 3 x K/16 truncating MMA steps and the dropped lo . lo term


def _pair(shape, scale, g):
    """A random fp32 tensor and its fp16 hi/lo planes, stacked [2, *shape] as the library stores pairs."""
    v = (torch.rand(shape, generator=g) * 2 - 1).to(dev) * scale
    hi = v.half()
    lo = (v - hi.float()).half()
    return torch.stack([hi, lo]).contiguous()


@pytest.mark.parametrize("B,H,W,C", [(24, 64, 64, 1024), (1, 18, 34, 512)])
def test_per_position_gemm_vs_float64(B, H, W, C):
    from rendernet_b200._lib import check, lib
    g = torch.Generator().manual_seed(B * H * W + C)
    H2, W2 = H // 2, W // 2
    rows = B * H2 * W2
    v = _pair((16, rows, C), 4.0, g)                  # V [2][16][B, H/2, W/2, C]
    u = _pair((16, C, C), C ** -0.5, g)                # U [2][16][Cout][Cin]
    tail = 4096
    m = torch.full((16 * rows * C + tail,), float("nan"), device=dev)
    check(lib.rn_winograd_gemm(v.data_ptr(), u.data_ptr(), m.data_ptr(), B, H, W, C, None, None), "rn_winograd_gemm")
    torch.cuda.synchronize()
    assert bool(torch.isnan(m[16 * rows * C:]).all()), "the GEMM wrote past the end of M"
    mm = m[:16 * rows * C].view(16, rows, C)
    worst = 0.0
    for p in range(16):
        vp = v[0, p].double() + v[1, p].double()
        up = u[0, p].double() + u[1, p].double()
        ref = vp @ up.T
        bound = vp.abs() @ up.abs().T
        got = mm[p].double()
        assert bool(torch.isfinite(got).all()), f"position {p}: rows left unwritten"
        ratio = float(((got - ref).abs() / bound).max())
        worst = max(worst, ratio)
        assert ratio <= BAR, f"position {p}: error {ratio:.2e} of sum |v||u|"
    print(f"winograd gemm B={B} {H}x{W} C={C}: max error {worst:.2e} of sum |v||u|")
