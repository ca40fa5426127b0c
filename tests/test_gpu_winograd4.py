"""Exact-mode Winograd F(4x4, 3x3) trunk convolution on the device (rn_winograd.cu): each transform kernel against its float64
formula (borders, a 4x4 image, a 20x36 image), the 36-position GEMM alone with a NaN tail on M, the whole convolution at B = 24
against a float64 convolution at the trunk's bar, large activations, F(2x2)'s bits when the tile is forced to 2, and the same
bits at B = 24, 8 and 1."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
dev = "cuda"
BAR = 2.5e-5     # test_gpu_exact_trunk_b24.py: the trunk's accumulation bar, of the output scale


def _ops():
    from rendernet_b200 import ops
    return ops


def _mats():
    BT, G, AT = _ops().wino4_matrices()
    return torch.from_numpy(BT), torch.from_numpy(G), torch.from_numpy(AT)


def _pair_f64(planes):
    return planes[0].double() + planes[1].double()


@pytest.mark.parametrize("B,H,W,C", [(1, 4, 4, 64), (2, 20, 36, 64), (3, 8, 8, 128)])
def test_input_transform_vs_float64(B, H, W, C):
    ops = _ops()
    from rendernet_b200._lib import check, lib
    BT = _mats()[0]
    g = torch.Generator().manual_seed(H * W + C)
    x = torch.randn(B, H, W, C, generator=g) * 5
    xs = ops.cast_to_16(x.to(dev), fmt=2)
    v = torch.empty(2, 36, B, H // 4, W // 4, C, device=dev, dtype=torch.float16)
    check(lib.rn_winograd4_in(xs.planes.data_ptr(), v.data_ptr(), B, H, W, C, None), "rn_winograd4_in")
    torch.cuda.synchronize()
    d = F.pad(_pair_f64(xs.planes.cpu()), (0, 0, 1, 1, 1, 1))               # the operand the kernel reads, SAME-padded
    d = d.unfold(1, 6, 4).unfold(2, 6, 4)                                   # [B, H/4, W/4, C, 6, 6]
    ref = 0.5 * torch.einsum("ai,nhwcij,bj->abnhwc", BT, d, BT).reshape(36, B, H // 4, W // 4, C)
    got = _pair_f64(v.cpu())
    s = float(ref.abs().max())
    assert float((got - ref).abs().max()) <= 2.0 ** -20 * s
    assert float(ref.abs().max()) <= 4.5 * float(x.abs().max())


@pytest.mark.parametrize("act,res,u_exp", [("prelu", "pair", 12), (None, "f32", 0), (None, None, -3)])
def test_output_transform_vs_float64(act, res, u_exp):
    ops = _ops()
    from rendernet_b200._lib import check, lib
    AT = _mats()[2]
    B, H, W, C = 2, 20, 36, 64
    g = torch.Generator().manual_seed(7 + u_exp)
    m = torch.randn(36, B, H // 4, W // 4, C, generator=g) * 10 * 2.0 ** (u_exp - 1)
    bias = torch.randn(C, generator=g)
    alpha = torch.rand(C, generator=g) * 0.3
    r = torch.randn(B, H, W, C, generator=g) * 4
    rdev, rf32 = (None, 0)
    if res == "pair":
        rdev = ops.cast_to_16(r.to(dev), fmt=2).planes
    elif res == "f32":
        rdev, rf32 = r.to(dev), 1
    out16 = torch.empty(2, B, H, W, C, device=dev, dtype=torch.float16)
    out32 = torch.empty(B, H, W, C, device=dev)
    a = ops._ACT[act]
    md, bd, ad = m.to(dev), bias.to(dev), alpha.to(dev)
    check(lib.rn_winograd4_out(md.data_ptr(), bd.data_ptr(), ad.data_ptr() if act else None, a,
                               rdev.data_ptr() if rdev is not None else None, rf32, out16.data_ptr(), out32.data_ptr(),
                               B, H, W, C, u_exp, None), "rn_winograd4_out")
    torch.cuda.synchronize()
    mm = m.double().reshape(6, 6, B, H // 4, W // 4, C)
    y = 2.0 ** (1 - u_exp) * torch.einsum("ia,abnhwc,jb->nhiwjc", AT, mm, AT).reshape(B, H, W, C) + bias.double()
    if act == "prelu":
        y = torch.clamp(y, min=0) + alpha.double() * torch.clamp(y, max=0)
    if res == "pair":
        y = y + _pair_f64(rdev.cpu())
    elif res == "f32":
        y = y + r.double()
    s = float(y.abs().max())
    assert float((out32.cpu().double() - y).abs().max()) <= 2.0 ** -20 * s
    assert float((_pair_f64(out16.cpu()) - y).abs().max()) <= 2.0 ** -20 * s


def _pair(shape, scale, g):
    v = (torch.rand(shape, generator=g) * 2 - 1).to(dev) * scale
    hi = v.half()
    lo = (v - hi.float()).half()
    return torch.stack([hi, lo]).contiguous()


@pytest.mark.parametrize("B,H,W,C", [(24, 64, 64, 1024), (1, 20, 36, 512)])
def test_36_position_gemm_vs_float64(B, H, W, C):
    """M = V . U for all 36 positions and every N tile; the 20 x 36 image's 9-wide position images leave part of every 128-row
    tile outside the image.  M has a NaN tail: every valid row must hold its own value and the tail must stay untouched."""
    from rendernet_b200._lib import check, lib
    g = torch.Generator().manual_seed(B * H * W + C)
    rows = B * (H // 4) * (W // 4)
    v = _pair((36, rows, C), 4.0, g)
    u = _pair((36, C, C), 2048.0, g)
    tail = 4096
    m = torch.full((36 * rows * C + tail,), float("nan"), device=dev)
    check(lib.rn_winograd4_gemm(v.data_ptr(), u.data_ptr(), m.data_ptr(), B, H, W, C, None, None), "rn_winograd4_gemm")
    torch.cuda.synchronize()
    assert bool(torch.isnan(m[36 * rows * C:]).all()), "the GEMM wrote past the end of M"
    mm = m[:36 * rows * C].view(36, rows, C)
    worst = 0.0
    for p in range(36):
        vp = v[0, p].double() + v[1, p].double()
        up = u[0, p].double() + u[1, p].double()
        ref = vp @ up.T
        bound = vp.abs() @ up.abs().T
        got = mm[p].double()
        assert bool(torch.isfinite(got).all()), f"position {p}: rows left unwritten"
        ratio = float(((got - ref).abs() / bound).max())
        worst = max(worst, ratio)
        assert ratio <= BAR, f"position {p}: error {ratio:.2e} of sum |v||u|"
    print(f"winograd4 gemm B={B} {H}x{W} C={C}: max error {worst:.2e} of sum |v||u|")


def _trunk(C, seed, scale=3.0, B=24):
    g = torch.Generator().manual_seed(seed)
    x = (torch.rand(B, 64, 64, C, generator=g) * 2 - 1) * scale
    w = (torch.rand(3, 3, C, C, generator=g) * 2 - 1) * (6.0 / (9 * 2 * C)) ** 0.5
    b = torch.randn(C, generator=g) * 0.1
    al = torch.rand(C, generator=g) * 0.3
    res = torch.randn(B, 64, 64, C, generator=g)
    return x, w, b, al, res


def _ref(x, w, b, items, co):
    return F.conv2d(x[items].double().permute(0, 3, 1, 2), w[:, :, :, co].double().permute(3, 2, 0, 1), b[co].double(),
                    padding=1).permute(0, 2, 3, 1)


def test_winograd4_conv_b24_prelu_residual_vs_float64():
    """The trunk's res-block layer shapes at B = 24 on the F(4x4) path: PReLU into the hi/lo pair, then no activation with the
    pair residual; both outputs (fp32 and the pair) against float64 at the direct kernel's bar."""
    ops = _ops()
    x, w, b, al, res = _trunk(1024, 21)
    L = ops.pack_conv("conv2d", w, b, al, device=dev, fmt=2)
    xs, rs = ops.cast_to_16(x.to(dev), fmt=2), ops.cast_to_16(res.to(dev), fmt=2)
    y16, y32 = ops.conv2d(xs, L, act="prelu", want16=True, want32=True)
    z16, z32 = ops.conv2d(xs, L, act=None, residual=rs, want16=True, want32=True)
    assert list(L.wino) == [4]                                         # the F(4x4) path ran, and only it
    items, co = [0, 11, 23], slice(448, 512)
    pre = _ref(x, w, b, items, co)
    refs = (torch.clamp(pre, min=0) + al[co].double() * torch.clamp(pre, max=0), pre + res[items][..., co].double())
    for name, (o16, o32), ref in (("prelu", (y16, y32), refs[0]), ("residual", (z16, z32), refs[1])):
        s = float(ref.abs().max())
        e32 = float((o32[items][..., co].double().cpu() - ref).abs().max())
        e16 = float((_pair_f64(o16.planes[:, items][..., co].cpu()) - ref).abs().max())
        print(f"winograd4 3x3 1024 B=24 {name}: fp32 out {e32 / s:.2e}, pair out {e16 / s:.2e} of scale")
        assert e32 <= BAR * s and e16 <= BAR * s


def test_winograd4_conv_large_activations():
    """|x| ~ 1e4: V reaches 4.5 |x| (inside fp16's range), the result stays finite and in the bar."""
    ops = _ops()
    x, w, b, _, _ = _trunk(1024, 22, scale=1.0e4, B=2)
    L = ops.pack_conv("conv2d", w, b, None, device=dev, fmt=2)
    y = ops.conv2d(ops.cast_to_16(x.to(dev), fmt=2), L, want16=False, want32=True)
    assert 4 in L.wino and bool(torch.isfinite(y).all())
    items, co = [0, 1], slice(960, 1024)
    ref = _ref(x, w, b, items, co)
    s = float(ref.abs().max())
    err = float((y[items][..., co].double().cpu() - ref).abs().max())
    print(f"winograd4 |x|~1e4: {err / s:.2e} of scale")
    assert err <= BAR * s


def test_tile_2_is_f2x2_bit_for_bit():
    ops = _ops()
    from rendernet_b200._lib import check, lib
    x, w, b, al, res = _trunk(1024, 23, B=2)
    xs, rs = ops.cast_to_16(x.to(dev), fmt=2), ops.cast_to_16(res.to(dev), fmt=2)
    L = ops.pack_conv("conv2d", w, b, al, device=dev, fmt=2)
    B, H, W, C = x.shape
    ws = torch.empty(lib.rn_winograd_workspace_bytes(B, H, W, C), device=dev, dtype=torch.uint8)
    for act, r in (("prelu", None), (None, rs)):
        t2 = ops.conv2d(xs, L, act=act, residual=r, want16=True, want32=True, tune=dict(wino_tile=2))
        f2 = (torch.empty(2, B, H, W, C, device=dev, dtype=torch.float16), torch.empty(B, H, W, C, device=dev))
        a = ops._ACT[act]
        check(lib.rn_conv2d_winograd(xs.planes.data_ptr(), ops.winograd_filter(L).data_ptr(), L.bias.data_ptr(),
                                     L.alpha.data_ptr() if act else None, a, r.planes.data_ptr() if r is not None else None,
                                     0, f2[0].data_ptr(), f2[1].data_ptr(), B, H, W, C, ws.data_ptr(), ws.numel(), None,
                                     None), "rn_conv2d_winograd")
        f4 = ops.conv2d(xs, L, act=act, residual=r, want16=True, want32=True)
        assert torch.equal(t2[0].planes, f2[0]) and torch.equal(t2[1], f2[1])
        assert not torch.equal(f4[1], f2[1])                            # the default really is the other tile
    assert sorted(L.wino) == [2, 4]


def test_batch_sizes_give_the_same_bits():
    """Every 128-row GEMM tile lies inside one 16 x 16 position image and the transforms are per block, so an item's output
    does not depend on the batch it runs in."""
    ops = _ops()
    x, w, b, al, res = _trunk(1024, 24)
    xs, rs = ops.cast_to_16(x.to(dev), fmt=2), ops.cast_to_16(res.to(dev), fmt=2)
    L = ops.pack_conv("conv2d", w, b, al, device=dev, fmt=2)
    full = ops.conv2d(xs, L, act=None, residual=rs, want16=True, want32=True)
    for n, i0 in ((8, 16), (1, 5)):
        xi = ops.cast_to_16(x[i0:i0 + n].to(dev), fmt=2)
        ri = ops.cast_to_16(res[i0:i0 + n].to(dev), fmt=2)
        part = ops.conv2d(xi, L, act=None, residual=ri, want16=True, want32=True)
        assert torch.equal(part[1], full[1][i0:i0 + n])
        assert torch.equal(part[0].planes, full[0].planes[:, i0:i0 + n])
