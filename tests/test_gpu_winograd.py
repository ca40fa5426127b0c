"""Exact-mode Winograd F(2x2, 3x3) trunk convolution on the device (rn_winograd.cu): each transform kernel against its float64
formula (borders, 2x2 and non-square images), the whole convolution at B = 24 against a float64 convolution at the trunk's bar,
large activations, the direct kernel's bits when Winograd is switched off, and a changed filter never running with a stale U."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
dev = "cuda"
BAR = 2.5e-5     # test_gpu_exact_trunk_b24.py: the trunk's accumulation bar, of the output scale

BT = torch.tensor([[1, 0, -1, 0], [0, 1, 1, 0], [0, -1, 1, 0], [0, 1, 0, -1]], dtype=torch.float64)
AT = torch.tensor([[1, 1, 1, 0], [0, 1, -1, -1]], dtype=torch.float64)


def _ops():
    from rendernet_b200 import ops
    return ops


def _pair_f64(planes):
    return planes[0].double() + planes[1].double()


@pytest.mark.parametrize("B,H,W,C", [(1, 2, 2, 64), (2, 18, 34, 64), (3, 8, 8, 128)])
def test_input_transform_vs_float64(B, H, W, C):
    ops = _ops()
    from rendernet_b200._lib import check, lib
    g = torch.Generator().manual_seed(H * W + C)
    x = torch.randn(B, H, W, C, generator=g) * 5
    xs = ops.cast_to_16(x.to(dev), fmt=2)
    v = torch.empty(2, 16, B, H // 2, W // 2, C, device=dev, dtype=torch.float16)
    check(lib.rn_winograd_in(xs.planes.data_ptr(), v.data_ptr(), B, H, W, C, None), "rn_winograd_in")
    torch.cuda.synchronize()
    d = F.pad(_pair_f64(xs.planes.cpu()), (0, 0, 1, 1, 1, 1))               # the operand the kernel reads, SAME-padded
    d = d.unfold(1, 4, 2).unfold(2, 4, 2)                                   # [B, H/2, W/2, C, 4, 4]
    ref = torch.einsum("ai,nhwcij,bj->abnhwc", BT, d, BT).reshape(16, B, H // 2, W // 2, C)
    got = _pair_f64(v.cpu())
    s = float(ref.abs().max())
    assert float((got - ref).abs().max()) <= 2.0 ** -20 * s


@pytest.mark.parametrize("act,res", [("prelu", "pair"), (None, "f32"), (None, None)])
def test_output_transform_vs_float64(act, res):
    ops = _ops()
    from rendernet_b200._lib import check, lib
    B, H, W, C = 2, 18, 34, 64
    g = torch.Generator().manual_seed(7)
    m = torch.randn(16, B, H // 2, W // 2, C, generator=g) * 10
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
    check(lib.rn_winograd_out(md.data_ptr(), bd.data_ptr(), ad.data_ptr() if act else None, a,
                              rdev.data_ptr() if rdev is not None else None, rf32, out16.data_ptr(), out32.data_ptr(),
                              B, H, W, C, None), "rn_winograd_out")
    torch.cuda.synchronize()
    mm = m.double().reshape(4, 4, B, H // 2, W // 2, C)
    y = torch.einsum("ia,abnhwc,jb->nhiwjc", AT, mm, AT).reshape(B, H, W, C) + bias.double()
    if act == "prelu":
        y = torch.clamp(y, min=0) + alpha.double() * torch.clamp(y, max=0)
    if res == "pair":
        y = y + _pair_f64(rdev.cpu())
    elif res == "f32":
        y = y + r.double()
    s = float(y.abs().max())
    assert float((out32.cpu().double() - y).abs().max()) <= 2.0 ** -21 * s
    assert float((_pair_f64(out16.cpu()) - y).abs().max()) <= 2.0 ** -21 * s


def _trunk(C, seed, scale=3.0):
    g = torch.Generator().manual_seed(seed)
    x = (torch.rand(24, 64, 64, C, generator=g) * 2 - 1) * scale
    w = (torch.rand(3, 3, C, C, generator=g) * 2 - 1) * (6.0 / (9 * 2 * C)) ** 0.5
    b = torch.randn(C, generator=g) * 0.1
    al = torch.rand(C, generator=g) * 0.3
    res = torch.randn(24, 64, 64, C, generator=g)
    return x, w, b, al, res


def _ref(x, w, b, items, co):
    return F.conv2d(x[items].double().permute(0, 3, 1, 2), w[:, :, :, co].double().permute(3, 2, 0, 1), b[co].double(),
                    padding=1).permute(0, 2, 3, 1)


def test_winograd_conv_b24_prelu_residual_vs_float64():
    """The trunk's res-block layer shapes at B = 24: PReLU into the hi/lo pair, then no activation with the pair residual; both
    outputs (fp32 and the pair) against float64 at the direct kernel's bar."""
    ops = _ops()
    x, w, b, al, res = _trunk(1024, 11)
    L = ops.pack_conv("conv2d", w, b, al, device=dev, fmt=2)
    xs, rs = ops.cast_to_16(x.to(dev), fmt=2), ops.cast_to_16(res.to(dev), fmt=2)
    y16, y32 = ops.conv2d(xs, L, act="prelu", want16=True, want32=True)
    z16, z32 = ops.conv2d(xs, L, act=None, residual=rs, want16=True, want32=True)
    assert L.wino is not None                                          # the Winograd path ran
    items, co = [0, 23], slice(0, 64)
    pre = _ref(x, w, b, items, co)
    refs = (torch.clamp(pre, min=0) + al[co].double() * torch.clamp(pre, max=0), pre + res[items][..., co].double())
    for name, (o16, o32), ref in (("prelu", (y16, y32), refs[0]), ("residual", (z16, z32), refs[1])):
        s = float(ref.abs().max())
        e32 = float((o32[items][..., co].double().cpu() - ref).abs().max())
        e16 = float((_pair_f64(o16.planes[:, items][..., co].cpu()) - ref).abs().max())
        print(f"winograd 3x3 1024 B=24 {name}: fp32 out {e32 / s:.2e}, pair out {e16 / s:.2e} of scale")
        assert e32 <= BAR * s and e16 <= BAR * s


def test_winograd_conv_large_activations():
    """|x| ~ 1e4: V reaches 4 |x| (still inside fp16's range), the result stays finite and in the bar."""
    ops = _ops()
    x, w, b, _, _ = _trunk(1024, 12, scale=1.0e4)
    x = x[:2].contiguous()
    L = ops.pack_conv("conv2d", w, b, None, device=dev, fmt=2)
    y = ops.conv2d(ops.cast_to_16(x.to(dev), fmt=2), L, want16=False, want32=True)
    assert L.wino is not None and bool(torch.isfinite(y).all())
    items, co = [0, 1], slice(960, 1024)
    ref = _ref(x, w, b, items, co)
    s = float(ref.abs().max())
    err = float((y[items][..., co].double().cpu() - ref).abs().max())
    print(f"winograd |x|~1e4: {err / s:.2e} of scale")
    assert err <= BAR * s


def test_winograd_off_is_the_direct_kernel_bit_for_bit():
    ops = _ops()
    x, w, b, al, res = _trunk(1024, 13)
    x, res = x[:2].contiguous(), res[:2].contiguous()
    xs, rs = ops.cast_to_16(x.to(dev), fmt=2), ops.cast_to_16(res.to(dev), fmt=2)
    L = ops.pack_conv("conv2d", w, b, al, device=dev, fmt=2)
    Ld = ops.pack_conv("conv2d", w, b, al, device=dev, fmt=2, winograd=False)
    for act, r in (("prelu", None), (None, rs)):
        off = ops.conv2d(xs, L, act=act, residual=r, want16=True, want32=True, tune=dict(winograd=-1))
        direct = ops.conv2d(xs, Ld, act=act, residual=r, want16=True, want32=True)
        wino = ops.conv2d(xs, L, act=act, residual=r, want16=True, want32=True)
        assert torch.equal(off[0].planes, direct[0].planes) and torch.equal(off[1], direct[1])
        assert not torch.equal(wino[1], direct[1])                    # the default really is the other path
        assert Ld.wino is None


def test_changed_filter_is_repacked_not_run_with_a_stale_u():
    ops = _ops()
    x, w, b, _, _ = _trunk(1024, 14)
    x = x[:1].contiguous()
    wd = w.to(dev)
    xs = ops.cast_to_16(x.to(dev), fmt=2)
    L = ops.pack_conv("conv2d", wd, b, None, device=dev, fmt=2)
    y1 = ops.conv2d(xs, L, want16=False, want32=True)
    wd.mul_(-0.5)                                                      # an optimizer step on the master, in place
    with pytest.raises(RuntimeError, match="re-pack"):
        ops.conv2d(xs, L, want16=False, want32=True)
    L2 = ops.pack_conv("conv2d", wd, b, None, device=dev, fmt=2)
    y2 = ops.conv2d(xs, L2, want16=False, want32=True)
    co = slice(0, 64)
    ref = _ref(x, wd.cpu(), b, [0], co)
    s = float(ref.abs().max())
    assert float((y2[..., co].double().cpu() - ref).abs().max()) <= BAR * s
    assert not torch.allclose(y1, y2)
