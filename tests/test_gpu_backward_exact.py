"""The backward pass at the precision it claims: every data-gradient path of ShaderInputGradients._data_grad_of, the element-wise
backward kernels and the wgmma weight gradient, each against a float64 computation on the UNROUNDED fp32 inputs (not against
the fp32 oracle, whose own rounding would hide an error of the exact mode's size).

Bars (exact mode = fp16 hi/lo operand pairs, fp32-equivalent): 2e-5 of the gradient scale per layer, 2.5e-5 for the K = 9216
trunk convolution -- the forward pass's bars (tests/test_gpu_exact.py).  The fast mode (fp16 operands) is asserted at its
measured bound and more than 20x above the exact error, which shows each case can tell the two precisions apart; two LO-plane
ablations check that the exact bar would catch an operand silently reduced to fp16.
References of the >= 512-channel shapes are float64 torch convolutions on the GPU (cuDNN / cuBLAS, not this project's
kernels), the rest run on the CPU.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import rendernet_oracle as orc

pytestmark = pytest.mark.gpu
dev = "cuda"
LS = 64.0              # loss scale of the seeded gradients: keeps some LO halves in fp16's subnormal range


def _wide(rng, shape, scale=1.0):
    """fp32 values spanning several binades (incl. magnitudes whose LO half lands in fp16's subnormal range)."""
    return (rng.standard_normal(shape) * np.exp(rng.uniform(-6.0, 1.0, shape)) * scale).astype(np.float32)


def _layer64(kind, stride, x, w):
    """The forward convolution in float64 (TF SAME rules of oracle/rendernet_oracle.py), channel-last; w in TF layout."""
    if kind == "conv2d":
        k = w.shape[0]
        pb = (k - 1) // 2
        y = F.conv2d(F.pad(x.permute(0, 3, 1, 2), (pb, k - 1 - pb, pb, k - 1 - pb)), w.permute(3, 2, 0, 1))
        return y.permute(0, 2, 3, 1)
    if kind == "conv3d":
        st = (1, 1, stride)
        pads = []
        for d in (2, 1, 0):
            pads += list(orc.same_pads(x.shape[1 + d], w.shape[d], st[d]))
        y = F.conv3d(F.pad(x.permute(0, 4, 1, 2, 3), pads), w.permute(4, 3, 0, 1, 2), stride=st)
        return y.permute(0, 2, 3, 4, 1)
    H, W, k = x.shape[1], x.shape[2], w.shape[0]
    full = F.conv_transpose2d(x.permute(0, 3, 1, 2), w.permute(3, 2, 0, 1), stride=stride)
    p = max(k - stride, 0) // 2
    return full[:, :, p:p + H * stride, p:p + W * stride].permute(0, 2, 3, 1)


def _dgrad64(kind, stride, xshape, w, g):
    """dL/dx = vjp of the float64 layer with cotangent g (fp32 values, unrounded); computed where `g` lives."""
    on = g.device
    x = torch.zeros(xshape, dtype=torch.float64, device=on, requires_grad=True)
    y = _layer64(kind, stride, x, torch.from_numpy(w).to(on, torch.float64))
    return torch.autograd.grad(y, x, g.double())[0]


def _err(got, ref):
    """(max |got - ref| / max |ref|, rel-rms) in float64."""
    d = got.double().to(ref.device) - ref
    return float(d.abs().max() / ref.abs().max()), float(d.pow(2).mean().sqrt() / ref.pow(2).mean().sqrt())


def _record(precision, kind, x, w, stride):
    """Forward of one layer through layer_util's deferred convolution with a tape -> (ShaderInputGradients, tape record)."""
    from rendernet_b200 import layer_util as lu, ops, tfcompat as tf
    from rendernet_b200.backward import ShaderInputGradients
    ig = ShaderInputGradients(None, 1, precision=precision)
    tape = []
    ig.store.tape = tape
    with tf.use_store(ig.store):
        xs = ops.cast_to_16(torch.from_numpy(x).to(dev), fmt=ig.store.fmt)
        with tf.variable_scope("t"):
            wv = tf.get_variable("weights", initializer=w)
        lu._deferred_conv(kind, xs, wv, None, stride).realize()
    ig.store.tape = None
    return ig, tape[-1]


# name, kind, stride, TF filter shape, input shape.  Real channel counts of the Shader network; spatial sizes reduced where the
# dispatch and the kernel plan do not depend on them, 64x64 kept for the >= 512-channel layers; 20 / 12 / 36 are ragged tiles.
DGRAD_CASES = [
    ("res1", "conv3d", 1, (3, 3, 3, 32, 32), (1, 12, 20, 32, 32)),                  # banded
    ("e_conv3", "conv3d", 1, (3, 3, 3, 16, 32), (1, 16, 12, 32, 16)),               # banded, 32 -> 16 gradient
    ("e_conv2", "conv3d", 2, (3, 3, 3, 8, 16), (1, 12, 16, 64, 8)),                 # conv3d_backward_data_direct, 16-bit out
    ("projection", "conv2d", 1, (1, 1, 1024, 1024), (1, 64, 64, 1024)),
    ("res2", "conv2d", 1, (3, 3, 1024, 1024), (1, 64, 64, 1024)),                   # K = 9216
    ("res3", "conv2d", 1, (3, 3, 512, 512), (1, 64, 64, 512)),
    ("e_conv5", "conv2d", 1, (4, 4, 1024, 512), (1, 64, 64, 1024)),                 # conv2d_taps, 48 pseudo-taps, ny = 4
    ("e_conv6", "conv2d", 1, (4, 4, 512, 256), (1, 64, 64, 512)),
    ("e_conv7", "conv2d_transpose", 2, (4, 4, 128, 256), (1, 16, 16, 256)),         # space-to-depth + 3x3
    ("e_conv8", "conv2d_transpose", 2, (4, 4, 64, 128), (1, 20, 24, 128)),
    ("e_conv9", "conv2d_transpose", 2, (4, 4, 32, 64), (1, 24, 20, 64)),
    ("e_conv7_1", "conv2d_transpose", 1, (4, 4, 128, 128), (1, 20, 24, 128)),       # forward SAME conv with the same filter
    ("e_conv10", "conv2d_transpose", 1, (4, 4, 16, 32), (1, 36, 40, 32)),
    ("e_conv11", "conv2d_transpose", 1, (4, 4, 3, 16), (1, 40, 36, 16)),            # gradient zero-padded 3 -> 16 channels
]


def _case_data(name, kind, wshape, xshape, stride):
    rng = np.random.default_rng(sum(map(ord, name)))
    fan = int(np.prod(wshape[:-2])) * (wshape[-1] if kind == "conv2d_transpose" else wshape[-2])
    w = (rng.uniform(-1, 1, wshape) * np.sqrt(3.0 / fan)).astype(np.float32)
    x = rng.standard_normal(xshape).astype(np.float32)
    big = max(wshape[-1], wshape[-2]) >= 512
    on = dev if big else "cpu"
    if kind == "conv2d_transpose":
        yshape = (xshape[0], xshape[1] * stride, xshape[2] * stride, wshape[2])
    elif kind == "conv3d":
        yshape = xshape[:3] + (-(-xshape[3] // stride), wshape[-1])
    else:
        yshape = xshape[:-1] + (wshape[-1],)
    g = torch.from_numpy(_wide(rng, yshape, LS)).to(on)
    acc = torch.from_numpy(_wide(rng, xshape, LS)).to(on)
    return w, x, g, acc


def _device_grad(ig, rec, g, acc, c_pad=16):
    """gx from _data_grad_of with g (and acc) cast to the store's 16-bit format; g zero padded to 16 channels when thinner."""
    from rendernet_b200 import ops, tfcompat as tf
    fmt = ig.store.fmt
    gd = g.to(dev).float()
    if gd.shape[-1] % 16:
        gp = torch.zeros(tuple(gd.shape[:-1]) + (c_pad,), device=dev)
        gp[..., :gd.shape[-1]] = gd
        gd = gp
    g16 = ops.cast_to_16(gd.contiguous(), fmt=fmt)
    a16 = None if acc is None else ops.cast_to_16(acc.to(dev).float().contiguous(), fmt=fmt)
    return g16, lambda gg: tf.to_float(ig._data_grad_of(rec, gg, a16))


@pytest.mark.parametrize("name,kind,stride,wshape,xshape", DGRAD_CASES, ids=[c[0] for c in DGRAD_CASES])
def test_layer_data_gradient_matches_float64(name, kind, stride, wshape, xshape):
    """ShaderInputGradients._data_grad_of (the dispatch backward() runs) for one recorded layer of each path, without and with a
    gradient already collected for x (`residual=acc`, the fused fan-out sum), vs float64 autograd of the same layer."""
    w, x, g, acc = _case_data(name, kind, wshape, xshape, stride)
    ref = _dgrad64(kind, stride, xshape, w, g)
    bar = 2.5e-5 if name == "res2" else 2e-5
    for with_acc in (False, True):
        want = ref + acc.double() if with_acc else ref
        errs = {}
        for precision in ("exact", "fast"):
            ig, rec = _record(precision, kind, x, w, stride)
            g16, run = _device_grad(ig, rec, g, acc if with_acc else None)
            errs[precision] = _err(run(g16), want)
        (e, r), (f, fr) = errs["exact"], errs["fast"]
        print(f"{name} {wshape} acc={with_acc}: exact max {e:.2e} rms {r:.2e}; fast max {f:.2e} rms {fr:.2e}")
        assert e <= bar, (name, with_acc, e)
        assert f <= 1e-3 and f > 20 * e, (name, with_acc, f, e)


@pytest.mark.parametrize("name", ["res3", "res1"])
def test_exact_bar_catches_a_missing_lo_plane(name):
    """Rerun of an odd conv2d and a banded case with the LO plane of g, then of the packed gradient filter, zeroed: each
    reduces one operand to fp16 precision, and each must break the exact bar by >= 5x (else the bar is too loose)."""
    _, kind, stride, wshape, xshape = next(c for c in DGRAD_CASES if c[0] == name)
    w, x, g, _ = _case_data(name, kind, wshape, xshape, stride)
    ref = _dgrad64(kind, stride, xshape, w, g)
    ig, rec = _record("exact", kind, x, w, stride)
    g16, run = _device_grad(ig, rec, g, None)
    e_ok = _err(run(g16), ref)[0]
    g_hi = type(g16)(g16.planes.clone())
    g_hi.planes[1].zero_()
    e_g = _err(run(g_hi), ref)[0]
    L = ig._dgrad_layer(rec)
    keep = L.w.clone()
    L.w[1].zero_()
    e_w = _err(run(g16), ref)[0]
    L.w.copy_(keep)
    print(f"{name}: exact {e_ok:.2e}, LO of g zeroed {e_g:.2e}, LO of the gradient filter zeroed {e_w:.2e}")
    assert e_ok <= 2e-5
    assert e_g >= 5 * 2e-5 and e_w >= 5 * 2e-5, (e_g, e_w)


# ----------------------------------------------------------------------------------------- element-wise backward kernels
def _close(got, want, rel, absb):
    got, want = got.double().cpu(), want.double().cpu()
    q = (got - want).abs() / (want.abs() * rel + absb)
    return int((q > 1).sum()), float(q.max())


@pytest.mark.parametrize("C", [24, 5, 3])
def test_prelu_backward_matches_float64(C):
    """rn_prelu_backward_16, fmt 2 and 0: y exactly 0 takes the slope branch; a pre-activation passed with negative slopes (what
    backward() passes once a slope is negative) selects by its own sign; channel counts that are not multiples of 16."""
    from rendernet_b200 import ops
    rng = np.random.default_rng(C)
    shape = (3, 7, 11, C)
    g = _wide(rng, shape, LS)
    z = rng.standard_normal(shape).astype(np.float32)                     # no value that fp16 rounds to zero ...
    z.reshape(-1, C)[::5] = 0.0                                           # ... except these exact zeros
    alpha = rng.uniform(-0.3, 0.3, C).astype(np.float32)
    alpha[0] = -0.2
    want = torch.from_numpy(np.where(z > 0, g.astype(np.float64), g.astype(np.float64) * alpha.astype(np.float64)))
    for fmt, rel, absb in ((2, 2.0 ** -20, 2.0 ** -23), (0, 2.0 ** -10, 2.0 ** -23)):     # two hi/lo roundings of 2^-22
        g16 = ops.cast_to_16(torch.from_numpy(g).to(dev), fmt=fmt)
        z16 = ops.cast_to_16(torch.from_numpy(z).to(dev), fmt=fmt)
        got = ops.prelu_backward(g16, z16, torch.from_numpy(alpha).to(dev)).float()
        nbad, worst = _close(got, want, rel, absb)
        print(f"prelu_backward C={C} fmt={fmt}: {nbad} elements off, worst {worst:.2f} of the bound")
        assert nbad == 0, (fmt, worst)


@pytest.mark.parametrize("C", [3, 1])
def test_sigmoid_backward_matches_float64(C):
    """rn_sigmoid_backward: scale * g * s * (1 - s), channels C padded to 16 with exact zeros in both planes; fmt 2 holds
    2^-21 of each value, fmt 0 its fp16 rounding."""
    from rendernet_b200 import ops
    rng = np.random.default_rng(10 + C)
    shape = (2, 9, 13, C)
    g = rng.standard_normal(shape).astype(np.float32) * np.float32(1e-3)
    s = rng.uniform(0.0, 1.0, shape).astype(np.float32)
    s.reshape(-1)[:4] = [0.0, 1.0, 0.5, 1e-6]
    scale = 4096.0
    want = scale * g.astype(np.float64) * s.astype(np.float64) * (1.0 - s.astype(np.float64))
    for fmt, rel in ((2, 2.0 ** -21), (0, 2.0 ** -10)):
        out = ops.sigmoid_backward(torch.from_numpy(g).to(dev), torch.from_numpy(s).to(dev), 16, scale, fmt)
        assert tuple(out.shape) == shape[:-1] + (16,)
        planes = out.planes if fmt == 2 else out[None]
        assert bool((planes[..., C:] == 0).all()) and not bool(torch.signbit(planes[..., C:].float()).any())
        nbad, worst = _close(out.float()[..., :C], torch.from_numpy(want), rel, 2.0 ** -24)
        print(f"sigmoid_backward C={C} fmt={fmt}: {nbad} elements off, worst {worst:.2f} of the bound")
        assert nbad == 0, (fmt, worst)


def test_bias_act_adds_split16_gradients_at_a_fan_out():
    """bias_act(g, residual=acc) on fp16 hi/lo pairs (the gradient sum where a forward tensor has two consumers): g + acc to
    2^-21 of |g| + |acc| (three hi/lo roundings of <= 2^-22 each), i.e. neither LO plane dropped."""
    from rendernet_b200 import ops
    rng = np.random.default_rng(11)
    shape = (2, 10, 12, 48)
    a, b = _wide(rng, shape, LS), _wide(rng, shape, LS)
    want = a.astype(np.float64) + b.astype(np.float64)
    got = ops.bias_act(ops.cast_to_16(torch.from_numpy(a).to(dev), fmt=2), None, None, None,
                       residual=ops.cast_to_16(torch.from_numpy(b).to(dev), fmt=2))
    assert isinstance(got, ops.Split16)
    d = (got.float().double().cpu().numpy() - want)
    bound = (np.abs(a).astype(np.float64) + np.abs(b)) * 2.0 ** -21 + 2.0 ** -23
    print(f"fan-out add: worst {float((np.abs(d) / bound).max()):.2f} of the 2^-21 bound")
    assert bool((np.abs(d) <= bound).all())


@pytest.mark.parametrize("cin,cout,k,stride,xshape", [(8, 16, 3, (1, 1, 2), (1, 12, 16, 64, 8)),
                                                      (5, 8, 5, (2, 2, 2), (1, 20, 16, 24, 5))])
def test_thin_conv3d_data_gradient_16bit_output_matches_float64(cin, cout, k, stride, xshape):
    """rn_conv3d_backward_data_direct: the fp16 hi/lo (fmt 2) output and the fp32 output hold 2e-5 of the gradient scale vs
    float64; fp16 (fmt 0) is > 20x above."""
    from rendernet_b200 import ops, tfcompat as tf
    rng = np.random.default_rng(cin * 10 + k)
    w = (rng.uniform(-1, 1, (k, k, k, cin, cout)) * np.sqrt(3.0 / (k ** 3 * cin))).astype(np.float32)
    xt = torch.zeros(xshape, dtype=torch.float64, requires_grad=True)
    pads = []
    for d in (2, 1, 0):
        pads += list(orc.same_pads(xshape[1 + d], k, stride[d]))
    y64 = F.conv3d(F.pad(xt.permute(0, 4, 1, 2, 3), pads), torch.from_numpy(w).double().permute(4, 3, 0, 1, 2),
                   stride=stride).permute(0, 2, 3, 4, 1)
    gy = torch.from_numpy(_wide(rng, tuple(y64.shape), LS))
    ref = torch.autograd.grad(y64, xt, gy.double())[0]
    res = {}
    for fmt in (2, 0):
        g16 = ops.cast_to_16(gy.to(dev), fmt=fmt)
        wd = torch.from_numpy(w).to(dev)
        out16 = tf.to_float(ops.conv3d_backward_data_direct(g16, wd, xshape, stride))
        out32 = ops.conv3d_backward_data_direct(g16, wd, xshape, stride, want32=True)
        res[fmt] = (_err(out16, ref)[0], _err(out32, ref)[0])
    print(f"thin conv3d dgrad {cin}->{cout} k{k} s{stride}: exact 16-bit {res[2][0]:.2e} fp32 {res[2][1]:.2e}; "
          f"fast {res[0][0]:.2e} / {res[0][1]:.2e}")
    assert res[2][0] <= 2e-5 and res[2][1] <= 2e-5
    assert res[0][1] > 20 * res[2][1]


# ----------------------------------------------------------------------------------------- weight gradients (rn_wgrad.cu)
def _wgrad64(x, g, kh, kw):
    """dW[ky,kx,ci,co] = sum_p x[p + (kx - pbx, ky - pby)][ci] g[p][co] in float64 on x's device (one matmul per tap)."""
    B, H, W, Ci = x.shape
    Co = g.shape[-1]
    pby, pbx = (kh - 1) // 2, (kw - 1) // 2
    xp = F.pad(x, (0, 0, pbx, kw - 1 - pbx, pby, kh - 1 - pby))
    g2 = g.reshape(-1, Co)
    return torch.stack([xp[:, ky:ky + H, kx:kx + W, :].reshape(-1, Ci).T @ g2 for ky in range(kh) for kx in range(kw)]
                       ).reshape(kh, kw, Ci, Co)


def _wgrad_errors(k, cin, cout, hw, B, seed):
    from rendernet_b200 import ops
    gen = torch.Generator(device=dev).manual_seed(seed)
    H, W = hw
    x = torch.randn((B, H, W, cin), device=dev, generator=gen)
    g = torch.randn((B, H, W, cout), device=dev, generator=gen)
    ref = _wgrad64(x.double(), g.double(), k, k)
    s, mabs = float(ref.abs().max()), float(ref.abs().mean())
    out = {}
    for name, fmt in (("exact", 2), ("fast", 0)):
        d = ops.conv2d_weight_grad(ops.cast_to_16(x, fmt=fmt), ops.cast_to_16(g, fmt=fmt), k, k).double() - ref
        out[name] = (float(d.abs().max()) / s, float((d * ref.sign()).mean()) / mabs)
    del x, g, ref
    torch.cuda.empty_cache()
    return out


@pytest.mark.parametrize("k,cin,cout,hw,B", [(3, 1024, 1024, (64, 64), 1), (3, 1024, 1024, (64, 64), 8),
                                             (3, 1024, 1024, (64, 64), 24),       # trunk: 288 tiles, one CTA per tile
                                             (1, 1024, 1024, (64, 64), 24),       # projection unit
                                             (4, 1024, 512, (64, 64), 1),         # e_conv5
                                             (3, 512, 512, (64, 64), 1),          # res3
                                             (4, 512, 256, (64, 64), 1),          # e_conv6
                                             (3, 128, 256, (6, 32), 2),           # W < 64: pixel blocks of 32 x 2
                                             (3, 256, 128, (8, 16), 3),           # 16 x 4
                                             (4, 128, 128, (16, 8), 2)])          # 8 x 8
def test_weight_gradient_matches_float64_at_production_shapes(k, cin, cout, hw, B):
    """rn_conv2d_weight_grad vs float64: max error over the gradient scale, and the mean signed relative error
    mean((got - ref) sign(ref)) / mean|ref|, which exposes accumulator truncation as a bias toward zero.  Measured on an H100:
    exact max <= 6.3e-6, bias -4.2e-6 at every shape and batch (one uncapped chain over B = 24 gave 1.3e-4 / -9.9e-5); fast
    max <= 3.3e-4."""
    out = _wgrad_errors(k, cin, cout, hw, B, seed=k * 7919 + cin + B)
    (e, bias), (f, fb) = out["exact"], out["fast"]
    print(f"wgrad k{k} {cin}->{cout} @{hw} B={B}: exact max {e:.2e} bias {bias:+.2e}; fast max {f:.2e} bias {fb:+.2e}")
    assert e <= 2e-5 and abs(bias) <= 1e-5, (e, bias)
    assert f <= 1e-3 and f > 20 * e, (f, e)


@pytest.mark.parametrize("H,W", [(6, 16), (7, 32), (10, 48)])
def test_weight_gradient_rejects_a_height_the_pixel_block_does_not_tile(H, W):
    """W < 64 folds PY = 64 / W rows into a pixel block; H % PY != 0 (or W not a power-of-two divisor of 64 pixels) is an
    error, not a silently truncated sum."""
    from rendernet_b200 import ops
    from rendernet_b200._lib import RenderNetCudaError
    x = ops.cast_to_16(torch.ones((1, H, W, 128), device=dev), fmt=2)
    g = ops.cast_to_16(torch.ones((1, H, W, 128), device=dev), fmt=2)
    with pytest.raises(RenderNetCudaError):
        ops.conv2d_weight_grad(x, g, 3, 3)
