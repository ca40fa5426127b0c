"""The training step at the reference's training batch, B = 24 (RenderNet_Shader.py's batch; 32^2 and 64^2 patches,
patch_size_for_epoch).  Every weight-gradient reduction of the step sums over the batch, so B is the dimension along which its
rounding error grows.  Checked here against float64 on the unrounded fp32 operands (torch on the device: cuDNN / cuBLAS, never
this project's kernels):

  * rn_conv_weight_grad_direct (the 32 x 32-tile kernel and the thin (8,1) / (16,3) kernels) at every layer that uses it, at
    whole-frame size, driven through ShaderInputGradients._weight_grads_of (operand roles, SAME pads, 1/scale, permutes);
  * the depth-folded 3^3 gradient (wgmma on [B,H,W,D*C] + block-diagonal sums) of res1 and e_conv3;
  * rn_bias_grad_16 and rn_prelu_alpha_grad at every Shader site;
  * a whole B = 24 step (ShaderTrainer, TextureTrainer) against the float64 mean of 24 single-item steps;
  * rn_dropout_16 at its largest site.

Operands come in two kinds: white noise, and coherent (x = |N(0,1)| with ~40 % exact zeros, g = (0.5 + N(0,1)) spread over
several binades, times a loss scale), whose sums grow linearly with the batch.  Metrics are those of test_gpu_backward_exact:
max |err| / max |ref|, and the signed bias mean((got - ref) sign(ref)) / mean |ref|."""
import types
import zlib

import numpy as np
import pytest
import torch

from oracle import rendernet_oracle as orc

from test_gpu_backward_exact import LS, _layer64

pytestmark = pytest.mark.gpu
dev = "cuda"
B = 24
KINDS = ("white", "coherent")


def _x(kind, shape, gen):
    """Activation-like operand: white N(0,1), or coherent |N(0,1)| with ~40 % exact zeros (post-PReLU)."""
    v = torch.randn(shape, device=dev, generator=gen)
    if kind == "white":
        return v
    return v.abs_() * (torch.rand(shape, device=dev, generator=gen) >= 0.4)


def _g(kind, shape, gen):
    """Gradient-like operand (unscaled): white N(0,1), or coherent (0.5 + N(0,1)) * exp(U(-6, 1)) -- a mean, several binades."""
    v = torch.randn(shape, device=dev, generator=gen)
    if kind == "white":
        return v
    return (v + 0.5) * torch.empty(shape, device=dev).uniform_(-6.0, 1.0, generator=gen).exp_()


def _metrics(got, ref):
    """(max |got - ref| / max |ref|, mean((got - ref) sign(ref)) / mean |ref|), float64."""
    d = got.double() - ref
    return float(d.abs().max() / ref.abs().max()), float((d * ref.sign()).mean() / ref.abs().mean())


def _pad16(g):
    """Zero-pad the channels of a gradient thinner than 16 (e_conv11: 3 of 16), as the walk's sigmoid backward does."""
    c = int(g.shape[-1])
    if c >= 8:                                          # e_conv1's 8-channel gradient is not padded
        return g
    out = torch.zeros(tuple(g.shape[:-1]) + (16,), device=g.device, dtype=g.dtype)
    out[..., :c] = g
    return out


def _drive(rec, g, fmt, tensor_core=False):
    """ShaderInputGradients._weight_grads_of on a fake walker: g (unscaled fp32) enters as 16-bit carrying the loss scale LS,
    1/LS is applied by the callee -> the filter gradient in TF layout."""
    from rendernet_b200 import ops
    from rendernet_b200.backward import ShaderInputGradients
    fake = types.SimpleNamespace(weight_grads={}, new_size=128)
    g16 = ops.cast_to_16((_pad16(g) * LS).contiguous(), fmt=fmt)
    ShaderInputGradients._weight_grads_of(fake, rec, g16, 1.0 / LS, tensor_core)
    return fake.weight_grads["w"]


def _wvar(wshape):
    w = torch.zeros(wshape, dtype=torch.float32)        # only the shape and the name are read by the weight-gradient path
    w._rn_name = "w"
    return w


def _ref(layer, x, wshape, g):
    """dL/dW = vjp of the float64 layer at the unrounded fp32 operands, on the device."""
    w = torch.zeros(wshape, dtype=torch.float64, device=dev, requires_grad=True)
    y = layer(x.double(), w)
    return torch.autograd.grad(y, w, g.double())[0]


# ------------------------------------------------------------------------------------------ 1. the direct correlation
# name, kind, stride, TF filter shape, input shape per item.  Whole-frame sizes; channel counts of RenderNet_Shader.py and
# RenderNet_Texture_Face_Normal.py (the Texture heads' e_conv10, 16 -> 3 at 512^2, has e_conv11's RGB shape).
DIRECT_CASES = [
    ("e_conv2", "conv3d", 2, (3, 3, 3, 8, 16), (64, 64, 64, 8)),
    ("e_conv7", "conv2d_transpose", 2, (4, 4, 128, 256), (64, 64, 256)),
    ("e_conv7_1", "conv2d_transpose", 1, (4, 4, 128, 128), (128, 128, 128)),
    ("e_conv8", "conv2d_transpose", 2, (4, 4, 64, 128), (128, 128, 128)),
    ("e_conv9", "conv2d_transpose", 2, (4, 4, 32, 64), (256, 256, 64)),
    ("e_conv10", "conv2d_transpose", 1, (4, 4, 16, 32), (512, 512, 32)),
    ("e_conv11_grey", "conv2d_transpose", 1, (4, 4, 1, 16), (512, 512, 16)),
    ("e_conv11_rgb", "conv2d_transpose", 1, (4, 4, 3, 16), (512, 512, 16)),         # thin (16,3)
    ("tex_e_conv7", "conv2d_transpose", 2, (4, 4, 64, 128), (64, 64, 128)),
    ("tex_e_conv8", "conv2d_transpose", 2, (4, 4, 32, 64), (128, 128, 64)),
    ("tex_e_conv9", "conv2d_transpose", 2, (4, 4, 16, 32), (256, 256, 32)),
]


def _out_shape(kind, stride, wshape, xshape):
    if kind == "conv3d":
        return xshape[:2] + (-(-xshape[2] // stride), wshape[-1])
    return (xshape[0] * stride, xshape[1] * stride, wshape[2])


def _check_pair(label, kind, run, ref, ref1=None, run1=None):
    """Exact and fast errors of one case, with the B = 1 exact error printed beside B = 24; asserts the exact and fast bars.
    The fast mode must be > 20x the exact error on white noise.  With coherent operands fp16's round-to-nearest errors stay
    independent while the sum grows with the batch, so the fast error relative to max |ref| falls like 1/sqrt(n) (measured
    2e-6 .. 3e-5 at B = 24) and cannot tell the formats apart by 20x;
    there it is held to the 1e-3 bar and to being above the exact error."""
    e, bias = _metrics(run(2), ref)
    f, fb = _metrics(run(0), ref)
    tail = ""
    if ref1 is not None:
        e1, b1 = _metrics(run1(2), ref1)
        tail = f" | B=1 exact max {e1:.2e} bias {b1:+.2e}"
    print(f"{label}: exact max {e:.2e} bias {bias:+.2e}; fast max {f:.2e} bias {fb:+.2e}{tail}")
    assert e <= 2e-5 and abs(bias) <= 1e-5, (label, e, bias)
    assert f <= 1e-3 and f > (20 * e if kind == "white" else e), (label, f, e)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("name,conv,stride,wshape,xshape", DIRECT_CASES, ids=[c[0] for c in DIRECT_CASES])
def test_direct_weight_gradient_b24_matches_float64(name, conv, stride, wshape, xshape, kind):
    """rn_conv_weight_grad_direct at B = 24 through _weight_grads_of: exact <= 2e-5 of scale with |bias| <= 1e-5 (the bars of
    the wgmma weight gradient), fast <= 1e-3 and > 20x the exact error."""
    from rendernet_b200 import ops
    gen = torch.Generator(device=dev).manual_seed(zlib.crc32(f"{name}/{kind}".encode()))
    x = _x(kind, (B,) + xshape, gen)
    g = _g(kind, (B,) + _out_shape(conv, stride, wshape, xshape), gen)

    def layer(xx, w):
        if conv == "conv3d":
            return orc.conv3d(xx, w, None, (1, 1, stride), dtype=torch.float64)
        return _layer64(conv, stride, xx, w)

    def runner(xx, gg):
        return lambda fmt: _drive(dict(op="conv", kind=conv, stride=stride, x=ops.cast_to_16(xx, fmt=fmt), w=_wvar(wshape), b=None),
                                  gg, fmt)

    ref = _ref(layer, x, wshape, g)
    ref1 = _ref(layer, x[:1], wshape, g[:1])
    _check_pair(f"{name} {wshape} {kind} B={B}", kind, runner(x, g), ref, ref1, runner(x[:1].contiguous(), g[:1].contiguous()))


@pytest.mark.parametrize("kind", KINDS)
def test_e_conv1_weight_gradient_b24_matches_float64(kind):
    """e_conv1 (thin (8,1) kernel, 125 taps, stride 2): the fused resample + conv record; the fine operand is the fp32
    resampled grid, re-made by the walk from a ResampledGrid.  White: voxels N(0,1); coherent: 10 % occupancy (bench config 2's
    density), g coherent."""
    from rendernet_b200 import ops
    from rendernet_b200.engine import pose_to_matrix
    from rendernet_b200.resampling_voxel_grid import ResampledGrid
    gen = torch.Generator(device=dev).manual_seed(11 if kind == "white" else 12)
    rng = np.random.default_rng(5)
    poses = np.stack([rng.uniform(0, 2 * np.pi, B), (90 - rng.uniform(10, 170, B)) * np.pi / 180,
                      3.3 / rng.uniform(2.5, 4.5, B)], axis=1).astype(np.float32)
    minv = torch.from_numpy(pose_to_matrix(poses, 64, 128)).to(dev)
    if kind == "white":
        vox = torch.randn((B, 64, 64, 64, 1), device=dev, generator=gen)
    else:
        vox = (torch.rand((B, 64, 64, 64, 1), device=dev, generator=gen) < 0.10).float()
    wshape = (5, 5, 5, 1, 8)
    g = _g(kind, (B, 64, 64, 64, 8), gen)
    q = ops.resample(vox, minv, 128, True)
    layer = lambda xx, w: orc.conv3d(xx, w, None, (2, 2, 2), dtype=torch.float64)          # noqa: E731

    def runner(n):
        grid = ResampledGrid(vox[:n].contiguous(), minv[:n].contiguous(), 128, transform=True)
        rec = dict(op="resample_conv1", grid=grid, window=None, stride=[2, 2, 2], w=_wvar(wshape), b=None)
        return lambda fmt: _drive(rec, g[:n].contiguous(), fmt)

    _check_pair(f"e_conv1 {wshape} {kind} B={B}", kind, runner(B), _ref(layer, q, wshape, g), _ref(layer, q[:1], wshape, g[:1]),
                runner(1))


# ------------------------------------------------------------------------------------------ 2. the depth-folded 3^3 gradient
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("name,wshape", [("res1", (3, 3, 3, 32, 32)), ("e_conv3", (3, 3, 3, 16, 32))])
def test_depth_folded_weight_gradient_b24_matches_float64(name, wshape, kind):
    """res1 (x 21 layers) and e_conv3 at B = 24, 64 x 64 x 32: the wgmma gradient of the depth-folded conv2d plus the
    torch.diagonal sums (_weight_grads_of with tensor_core=True), same bars as the direct kernel."""
    from rendernet_b200 import ops
    gen = torch.Generator(device=dev).manual_seed(zlib.crc32(f"{name}/{kind}".encode()))
    x = _x(kind, (B, 64, 64, 32, wshape[3]), gen)
    g = _g(kind, (B, 64, 64, 32, wshape[4]), gen)
    layer = lambda xx, w: orc.conv3d(xx, w, None, (1, 1, 1), dtype=torch.float64)          # noqa: E731

    def runner(xx, gg):
        return lambda fmt: _drive(dict(op="conv", kind="conv3d", stride=1, x=ops.cast_to_16(xx, fmt=fmt), w=_wvar(wshape), b=None),
                                  gg, fmt, tensor_core=True)

    _check_pair(f"{name} folded {wshape} {kind} B={B}", kind, runner(x, g), _ref(layer, x, wshape, g), _ref(layer, x[:1], wshape, g[:1]),
                runner(x[:1].contiguous(), g[:1].contiguous()))


# ------------------------------------------------------------------------------------------ 3. bias and slope sums
# channels, positions per item: e_conv1, e_conv2, e_conv3 / res1, trunk, e_conv5 / res3, e_conv6, e_conv7 / e_conv7_1, e_conv8,
# e_conv9, e_conv10 (and e_conv11's bias: 3 of its 16 channels used)
SUM_SITES = [(8, 64 ** 3), (16, 64 * 64 * 32), (32, 64 * 64 * 32), (1024, 64 * 64), (512, 64 * 64), (256, 64 * 64),
             (128, 128 * 128), (64, 256 * 256), (32, 512 * 512), (16, 512 * 512)]
# (sum, fmt, operand kind) -> bar: the largest error over the sites, measured on an H100 80GB HBM3, rounded up.  Exact mode on
# white noise is the exception: normalised by sum |terms|, an fp32 sum of random-sign terms in any order is off by a few units of
# u = 2^-24 whatever n is, and the order of the sums' atomics moves the error from run to run (slope: 3.6e-8, then 5.1e-8 =
# 0.85 u; bias <= 1.5e-8 = 0.25 u).  Its bar is 2 u, the rounding-error scale itself.
U = 2.0 ** -24
SUM_BARS = {("bias", 2, "white"): 2 * U, ("bias", 2, "coherent"): 2e-6, ("bias", 0, "white"): 4e-6, ("bias", 0, "coherent"): 1.2e-5,
            ("alpha", 2, "white"): 2 * U, ("alpha", 2, "coherent"): 3e-6, ("alpha", 0, "white"): 1e-5, ("alpha", 0, "coherent"): 3e-5}


@pytest.mark.parametrize("C,npos", SUM_SITES, ids=[f"C{c}" for c, _ in SUM_SITES])
def test_bias_and_slope_gradients_b24_match_float64(C, npos):
    """rn_bias_grad_16 (db = sum g) and rn_prelu_alpha_grad (dalpha = sum_{z<0} g z) over B = 24 items, both 16-bit formats,
    g carrying the loss scale and 1/scale applied as the walk applies it.  Errors are normalised by max |ref| for coherent g
    (whose sums grow with the batch) and per channel by sum |terms| for white noise.  Measured on an H100 80GB HBM3, largest
    over the sites: exact 1.6e-6 (bias) / 1.9e-6 (slope) coherent, 1.5e-8 / 5.1e-8 white; fast 9.2e-6 / 2.1e-5 coherent,
    2.9e-6 / 7.9e-6 white."""
    from rendernet_b200 import ops
    gen = torch.Generator(device=dev).manual_seed(C * 7 + 3)
    z = torch.randn((B * npos, C), device=dev, generator=gen)
    errs = {}
    for kind in KINDS:
        g = _g(kind, (B * npos, C), gen)
        g64, z64 = g.double(), z.double()
        t_a = g64 * z64 * (z64 < 0)
        refs = {"bias": (g64.sum(0), g64.abs().sum(0)), "alpha": (t_a.sum(0), t_a.abs().sum(0))}
        del g64, z64, t_a
        for fmt in (2, 0):
            g16 = ops.cast_to_16((g * LS).contiguous(), fmt=fmt)
            z16 = ops.cast_to_16(z, fmt=fmt)
            got = {"bias": ops.bias_grad(g16) * (1.0 / LS), "alpha": ops.prelu_alpha_grad(g16, z16, 1.0 / LS)}
            for what, (ref, l1) in refs.items():
                d = (got[what].double() - ref).abs()
                errs[(what, fmt, kind)] = float(d.max() / ref.abs().max()) if kind == "coherent" else float((d / l1).max())
            del g16, z16
        del g
    if C == 16:                      # e_conv11: the zero-padded channels 3..15 sum to exactly 0
        g = torch.zeros((B * npos, 16), device=dev)
        g[:, :3] = _g("coherent", (B * npos, 3), gen)
        for fmt in (2, 0):
            db = ops.bias_grad(ops.cast_to_16(g * LS, fmt=fmt))
            assert bool((db[3:] == 0).all())
    print(f"C={C} x {B}*{npos}: " + ", ".join(f"{w} fmt{f} {k} {e:.2e}" for (w, f, k), e in sorted(errs.items())))
    for (what, fmt, kind), e in errs.items():
        assert e <= SUM_BARS[(what, fmt, kind)], (what, fmt, kind, e)


# ------------------------------------------------------------------------------------------ 4. a B = 24 step vs 24 single steps
def _items():
    """24 distinct items: bench config 2's generator (10 % occupancy, random poses), seeded."""
    rng0, rng1 = np.random.default_rng(0), np.random.default_rng(1)
    vox = (rng0.random((B, 64, 64, 64, 1)) < 0.10).astype(np.float32)
    poses = np.stack([rng1.uniform(0, 2 * np.pi, B), (90 - rng1.uniform(10, 170, B)) * np.pi / 180,
                      3.3 / rng1.uniform(2.5, 4.5, B)], axis=1).astype(np.float32)
    return vox, poses


def _batch_vs_items(make, inputs, P):
    """loss and gradients of one B = 24 trainer vs the float64 mean over 24 B = 1 trainers' (one fixed origin) -> (loss24,
    mean of the single losses, {name: (error, error with one item left out of the mean)}, peak memory in GiB)."""
    origin = (64 - P // 2, 64 - P // 2) if P < 128 else None
    torch.cuda.reset_peak_memory_stats()
    tr = make(B)
    loss24, g24 = tr.loss_and_gradients(*inputs, patch_size=P, origin=origin)
    g24 = {n: t.clone() for n, t in g24.items()}
    del tr
    tr1 = make(1)
    acc, last, losses = None, None, []
    for i in range(B):
        loss, g = tr1.loss_and_gradients(*(a[i:i + 1] for a in inputs), patch_size=P, origin=origin)
        losses.append(loss)
        if acc is None:
            acc = {n: t.double() for n, t in g.items()}
        else:
            for n, t in g.items():
                acc[n] += t.double()
        if i == B - 1:
            last = {n: t.double() for n, t in g.items()}
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    errs = {}
    for n, s in acc.items():
        ref, drop = s / B, (s - last[n]) / (B - 1)
        scale = float(ref.abs().max())
        errs[n] = (float((g24[n].double() - ref).abs().max()) / scale, float((drop - ref).abs().max()) / scale)
    return loss24, float(np.mean(losses)), errs, peak


# fast precision: the largest per-variable error measured on an H100 80GB HBM3 (2.4e-3, the texture decoder's FC), rounded up
STEP_FAST_BAR = 3e-3
STEP_EXACT_BAR = 3e-5


def _report_step(label, loss24, loss1, errs, peak, precision, nvars):
    worst = max(errs.items(), key=lambda kv: kv[1][0])
    least_drop = min(errs.items(), key=lambda kv: kv[1][1])
    print(f"{label}: loss {loss24:.8f} vs mean of singles {loss1:.8f}; {len(errs)} variables, worst {worst[0]} "
          f"{worst[1][0]:.2e}; one item dropped: least {least_drop[0]} {least_drop[1][1]:.2e}; peak memory {peak:.2f} GiB")
    assert len(errs) == nvars
    assert abs(loss24 - loss1) <= 1e-6 * abs(loss1)
    bar = STEP_EXACT_BAR if precision == "exact" else STEP_FAST_BAR
    assert worst[1][0] <= bar, (worst, bar)
    if precision == "exact":
        assert least_drop[1][1] >= 10 * STEP_EXACT_BAR, least_drop


@pytest.mark.parametrize("P", [64, 32])
@pytest.mark.parametrize("precision", ["exact", "fast"])
@pytest.mark.parametrize("greyscale", [False, True], ids=["rgb_mse", "grey_bce"])
def test_shader_b24_step_equals_mean_of_single_item_steps(greyscale, precision, P):
    """ShaderTrainer.loss_and_gradients, keep_prob 1.0, one patch origin: the loss is a mean over items, so at B = 24 the loss
    and all 166 gradients equal the mean over 24 B = 1 steps (summed in float64).  Forward and data-gradient kernels do not
    depend on B; the 16-bit rounding of g (another loss scale) and the weight-gradient reductions do.  Exact: every variable
    within 3e-5 of its scale; leaving one item out of the mean must miss by >= 10x that.  Measured on an H100 80GB HBM3:
    exact <= 1.1e-5, fast <= 2.1e-3, one item left out >= 3.2e-3; peak memory 12.7 GiB at P = 64."""
    from rendernet_b200.training import ShaderTrainer
    vox, poses = _items()
    rng = np.random.default_rng(7)
    if greyscale:
        target = (rng.random((B, 512, 512, 1)) < 0.5).astype(np.float32)
    else:
        target = rng.random((B, 512, 512, 3)).astype(np.float32)
    W = orc.init_shader_weights(seed=4, is_greyscale=greyscale, alpha_range=(-0.05, 0.25), bias_jitter=0.02)

    def make(n):
        return ShaderTrainer(W, n, precision=precision, is_greyscale=greyscale, keep_prob=1.0)

    res = _batch_vs_items(make, (vox, poses, target), P)
    _report_step(f"[shader {'grey BCE' if greyscale else 'RGB MSE'} {precision} P={P}]", *res, precision, 166)


@pytest.mark.parametrize("P", [64, 32])
@pytest.mark.parametrize("precision", ["exact", "fast"])
def test_texture_b24_step_equals_mean_of_single_item_steps(precision, P):
    """TextureTrainer (two MSEs, all 186 variables, texture decoder included), as the Shader case.  Measured on an H100 80GB
    HBM3: exact <= 1.8e-5, fast <= 2.4e-3, one item left out >= 4.6e-4 (exact); peak memory 6.9 GiB at P = 64."""
    from rendernet_b200.training import TextureTrainer
    vox, poses = _items()
    tex = np.random.default_rng(2).standard_normal((B, 199)).astype(np.float32)
    rng = np.random.default_rng(8)
    img_t = rng.random((B, 512, 512, 3)).astype(np.float32)
    nrm_t = rng.random((B, 512, 512, 3)).astype(np.float32)
    W = orc.init_texture_weights(seed=4, alpha_range=(-0.05, 0.25), bias_jitter=0.02)

    def make(n):
        return TextureTrainer(W, n, precision=precision, keep_prob=1.0)

    res = _batch_vs_items(make, (vox, tex, poses, img_t, nrm_t), P)
    _report_step(f"[texture {precision} P={P}]", *res, precision, 186)


# ------------------------------------------------------------------------------------------ 5. dropout at its largest site
@pytest.mark.parametrize("fmt", [2, 0])
def test_dropout_at_e_conv9_output_b24(fmt):
    """rn_dropout_16 on e_conv9's output at B = 24 (24 * 512^2 * 32 = 201 M elements, past 2^27): the kept set equals
    rn_dropout_mask_host's, and the kept values are x / keep to the format's rounding: 2^-21 (fmt 2) or 2^-11 (fmt 0) of the
    value, plus 2^-25 where the fp16 LO half of a small value is subnormal."""
    from rendernet_b200 import ops, tfcompat as tf
    n_shape = (B, 512, 512, 32)
    gen = torch.Generator(device=dev).manual_seed(21)
    x = torch.randn(n_shape, device=dev, generator=gen)
    x[x.abs() < 1e-3] = 1.0                               # no input that rounds to 0 in fp16: kept <=> nonzero output
    keep, seed, salt = 0.75, 0x5EED, 9
    x16 = ops.cast_to_16(x, fmt=fmt)
    y = tf.to_float(ops.dropout(x16, keep, seed=seed, salt=salt))
    xq = tf.to_float(x16)
    del x16
    mask = torch.from_numpy(ops.dropout_mask_host(x.numel(), keep, seed, salt)).to(dev).reshape(n_shape).bool()
    same = bool(torch.equal(y != 0, mask))
    want = xq.double() / keep
    rel = 2.0 ** -21 if fmt == 2 else 2.0 ** -11
    worst = float(((y.double() - want).abs() / (want.abs() * rel + 2.0 ** -25))[mask].max())
    frac = float(mask.float().mean())
    print(f"dropout fmt {fmt}, {x.numel()} elements: kept fraction {frac:.5f}, kept set equal {same}, kept values at {worst:.2f} of the bound")
    assert same
    assert worst <= 1.0
    assert abs(frac - keep) < 1e-3
