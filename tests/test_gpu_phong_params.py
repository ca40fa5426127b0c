"""GPU tests of the shading-parameter gradients: the three *_params backward entries (rn_phong_shade_backward_params,
rn_phong_composite_loss_grad_params, rn_phong_recon_loss_grad_params), their fixed-order twins, rn_phong_shade_ambient,
nn.phong_shade with a fitted colour and ambient term, the fits with fit_shading, and RenderEngine's per-step light.

Inputs: test_gpu_phong_edges.py's catalogue of singular pixels (n = (0.5, 0.5, 0.5), n = 0 and 1, one-ulp neighbours of 0.5,
d = 0 and 1, composites at 0 and 1, saturated masks, the mask's transition band, col up to 1.2) at 512 x 512, its four items
repeated to B = 5 and B = 24 with a different ambient term per item; pixels within 1e-6 of a kink get no upstream gradient, as
there.

The bar for d_light_col and d_ambient.  Each is a sum of 512^2 per-pixel fp32 terms: a 5-level warp butterfly, 8 warp partials
added in order, then one atomic per 256-pixel block (1024 of them, in any order).  Every term passes through at most
1024 + 8 + 5 = 1037 fp32 additions, and recursive summation errs by at most (n - 1) u sum |x_i| (u = 2^-24), so
|error| <= (nblk + 13) u sum |term|.  Each term also carries a few roundings of its own and the fp32 forward's m and
k_d max(d, 0) against float64's; 32 u covers them.  The bar is (nblk + 45) u sum|term| = 6.4e-5 sum|term| at 512^2, with
sum|term| the float64 sum of the terms' magnitudes.  A missing mask factor, a clip in the wrong place or a dropped block misses it
by orders of magnitude; the measured errors are printed."""
import gc
import math

import numpy as np
import pytest
import torch

from phong_params_ref import np_vjp64, tf_vjp64
from test_gpu_phong_edges import _catalogue, _excluded

pytestmark = pytest.mark.gpu
dev = "cuda"
U = 2.0 ** -24
H = W = 512
NBLK = H * W // 256
BAR = (NBLK + 45) * U


def _d(a):
    return torch.from_numpy(np.array(a, copy=True, order="C")).to(dev)


@pytest.fixture(autouse=True)
def _release_device_memory():
    """The engines and fit objects built here hold CUDA graphs and recorded activations, some of them in reference cycles.
    Collect them and hand the cached blocks back to the driver after each test, so that the tests after this module, and the
    child processes some of them start, find the device as free as they would without it."""
    yield
    gc.collect()
    torch.cuda.empty_cache()


def _inputs(B, composite, white, kd=0.9):
    n4, ld4, col4, half4, near4 = _catalogue(H, W, composite, white)
    idx = np.arange(B) % 4
    amb = np.linspace(0.0, 0.35, B).astype(np.float32)
    return n4[idx], ld4[idx], col4[idx], amb, near4[idx]


def _vjp(composite, white, mask, n, ld, col, amb, kd, g, alb):
    if composite == "tf":
        return tf_vjp64(n, ld, col, amb, kd, not white, mask, g, alb)
    return np_vjp64(n, ld, col, amb, kd, white, mask, g, alb)


def _param_err(d_col, d_amb, ref, ref_abs):
    """max over items of |error| / sum|term| for the colour (per component) and the ambient term."""
    e_col = np.abs(d_col.double().cpu().numpy() - ref[4]) / np.maximum(ref_abs[4], 1e-300)
    e_amb = np.abs(d_amb.double().cpu().numpy() - ref[5]) / np.maximum(ref_abs[5], 1e-300)
    assert np.isfinite(d_col.cpu().numpy()).all() and np.isfinite(d_amb.cpu().numpy()).all()
    return float(e_col.max()), float(e_amb.max())


def _configs(B):
    """Backgrounds x mask at B = 5; the white background with the mask alone at B = 24 (the float64 reference is the cost)."""
    return [(white, mask) for white in (False, True) for mask in (False, True)] if B <= 5 else [(True, True)]


def _fixed(on=True):
    class _Ctx:
        def __enter__(self):
            self.was = (torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled())
            torch.use_deterministic_algorithms(on)

        def __exit__(self, *a):
            torch.use_deterministic_algorithms(self.was[0], warn_only=self.was[1])
    return _Ctx()


# ----------------------------------------------------------------------------------------- kernels vs float64, no drift
@pytest.mark.parametrize("B", [5, 24])
@pytest.mark.parametrize("with_albedo", [False, True])
@pytest.mark.parametrize("composite", ["tf", "numpy"])
def test_shade_backward_params_vs_float64(composite, with_albedo, B):
    """rn_phong_shade_backward_params (and its twin) against float64 at the module's bar; with a uniform ambient array, d_normal,
    d_albedo of the atomic entry and every output of the twin equal the scalar entries' bit for bit."""
    from rendernet_b200 import ops
    worst = np.zeros(4)
    kd = 0.9
    for white, mask in _configs(B):
        n, ld, col, amb, near = _inputs(B, composite, white)
        ex = _excluded(n, ld, col, amb.reshape(B, 1, 1, 1), kd, composite, white, mask)
        rng = np.random.default_rng(B + 3 * white + 5 * mask)
        alb = rng.random(n.shape).astype(np.float32) if with_albedo else None
        g = rng.standard_normal(n.shape).astype(np.float32)
        g[ex] = 0.0
        kw = dict(albedo=None if alb is None else _d(alb), composite=composite, background_white=white, with_mask=mask)
        N, G, LD, LC, A = _d(n), _d(g), _d(ld), _d(col), _d(amb)
        dn, da, dl, dcol, damb = ops.phong_shade_backward(N, G, LD, LC, A, kd, want_shading_grad=True, **kw)
        with _fixed():
            fx = ops.phong_shade_backward(N, G, LD, LC, A, kd, want_shading_grad=True, **kw)
            fx2 = ops.phong_shade_backward(N, G, LD, LC, A, kd, want_shading_grad=True, **kw)
        for a, b in zip(fx, fx2):                                   # the twin repeats bit for bit
            assert a is None or torch.equal(a, b)
        ref = _vjp(composite, white, mask, n, ld, col, amb, kd, g, alb)
        ref_abs = _vjp(composite, white, mask, n, ld, col, amb, kd, np.abs(g), None if alb is None else np.abs(alb))
        e = _param_err(dcol, damb, ref, ref_abs)
        e_fx = _param_err(fx[3], fx[4], ref, ref_abs)
        worst = np.maximum(worst, [*e, *e_fx])
        # no drift: a uniform ambient array gives the scalar entries' bits
        a0 = float(amb[1])
        A0 = torch.full((B,), a0, device=dev)
        s_dn, s_da, _ = ops.phong_shade_backward(N, G, LD, LC, a0, kd, **kw)
        p_dn, p_da, _, _, _ = ops.phong_shade_backward(N, G, LD, LC, A0, kd, want_shading_grad=True, **kw)
        assert torch.equal(s_dn, p_dn) and (s_da is None or torch.equal(s_da, p_da))
        with _fixed():
            s = ops.phong_shade_backward(N, G, LD, LC, a0, kd, **kw)
            p = ops.phong_shade_backward(N, G, LD, LC, A0, kd, want_shading_grad=True, **kw)
        for x, y in zip(s, p[:3]):
            assert x is None or torch.equal(x, y)
        print(f"{composite} albedo={with_albedo} B={B} white={white} mask={mask}: {int(ex.sum())} excluded; atomic d_col "
              f"{e[0]:.2e} d_amb {e[1]:.2e}; fixed d_col {e_fx[0]:.2e} d_amb {e_fx[1]:.2e} (of sum|term|)")
    print(f"worst: atomic {worst[0]:.2e} / {worst[1]:.2e}, fixed {worst[2]:.2e} / {worst[3]:.2e}; bar {BAR:.2e}")
    assert worst.max() <= BAR


@pytest.mark.parametrize("B", [5, 24])
def test_composite_loss_grad_params_vs_float64(B):
    """The Shader fit's objective with per-item ambient: d_light_col, d_ambient at the bar (atomic and twin); loss, d_img and
    d_light_dir with a uniform ambient array equal the scalar entry's bit for bit (d_img from the atomic entries, loss and
    d_light_dir from the twins, whose sums have a fixed order)."""
    from rendernet_b200 import ops
    worst = np.zeros(4)
    kd = 0.9
    for white, mask in _configs(B):
        n, ld, col, amb, near = _inputs(B, "numpy", white)
        ex = _excluded(n, ld, col, amb.reshape(B, 1, 1, 1), kd, "numpy", white, mask)
        N, LD, LC, A = _d(n), _d(ld), _d(col), _d(amb)
        out = ops.phong_shade(N, LD, LC, A, kd, composite="numpy", background_white=white, with_mask=mask)[0].cpu().numpy()
        tgt = np.random.default_rng(B + 3 * white + 5 * mask).random(n.shape).astype(np.float32)
        tgt[ex] = out[ex]                                         # the device's own image there: no gradient
        T = _d(tgt)
        loss, dimg, dl, dcol, damb = ops.phong_composite_loss_grad(N, T, LD, LC, A, kd, white, mask, want_shading_grad=True)
        with _fixed():
            fx = ops.phong_composite_loss_grad(N, T, LD, LC, A, kd, white, mask, want_shading_grad=True)
        assert torch.equal(fx[1], dimg)                           # per-pixel outputs: the same bits in both
        g = 2.0 * (out.astype(np.float64) - tgt) / (3 * H * W)
        ref = np_vjp64(n, ld, col, amb, kd, white, mask, g)
        ref_abs = np_vjp64(n, ld, col, amb, kd, white, mask, np.abs(g))
        e, e_fx = _param_err(dcol, damb, ref, ref_abs), _param_err(fx[3], fx[4], ref, ref_abs)
        worst = np.maximum(worst, [*e, *e_fx])
        a0 = float(amb[2])
        A0 = torch.full((B,), a0, device=dev)
        s = ops.phong_composite_loss_grad(N, T, LD, LC, a0, kd, white, mask)
        p = ops.phong_composite_loss_grad(N, T, LD, LC, A0, kd, white, mask, want_shading_grad=True)
        assert torch.equal(s[1], p[1])
        with _fixed():
            s = ops.phong_composite_loss_grad(N, T, LD, LC, a0, kd, white, mask)
            p = ops.phong_composite_loss_grad(N, T, LD, LC, A0, kd, white, mask, want_shading_grad=True)
        for x, y in zip(s, p[:3]):
            assert torch.equal(x, y)
        print(f"composite loss B={B} white={white} mask={mask}: atomic {e[0]:.2e} / {e[1]:.2e}, fixed {e_fx[0]:.2e} / "
              f"{e_fx[1]:.2e}")
    print(f"worst {worst}; bar {BAR:.2e}")
    assert worst.max() <= BAR


@pytest.mark.parametrize("B", [5, 24])
def test_recon_loss_grad_params_vs_float64(B):
    """The face-reconstruction objective with per-item ambient, as the composite objective's test."""
    from rendernet_b200 import ops
    worst = np.zeros(4)
    kd = 0.9
    for white, mask in _configs(B):
        n, ld, col, amb, near = _inputs(B, "tf", white)
        ex = _excluded(n, ld, col, amb.reshape(B, 1, 1, 1), kd, "tf", white, mask)
        rng = np.random.default_rng(B + 3 * white + 5 * mask)
        alb = rng.random(n.shape).astype(np.float32)
        tgt = rng.random(n.shape).astype(np.float32)
        alb[ex] = tgt[ex] = 0.0
        AL, N, T, LD, LC, A = _d(alb), _d(n), _d(tgt), _d(ld), _d(col), _d(amb)
        kw = dict(black_background=not white, with_mask=mask)
        loss, da, dn, dl, dcol, damb = ops.phong_recon_loss_grad(AL, N, T, LD, LC, A, kd, want_shading_grad=True, **kw)
        with _fixed():
            fx = ops.phong_recon_loss_grad(AL, N, T, LD, LC, A, kd, want_shading_grad=True, **kw)
        assert torch.equal(fx[1], da) and torch.equal(fx[2], dn)
        shade = tf_vjp64(n, ld, col, amb, kd, not white, mask, np.zeros(n.shape))[0]
        g = 2.0 * (alb * shade - tgt) / (3 * H * W)
        ref = tf_vjp64(n, ld, col, amb, kd, not white, mask, g, alb)
        ref_abs = tf_vjp64(n, ld, col, amb, kd, not white, mask, np.abs(g), alb)
        e, e_fx = _param_err(dcol, damb, ref, ref_abs), _param_err(fx[4], fx[5], ref, ref_abs)
        worst = np.maximum(worst, [*e, *e_fx])
        a0 = float(amb[3])
        A0 = torch.full((B,), a0, device=dev)
        s = ops.phong_recon_loss_grad(AL, N, T, LD, LC, a0, kd, **kw)
        p = ops.phong_recon_loss_grad(AL, N, T, LD, LC, A0, kd, want_shading_grad=True, **kw)
        assert torch.equal(s[1], p[1]) and torch.equal(s[2], p[2])
        with _fixed():
            s = ops.phong_recon_loss_grad(AL, N, T, LD, LC, a0, kd, **kw)
            p = ops.phong_recon_loss_grad(AL, N, T, LD, LC, A0, kd, want_shading_grad=True, **kw)
        for x, y in zip(s, p[:4]):
            assert torch.equal(x, y)
        print(f"recon loss B={B} white={white} mask={mask}: atomic {e[0]:.2e} / {e[1]:.2e}, fixed {e_fx[0]:.2e} / {e_fx[1]:.2e}")
    print(f"worst {worst}; bar {BAR:.2e}")
    assert worst.max() <= BAR


@pytest.mark.parametrize("composite", ["tf", "numpy"])
def test_shade_ambient_forward_is_the_scalar_entry(composite):
    """rn_phong_shade_ambient: a uniform array gives rn_phong_shade's bits, and item b of a per-item array gives the scalar
    entry's image at ambient[b] bit for bit (shade, compos and uint8), with and without albedo, mask on and off."""
    from rendernet_b200 import ops
    B = 5
    for white, mask in _configs(B):
        n, ld, col, amb, _ = _inputs(B, composite, white)
        alb = np.random.default_rng(3).random(n.shape).astype(np.float32)
        for albedo in (None, _d(alb)):
            kw = dict(albedo=albedo, composite=composite, background_white=white, with_mask=mask)
            got = ops.phong_shade(_d(n), _d(ld), _d(col), _d(amb), 0.9, **kw)
            uni = ops.phong_shade(_d(n), _d(ld), _d(col), torch.full((B,), float(amb[2]), device=dev), 0.9, **kw)
            ref = ops.phong_shade(_d(n), _d(ld), _d(col), float(amb[2]), 0.9, **kw)
            for x, y in zip(uni, ref):
                assert torch.equal(x, y)
            for b in range(B):
                one = ops.phong_shade(_d(n[b:b + 1]), _d(ld[b:b + 1]), _d(col[b:b + 1]), float(amb[b]), 0.9,
                                      **dict(kw, albedo=None if albedo is None else albedo[b:b + 1]))
                for x, y in zip(got, one):
                    assert torch.equal(x[b:b + 1], y)


# ----------------------------------------------------------------------------------------- twins: batch invariance
def test_twins_item_alone_equals_item_in_batch():
    """Each fixed twin gives an item the same bits alone as inside a batch of three."""
    from rendernet_b200 import ops
    n, ld, col, amb, _ = _inputs(3, "tf", True)
    rng = np.random.default_rng(5)
    alb, tgt, g = (rng.random(n.shape).astype(np.float32) for _ in range(3))
    with _fixed():
        def run(sl):
            args = [_d(x[sl]) for x in (n, ld, col, amb, alb, tgt, g)]
            N, LD, LC, A, AL, T, G = args
            return (ops.phong_shade_backward(N, G, LD, LC, A, 0.9, albedo=AL, want_shading_grad=True),
                    ops.phong_recon_loss_grad(AL, N, T, LD, LC, A, 0.9, want_shading_grad=True),
                    ops.phong_composite_loss_grad(N, T, LD, LC, A, 0.9, True, True, want_shading_grad=True))
        whole = run(slice(0, 3))
        for b in range(3):
            alone = run(slice(b, b + 1))
            for w_out, a_out in zip(whole, alone):
                for x, y in zip(w_out, a_out):
                    assert torch.equal(x[b:b + 1], y)


# ----------------------------------------------------------------------------------------- nn.phong_shade
@pytest.mark.parametrize("rows", [1, 4])
@pytest.mark.parametrize("composite", ["tf", "numpy"])
def test_nn_phong_shade_shading_gradients(composite, rows):
    """Autograd of nn.phong_shade with light_col [rows,3] and ambient [rows] requiring grad, under
    torch.use_deterministic_algorithms(True): equal bit for bit to ops.phong_shade_backward's per-item gradients (summed over the
    batch for a single row) and from run to run; the atomic path agrees to 1e-4 of scale (the sums cancel: G is signed)."""
    from rendernet_b200 import ops
    from rendernet_b200.nn import phong_shade
    B = 4
    n, ld, col, amb, _ = _inputs(B, composite, True)
    rng = np.random.default_rng(11)
    alb, G = rng.random(n.shape).astype(np.float32), rng.standard_normal(n.shape).astype(np.float32)
    lc0 = np.float32([[0.8, 0.6, 0.5]]) if rows == 1 else col[:rows]
    a0 = np.float32([0.2]) if rows == 1 else amb[:rows]

    def run():
        lc, a = _d(lc0).requires_grad_(), _d(a0).requires_grad_()
        l = _d(ld).requires_grad_()
        (phong_shade(_d(n), l, albedo=_d(alb), composite=composite, light_col=lc, ambient=a, k_diffuse=0.9) * _d(G)).sum().backward()
        return lc.grad, a.grad, l.grad
    with _fixed():                                              # fixed-order sums: the comparison can be exact
        lc_g, a_g, l_g = run()
        r2 = run()
        _, _, dl, dcol, damb = ops.phong_shade_backward(_d(n), _d(G), _d(ld), _d(np.broadcast_to(lc0, (B, 3))),
                                                        _d(np.broadcast_to(a0, (B,))), 0.9, albedo=_d(alb),
                                                        composite=composite, want_shading_grad=True)
    want_c, want_a = (dcol.sum(0, keepdim=True), damb.sum(0, keepdim=True)) if rows == 1 else (dcol, damb)
    assert torch.equal(lc_g, want_c) and torch.equal(a_g, want_a) and torch.equal(l_g, dl)
    for x, y in zip((lc_g, a_g, l_g), r2):
        assert torch.equal(x, y)
    lc_a, a_a, _ = run()                                        # the atomic kernels: the same within the module's bar
    assert (lc_a - lc_g).abs().max() <= 1e-4 * lc_g.abs().max() and (a_a - a_g).abs().max() <= 1e-4 * a_g.abs().max()


# ----------------------------------------------------------------------------------------- the fits
TRUE_COL, TRUE_AMB = np.float32([0.8, 0.6, 0.5]), np.float32(0.2)


def _chair():
    import os
    bv = np.load(os.path.join(os.path.dirname(__file__), "golden", "binvox.npz"))
    return np.unpackbits(bv["chair_bits"]).reshape(1, 64, 64, 64, 1).astype(np.float32)


def test_shader_pose_fit_recovers_colour_and_ambient():
    """A target rendered through the Shader network (seeded weights) at a known pose, light direction, colour (0.8, 0.6, 0.5) and
    ambient 0.2.  ShaderPoseFit(fit_shading=True) starts from the true pose and direction with the default shading (white,
    0.1) and, after 300 plain steps at shading_eta 0.5, holds the colour within 0.05 and the ambient term within 0.02 of the
    truth in every hypothesis, at a lower loss than the same steps with fit_shading=False.  The colour is the slow direction of
    plain descent: its curvature carries (k_d max(d, 0))^2, the ambient term's does not.  Measured on an H100 80GB HBM3 (700 W)
    after 300 steps: colour error 0.033, ambient 0.0009, loss 3.0e-5 against 1.0e-2 without fit_shading.  Under the
    deterministic flag, fit_shading=False repeats today's trajectory bit for bit (the update written out here)."""
    from rendernet_b200.RenderNet_demo import compute_pose_param
    from rendernet_b200.shader_fit import ShaderPoseFit, shader_fit_gradients
    STEPS = 300
    pose = np.tile(compute_pose_param(262.0, 54.0, 3.3)[0].astype(np.float32), (5, 1))
    light = np.tile(np.float32([math.radians(280.0), math.radians(60.0)]), (5, 1))
    fit = ShaderPoseFit(None, _chair(), objective="phong", precision="fast", fit_shading=True, shading_eta=0.5)
    target = fit.render(dict(pose=pose, light=light, light_col=np.tile(TRUE_COL, (5, 1)),
                             ambient=np.full(5, TRUE_AMB)))["shaded"]
    state = dict(pose=pose, light=light, **fit.initial_shading())
    for _ in range(STEPS):
        state, loss_on, _ = fit.step(state, target)
    l_on = fit.loss(state, target)
    del fit                                                     # one network's recorded activations on the device at a time
    gc.collect()
    plain = ShaderPoseFit(None, _chair(), objective="phong", precision="fast")
    s2 = dict(pose=pose, light=light)
    for _ in range(STEPS):
        s2, loss_off, _ = plain.step(s2, target)
    l_off = plain.loss(s2, target)
    e_col = np.abs(state["light_col"] - TRUE_COL).max()
    e_amb = np.abs(state["ambient"] - TRUE_AMB).max()
    print(f"shader fit after {STEPS}: colour {state['light_col'][0]}, ambient {state['ambient'][0]:.4f} "
          f"(errors {e_col:.3e}, {e_amb:.3e}); loss {l_on.max():.3e} vs {l_off.min():.3e} without fit_shading")
    assert e_col <= 0.05 and e_amb <= 0.02 and l_on.max() < l_off.min()
    with _fixed():
        s3, s4 = dict(pose=pose, light=light), dict(pose=pose, light=light)
        for _ in range(2):
            s3, _, _ = plain.step(s3, target)
            _, g = shader_fit_gradients(plain.ig, plain.voxels, s4["pose"], plain._target_dev(target), "phong",
                                        light=s4["light"], **plain.phong)
            gp = np.asarray(g["pose"], np.float32).copy()
            gp[:, 2] = 0.0
            s4 = dict(pose=(s4["pose"] - np.float32(0.01) * gp).astype(np.float32),
                      light=(s4["light"] - np.float32(0.4) * np.asarray(g["light"], np.float32)).astype(np.float32))
        assert set(s3) == {"pose", "light"}
        assert np.array_equal(s3["pose"], s4["pose"]) and np.array_equal(s3["light"], s4["light"])


def test_face_reconstruction_recovers_colour_and_ambient():
    """The same through the pretrained-format Texture+Normal network (seeded weights) and TensorFlow's composite: the target
    has colour (0.8, 0.6, 0.5) and ambient 0.2; FaceReconstruction(fit_shading=True) starts from the true latent, texture, pose
    and light azimuth with the reference's white light and ambient 0.  The latent and texture are held (shape_eta = tex_eta =
    0): the albedo times the colour is what the image fixes, so a moving texture could take up the colour.  The colour's
    curvature here also carries the albedo squared, so plain descent moves it slowly: after 300 steps at shading_eta 1.0 the
    colour is within 0.25 of the truth (from 0.5) and the ambient term within 0.03, at under a tenth of the loss without
    fit_shading.  Measured on an H100 80GB HBM3 (700 W): colour error 0.183, ambient 0.006, loss 9.7e-5 against 9.1e-3."""
    from oracle.shape_decoder import init_shape_decoder_weights
    from oracle import rendernet_oracle as orc
    from rendernet_b200.Reconstruct_RenderNet_Face import FaceReconstruction, pretrained_dict_from_texture_weights
    STEPS = 300
    W = orc.init_texture_weights(seed=61, alpha_range=(-0.3, 0.3), bias_jitter=0.02)
    for k in list(W):
        if k.endswith("/alpha") and "/res" in k:
            W[k] = np.zeros_like(W[k])
    Wp, Wd = pretrained_dict_from_texture_weights(W), init_shape_decoder_weights(62)
    kw = dict(batch=5, precision="fast", shape_eta=0.0, tex_eta=0.0)
    rec = FaceReconstruction(Wp, Wd, fit_shading=True, shading_eta=1.0, **kw)
    rng = np.random.default_rng(63)
    truth = dict(latent=np.full((5, 200), 0.5, np.float32), texture=np.tile(rng.standard_normal(199).astype(np.float32), (5, 1)),
                 pose=np.tile(np.float32([math.radians(270.0), math.radians(5.0), 1.0]), (5, 1)),
                 light=np.full((5, 1), math.radians(290.0), np.float32))
    target = rec.render(dict(truth, light_col=np.tile(TRUE_COL, (5, 1)), ambient=np.full(5, TRUE_AMB)))["compos"]
    state = dict(truth, **rec.initial_shading())
    for _ in range(STEPS):
        state, _, _ = rec.step(state, target)
    l_on = rec.loss(state, target)
    del rec                                                     # one network's recorded activations on the device at a time
    gc.collect()
    plain = FaceReconstruction(Wp, Wd, **kw)
    s2 = dict(truth)
    for _ in range(STEPS):
        s2, _, _ = plain.step(s2, target)
    l_off = plain.loss(s2, target)
    e_col = np.abs(state["light_col"] - TRUE_COL).max()
    e_amb = np.abs(state["ambient"] - TRUE_AMB).max()
    print(f"face fit after {STEPS}: colour {state['light_col'][0]}, ambient {state['ambient'][0]:.4f} "
          f"(errors {e_col:.3e}, {e_amb:.3e}); loss {l_on.max():.3e} vs {l_off.min():.3e} without fit_shading")
    assert e_col <= 0.25 and e_amb <= 0.03 and l_on.max() < 0.1 * l_off.min()


# ----------------------------------------------------------------------------------------- RenderEngine per-step light
@pytest.mark.parametrize("fuse", [True, False])
def test_render_engine_per_step_light(fuse):
    """RenderEngine(phong=...) rendering with light_dir / light_col passed per step equals, bit for bit, a fresh engine built
    with that light, fused and unfused; the graph is captured once, and None keeps the last light."""
    from oracle import rendernet_oracle as orc
    from rendernet_b200.engine import RenderEngine
    B = 2
    vox = np.repeat(_chair(), B, 0)
    pose = np.stack([orc.compute_pose_param(250.0, 60.0, 3.3)[0], orc.compute_pose_param(100.0, 40.0, 3.0)[0]]).astype(np.float32)
    base = dict(light_dir=orc.generate_light_pos(60.0, 250.0).astype(np.float32), light_col=np.ones((1, 3), np.float32),
                ambient=0.1, k_diffuse=0.9)
    lights = [(np.float32([[0.3, 0.8, 0.5], [-0.5, 0.6, 0.2]]), np.float32([[0.8, 0.6, 0.5]])),
              (np.float32([[0.1, 0.9, -0.3]]), np.float32([[1.0, 0.7, 0.9], [0.4, 0.5, 0.6]]))]
    eng = RenderEngine(None, B, phong=base, fuse_phong=fuse, precision="fast")
    graph = eng.graph
    for ld, lc in lights:
        got = eng.render(vox, pose, light_dir=ld, light_col=lc)
        fresh = RenderEngine(None, B, phong=dict(base, light_dir=ld, light_col=lc), fuse_phong=fuse, precision="fast")
        want = fresh.render(vox, pose)
        assert eng.graph is graph
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
        again = eng.render(vox, pose)                                        # None: the last light stays
        assert torch.equal(again[1], want[1])
        t = eng.submit(vox, pose, light_dir=ld, light_col=lc)
        assert torch.equal(eng.result(t), want[1])
        del fresh, want                                         # one reference engine on the device at a time
        gc.collect()
