"""GPU tests of every Phong kernel at the pixels where such kernels go wrong, against the closed-form float64 vector-Jacobian
products of oracle/phong_vjp.py (which, unlike autograd of oracle/phong_tf.py and oracle/phong_np.py, are defined at n =
(0.5, 0.5, 0.5) and where the mask's |a| is 0): rn_phong_recon_loss_grad, rn_phong_shade_backward, rn_phong_composite_loss_grad,
rn_phong_shade and rn_phong_composite, and the face-reconstruction step through TextureInputGradients.

The catalogue (_catalogue) holds, in every item: the singular points n = (0.5, 0.5, 0.5), (0, 0, 0), (1, 1, 1) (some at thread 0
of a block, some in the last, partial block); one-ulp neighbours of 0.5 in one, two and three components (|v| ~ 2^-24, dL/dn
~ 1 / |v|); d = u.L exactly 0 and exactly 1; composites exactly 0 and 1; masks saturated to exactly 1.0 in double; a band on
the mask's transition; the diffuse clip at col up to 1.2; random pixels.  Items: light (0, 0, 2), light (-2, 0, 0) and two
random ones; images 37 x 29 (1073 pixels, 49 in the last block) and 509 x 511 (3 in the last block).

A pixel within 1e-6 of a kink in float64 but not on it (|d| or |pre - 1|, or the composite just above 1) may take the other
branch in fp32; such pixels get a zero upstream gradient, so they are compared but carry no gradient.  With the fixed seeds
below that is 6-26 pixels per configuration at 37 x 29 and 6-16 at 509 x 511, except on the black background at (ambient,
k_d) = (0.1, 0.9): 2452 (TF) and 3475 (NumPy) of the 1.04 M pixels, where a mask below 1e-6 leaves composites just above 1.
The tests print the counts and assert they stay under 1 %.  Errors are max |error| / max |reference| over the pixels that are
not one-ulp neighbours of 0.5 ("scale"); those are held to 1e-5 of their own magnitude instead, with an upstream gradient of
one sign in all three channels so that dL/dd is not a cancelling sum."""
import math

import numpy as np
import pytest
import torch

from oracle.phong_vjp import mask32, np_vjp64, tf_vjp64

dev = "cuda"
SIZES = [(37, 29), (509, 511)]
PAIRS = [(0.0, 1.0), (0.1, 0.9)]             # (ambient, k_diffuse)
H5 = np.float32(0.5)
UP, DN = np.nextafter(H5, np.float32(1)), np.nextafter(H5, np.float32(0))


def _d(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _lights():
    rng = np.random.default_rng(7)
    ld = np.array([[0.0, 0.0, 2.0], [-2.0, 0.0, 0.0], 1.7 * rng.standard_normal(3), 1.7 * rng.standard_normal(3)], np.float32)
    col = np.array([[1.0, 1.0, 1.0], [1.0, 1.0, 1.0], [1.2, 1.0, 0.7], rng.uniform(0.6, 1.2, 3)], np.float32)
    return ld, col


def _mask_arg(n, composite, white):
    """The argument s of the composite's soft mask sigmoid(s), float64 [..., 1]."""
    nn_ = np.linalg.norm(n.astype(np.float64), axis=-1, keepdims=True)
    if composite == "numpy":
        return 255.0 * np.linalg.norm(1.0 - n.astype(np.float64), axis=-1, keepdims=True) - 80 if white else 255.0 * nn_ - 150
    return 255.0 * (math.sqrt(3) - nn_) - 80 if white else 255.0 * nn_ - 80


def _catalogue(H, W, composite, white):
    """Normal maps [4,H,W,3] fp32 and the masks (half: n = 0.5; near: one-ulp neighbours of 0.5)."""
    ld, col = _lights()
    B, HW = len(ld), H * W
    rng = np.random.default_rng(H * W + 2 * white + (composite == "numpy"))
    n = rng.random((B, HW, 3)).astype(np.float32)
    # the mask's transition band (|s| < 15) at an eighth of the pixels, beyond the first two blocks
    idx = 512 + rng.choice(HW - 600, HW // 8, replace=False)
    dirs = rng.random((B, len(idx), 3)) + 0.05
    dirs /= np.linalg.norm(dirs, axis=-1, keepdims=True)
    r = rng.uniform(0.27, 0.36, (B, len(idx), 1))
    if composite == "numpy":
        band = 1.0 - dirs * r if white else dirs * rng.uniform(0.55, 0.63, (B, len(idx), 1))
    else:
        band = 0.818 + rng.uniform(-0.05, 0.05, (B, len(idx), 3)) if white else dirs * r
    n[:, idx] = np.clip(band, 0.0, 1.0)
    near = [[UP, H5, H5], [H5, DN, H5], [H5, H5, UP], [H5, H5, DN], [UP, UP, H5], [DN, H5, UP], [UP, UP, UP], [DN, DN, DN],
            [UP, DN, UP]]
    for b in range(B):
        L = ld[b].astype(np.float64) / np.linalg.norm(ld[b])
        perp = np.cross(L, [0.0, 1.0, 0.0] if abs(L[1]) < 0.9 else [1.0, 0.0, 0.0])
        perp /= np.linalg.norm(perp)
        spec = np.array([[0.5, 0.5, 0.5], [0.0, 0.0, 0.0], [1.0, 1.0, 1.0]] + near + [
            0.5 + 0.25 * perp,                                  # d = 0 (exactly, for the axis lights)
            0.5 + 0.25 * L,                                     # d = 1: pre = k_d col, composite 1 at k_d = col = 1
            0.5 + 0.4 * L,                                      # d = 1 elsewhere on the ray: pre > 1 where col > 1
            0.5 - 0.25 * L,                                     # unlit, saturated mask: composite 0 at ambient 0
            [0.9, 0.95, 1.0], [0.0, 0.02, 0.05]], np.float32)   # saturated masks (TF black / white)
        k = len(spec)
        n[b, :k] = spec                                         # thread 0 of block 0 is n = 0.5
        n[b, 256:256 + k] = np.roll(spec, -1, 0)                # thread 0 of block 1 is n = 0
        n[b, HW - k:] = np.roll(spec, 3, 0)                     # the last three pixels: n = 0.5, 0, 1
    n = np.clip(n, 0.0, 1.0).reshape(B, H, W, 3)
    half = (n == 0.5).all(-1)
    vn = np.linalg.norm(n.astype(np.float64) - 0.5, axis=-1)
    return n, ld, col, half, (vn > 0) & (vn < 1e-6)


def _excluded(n, ld, col, ambient, kd, composite, white, mask):
    """Pixels within 1e-6 of a kink in float64 but not on it: d = u.L near 0, pre near 1, or the composite just above 1 (it
    cannot fall below 0, nor be above 1 in fp32 where it is not in exact arithmetic)."""
    L = ld.astype(np.float64) / np.linalg.norm(ld.astype(np.float64), axis=-1, keepdims=True)
    v = n.astype(np.float64) - 0.5
    vn = np.linalg.norm(v, axis=-1, keepdims=True)
    with np.errstate(invalid="ignore", divide="ignore"):
        d = np.where(vn > 0, (v * L[:, None, None]).sum(-1, keepdims=True) / vn, 0.0)
    pre = kd * np.maximum(d, 0.0) * col.astype(np.float64)[:, None, None]
    x = ambient + np.clip(pre, 0.0, 1.0)
    if mask:
        m = mask32(n, white) if composite == "numpy" else 1.0 / (1.0 + np.exp(-_mask_arg(n, composite, white)))
        x = m * x + (1.0 - m)
    ex = (np.abs(d[..., 0]) < 1e-6) & (d[..., 0] != 0)
    ex |= ((np.abs(pre - 1.0) < 1e-6) & (pre != 1.0)).any(-1) & (d[..., 0] >= 0)
    ex |= ((x > 1.0) & (x < 1.0 + 1e-6)).any(-1)
    return ex


def _normal_errors(got, ref, band, half, near):
    """dL/dn: (off the band, on it) relative to the scale of the regular pixels, and the worst one-ulp neighbour of 0.5
    relative to its own magnitude.  Asserts it is finite and exactly 0 at n = 0.5 (the mask is saturated there)."""
    got = got.detach().double().cpu().numpy()
    assert np.isfinite(got).all()
    assert (got[half] == 0).all() and (ref[half] == 0).all()
    reg = ~near
    err = np.abs(got - ref).max(-1)
    scale = np.abs(ref[reg]).max()
    e_off = float(err[reg & ~band].max() / scale)
    e_band = float(err[reg & band].max() / scale) if (reg & band).any() else 0.0
    mag = np.abs(ref[near]).max(-1)
    assert ((err[near] == 0) | (mag > 0)).all()
    e_near = float((err[near] / np.where(mag > 0, mag, 1.0)).max())
    return e_off, e_band, e_near


def _plain_errors(got, ref, band=None):
    """(off the band, on it) relative to the scale of ref; the whole array when band is None."""
    got = got.detach().double().cpu().numpy()
    assert np.isfinite(got).all()
    err = np.abs(got - ref)
    scale = max(np.abs(ref).max(), 1e-300)
    if band is None:
        return float(err.max() / scale), 0.0
    err = err.max(-1)
    return float(err[~band].max() / scale), float(err[band].max() / scale) if band.any() else 0.0


def _configs():
    return [(white, mask, pair) for white in (False, True) for mask in (False, True) for pair in PAIRS]


# ----------------------------------------------------------------------------------------- rn_phong_recon_loss_grad
@pytest.mark.gpu
@pytest.mark.parametrize("H,W", SIZES)
def test_recon_loss_grad_on_the_catalogue(H, W):
    """The face-reconstruction objective against float64, both backgrounds, mask on and off, (ambient, k_d) = (0, 1) and
    (0.1, 0.9): loss 1e-6 relative; d_albedo and d_normal 1e-6 of scale off the mask band and 1e-5 on it, the one-ulp
    neighbours of 0.5 1e-5 of their own magnitude, n = 0.5 exactly 0; d_light 1e-5 of scale; every output finite.  Measured on
    an H100 80GB HBM3 (700 W), worst over the configurations and both sizes: loss 7.0e-8, d_normal 1.4e-7 (band 1.6e-7, ulp
    neighbours 4.2e-7), d_albedo 4.0e-7 (band 3.5e-7), d_light 9.7e-7."""
    from rendernet_b200 import ops
    worst = np.zeros(7)
    for white, mask, (amb, kd) in _configs():
        n, ld, col, half, near = _catalogue(H, W, "tf", white)
        ex = _excluded(n, ld, col, amb, kd, "tf", white, mask)
        rng = np.random.default_rng(H + 3 * white + 5 * mask)
        alb = rng.random(n.shape).astype(np.float32)
        tgt = rng.random(n.shape).astype(np.float32)
        alb[ex] = tgt[ex] = 0.0                                 # r = 0: the excluded pixels carry no gradient
        tgt[near] = 0.0                                         # r >= 0 in every channel: no cancellation in dL/dd
        loss, da, dn, dl = ops.phong_recon_loss_grad(_d(alb), _d(n), _d(tgt), _d(ld), _d(col), amb, kd,
                                                      black_background=not white, with_mask=mask)
        shade = tf_vjp64(n, ld, col, amb, kd, not white, mask, np.zeros(n.shape))[0]
        r = alb * shade - tgt
        g = 2.0 * r / (3 * H * W)
        _, dn_ref, da_ref, dl_ref = tf_vjp64(n, ld, col, amb, kd, not white, mask, g, alb)
        band = (np.abs(_mask_arg(n, "tf", white)[..., 0]) < 15) if mask else np.zeros(half.shape, bool)
        loss_ref = (r ** 2).mean(axis=(1, 2, 3))
        e_loss = float((np.abs(loss.cpu().numpy() - loss_ref) / loss_ref).max())
        e_n = _normal_errors(dn, dn_ref, band, half, near)
        e_a = _plain_errors(da, da_ref, band)
        e_l = _plain_errors(dl, dl_ref)[0]
        if not mask:
            assert (dn.cpu().numpy()[half] == 0).all()
        print(f"{H}x{W} white={white} mask={mask} amb,kd={amb},{kd}: {int(ex.sum())} excluded; loss {e_loss:.2e}; d_normal "
              f"{e_n[0]:.2e} (band {e_n[1]:.2e}, ulp neighbours {e_n[2]:.2e}); d_albedo {e_a[0]:.2e} (band {e_a[1]:.2e}); "
              f"d_light {e_l:.2e}")
        assert ex.mean() < 0.01
        worst = np.maximum(worst, [e_loss, *e_n, *e_a, e_l])
    print(f"worst: loss {worst[0]:.2e}, d_normal {worst[1]:.2e} / band {worst[2]:.2e} / ulp {worst[3]:.2e}, d_albedo "
          f"{worst[4]:.2e} / band {worst[5]:.2e}, d_light {worst[6]:.2e}")
    assert worst[0] <= 1e-6 and worst[1] <= 1e-6 and worst[2] <= 1e-5 and worst[3] <= 1e-5
    assert worst[4] <= 1e-6 and worst[5] <= 1e-5 and worst[6] <= 1e-5


# ----------------------------------------------------------------------------------------- rn_phong_shade_backward
@pytest.mark.gpu
@pytest.mark.parametrize("H,W", SIZES)
@pytest.mark.parametrize("with_albedo", [False, True])
@pytest.mark.parametrize("composite", ["tf", "numpy"])
def test_phong_shade_backward_on_the_catalogue(composite, with_albedo, H, W):
    """rn_phong_shade_backward for a random upstream gradient against float64, at the bars of the recon objective's test.
    Measured on an H100 80GB HBM3 (700 W), worst over all cases: d_normal 3.0e-7 (band 1.8e-7, ulp neighbours 4.0e-7),
    d_albedo 2.0e-7 (band 2.2e-6, the NumPy composite's fp32 mask), d_light 1.9e-6."""
    from rendernet_b200 import ops
    worst = np.zeros(6)
    vjp = tf_vjp64 if composite == "tf" else np_vjp64
    for white, mask, (amb, kd) in _configs():
        n, ld, col, half, near = _catalogue(H, W, composite, white)
        ex = _excluded(n, ld, col, amb, kd, composite, white, mask)
        rng = np.random.default_rng(W + 3 * white + 5 * mask)
        alb = rng.random(n.shape).astype(np.float32) if with_albedo else None
        g = rng.standard_normal(n.shape).astype(np.float32)
        g[ex] = 0.0
        g[near] = np.abs(g[near])
        dn, da, dl = ops.phong_shade_backward(_d(n), _d(g), _d(ld), _d(col), amb, kd, albedo=None if alb is None else _d(alb),
                                              composite=composite, background_white=white, with_mask=mask)
        _, dn_ref, da_ref, dl_ref = vjp(n, ld, col, amb, kd, white if composite == "numpy" else not white, mask, g, alb)
        band = (np.abs(_mask_arg(n, composite, white)[..., 0]) < 15) if mask else np.zeros(half.shape, bool)
        e_n = _normal_errors(dn, dn_ref, band, half, near)
        e_a = _plain_errors(da, da_ref, band) if with_albedo else (0.0, 0.0)
        e_l = _plain_errors(dl, dl_ref)[0]
        print(f"{composite} albedo={with_albedo} {H}x{W} white={white} mask={mask} amb,kd={amb},{kd}: {int(ex.sum())} excluded; "
              f"d_normal {e_n[0]:.2e} (band {e_n[1]:.2e}, ulp neighbours {e_n[2]:.2e}); d_albedo {e_a[0]:.2e} "
              f"(band {e_a[1]:.2e}); d_light {e_l:.2e}")
        assert ex.mean() < 0.01
        worst = np.maximum(worst, [*e_n, *e_a, e_l])
    print(f"worst: d_normal {worst[0]:.2e} / band {worst[1]:.2e} / ulp {worst[2]:.2e}, d_albedo {worst[3]:.2e} / band "
          f"{worst[4]:.2e}, d_light {worst[5]:.2e}")
    assert worst[0] <= 1e-6 and worst[1] <= 1e-5 and worst[2] <= 1e-5
    assert worst[3] <= 1e-6 and worst[4] <= 1e-5 and worst[5] <= 1e-5


# ----------------------------------------------------------------------------------------- rn_phong_composite_loss_grad
@pytest.mark.gpu
@pytest.mark.parametrize("H,W", SIZES)
def test_composite_loss_grad_on_the_catalogue(H, W):
    """The Shader fit's objective (the NumPy composite, no albedo) against float64 at the same bars.  Measured on an H100 80GB
    HBM3 (700 W): loss 3.5e-8, d_img 1.8e-7 (band 8.1e-6, ulp neighbours 2.7e-7), d_light 8.6e-7."""
    from rendernet_b200 import ops
    worst = np.zeros(5)
    for white, mask, (amb, kd) in _configs():
        n, ld, col, half, near = _catalogue(H, W, "numpy", white)
        ex = _excluded(n, ld, col, amb, kd, "numpy", white, mask)
        out = ops.phong_composite(_d(n), _d(ld), _d(col), amb, kd, background_white=white, with_mask=mask).cpu().numpy()
        tgt = np.random.default_rng(H + 3 * white + 5 * mask).random(n.shape).astype(np.float32)
        tgt[near] = 0.0                                         # r >= 0 in every channel: no cancellation in dL/dd
        tgt[ex] = out[ex]                                       # the device's own image there: no gradient
        loss, dn, dl = ops.phong_composite_loss_grad(_d(n), _d(tgt), _d(ld), _d(col), amb, kd, white, mask)
        shade = np_vjp64(n, ld, col, amb, kd, white, mask, np.zeros(n.shape))[0]
        r = np.where(ex[..., None], 0.0, shade - tgt)
        _, dn_ref, _, dl_ref = np_vjp64(n, ld, col, amb, kd, white, mask, 2.0 * r / (3 * H * W))
        band = (np.abs(_mask_arg(n, "numpy", white)[..., 0]) < 15) if mask else np.zeros(half.shape, bool)
        loss_ref = (r ** 2).mean(axis=(1, 2, 3))
        e_loss = float((np.abs(loss.cpu().numpy() - loss_ref) / loss_ref).max())
        e_n = _normal_errors(dn, dn_ref, band, half, near)
        e_l = _plain_errors(dl, dl_ref)[0]
        print(f"{H}x{W} white={white} mask={mask} amb,kd={amb},{kd}: {int(ex.sum())} excluded; loss {e_loss:.2e}; d_img "
              f"{e_n[0]:.2e} (band {e_n[1]:.2e}, ulp neighbours {e_n[2]:.2e}); d_light {e_l:.2e}")
        assert ex.mean() < 0.01
        worst = np.maximum(worst, [e_loss, *e_n, e_l])
    print(f"worst: loss {worst[0]:.2e}, d_img {worst[1]:.2e} / band {worst[2]:.2e} / ulp {worst[3]:.2e}, d_light {worst[4]:.2e}")
    assert worst[0] <= 1e-6 and worst[1] <= 1e-6 and worst[2] <= 1e-5 and worst[3] <= 1e-5 and worst[4] <= 1e-5


# ----------------------------------------------------------------------------------------- the forward kernels
@pytest.mark.gpu
@pytest.mark.parametrize("H,W", SIZES)
def test_forward_on_the_catalogue(H, W):
    """rn_phong_shade (both composites) and rn_phong_composite against the float64 shading, n = 0.5 shaded as unlit: 1e-6
    off the mask band, 1e-5 on it (absolute; the shading lies in [0, 1]).  Measured on an H100 80GB HBM3 (700 W): 2.6e-7 off
    the band, 3.9e-6 on it."""
    from rendernet_b200 import ops
    worst = np.zeros(2)
    for composite in ("tf", "numpy"):
        for white, mask, (amb, kd) in _configs():
            n, ld, col, half, _ = _catalogue(H, W, composite, white)
            if composite == "tf":
                ref = tf_vjp64(n, ld, col, amb, kd, not white, mask, np.zeros(n.shape))[0]
            else:
                ref = np_vjp64(n, ld, col, amb, kd, white, mask, np.zeros(n.shape))[0]
            assert np.isfinite(ref).all()
            shade, _, _ = ops.phong_shade(_d(n), _d(ld), _d(col), amb, kd, composite=composite, background_white=white,
                                          with_mask=mask, want_compos=False, want_u8=False)
            outs = [shade]
            if composite == "numpy":
                outs.append(ops.phong_composite(_d(n), _d(ld), _d(col), amb, kd, background_white=white, with_mask=mask))
            band = (np.abs(_mask_arg(n, composite, white)[..., 0]) < 15) if mask else np.zeros(half.shape, bool)
            for o in outs:
                got = o.double().cpu().numpy()
                assert np.isfinite(got).all()
                err = np.abs(got - ref).max(-1)
                worst = np.maximum(worst, [err[~band].max(), err[band].max() if band.any() else 0.0])
    print(f"{H}x{W} forward vs float64: {worst[0]:.2e} off the band, {worst[1]:.2e} on it")
    assert worst[0] <= 1e-6 and worst[1] <= 1e-5


# ----------------------------------------------------------------------------------------- fused against composed
@pytest.mark.gpu
@pytest.mark.parametrize("H,W", SIZES)
def test_fused_objective_matches_composed_on_the_catalogue(H, W):
    """With g = the MSE gradient, rn_phong_recon_loss_grad and rn_phong_shade_backward (TF composite, albedo) agree at the bars
    of tests/test_gpu_nn.py::test_phong_backward_matches_the_fused_objectives (1e-6 / 1e-6 / 1e-5 of scale), and both are
    finite at every pixel.  Measured on an H100 80GB HBM3 (700 W): d_normal 1.2e-7, d_albedo 9.8e-8 (the fused objective forms
    g in double, this test in fp32), d_light 8.5e-7."""
    from rendernet_b200 import ops
    worst = np.zeros(3)
    for white, mask, (amb, kd) in _configs():
        n, ld, col, _, _ = _catalogue(H, W, "tf", white)
        rng = np.random.default_rng(W + 7 * white + 11 * mask)
        alb, tgt = (_d(rng.random(n.shape).astype(np.float32)) for _ in range(2))
        nd, ldd, cd = _d(n), _d(ld), _d(col)
        opts = dict(ambient=amb, k_diffuse=kd, composite="tf", background_white=white, with_mask=mask)
        _, compos, _ = ops.phong_shade(nd, ldd, cd, albedo=alb, want_u8=False, **opts)
        g = (compos - tgt) * (2.0 / (3 * H * W))
        dn, da, dl = ops.phong_shade_backward(nd, g, ldd, cd, albedo=alb, **opts)
        _, da_f, dn_f, dl_f = ops.phong_recon_loss_grad(alb, nd, tgt, ldd, cd, amb, kd, black_background=not white,
                                                        with_mask=mask)
        for t in (dn, da, dl, da_f, dn_f, dl_f):
            assert torch.isfinite(t).all()
        e = [_plain_errors(a, b.double().cpu().numpy())[0] for a, b in ((dn_f, dn), (da_f, da), (dl_f, dl))]
        worst = np.maximum(worst, e)
    print(f"{H}x{W} fused vs composed: d_normal {worst[0]:.2e}, d_albedo {worst[1]:.2e}, d_light {worst[2]:.2e}")
    assert worst[0] <= 1e-6 and worst[1] <= 1e-6 and worst[2] <= 1e-5


# ----------------------------------------------------------------------------------------- a reconstruction step
@pytest.mark.gpu
def test_reconstruction_step_with_singular_normals():
    """A face-reconstruction step (TextureInputGradients at B = 2, white background, mask) whose normal map holds n = 0 and
    n = (0.5, 0.5, 0.5): the objective's image gradients are finite, tig.backward chooses its loss scale without a
    FloatingPointError, and dvox, dtex, dpose and d_light are finite."""
    from oracle import rendernet_oracle as orc
    from rendernet_b200 import ops
    from rendernet_b200.backward import TextureInputGradients
    from rendernet_b200.Reconstruct_RenderNet_Face import light_pos
    B = 2
    rng = np.random.default_rng(71)
    W = orc.init_texture_weights(seed=72, alpha_range=(-0.3, 0.3), bias_jitter=0.02)
    vox = ((rng.random((B, 64, 64, 64, 1)) < 0.25) * rng.uniform(0.5, 1.0, (B, 64, 64, 64, 1))).astype(np.float32)
    z = rng.standard_normal((B, 199)).astype(np.float32)
    poses = np.concatenate([orc.compute_pose_param(45.0, 30.0, 2.5), orc.compute_pose_param(130.0, 75.0, 3.0)]).astype(np.float32)
    tig = TextureInputGradients(W, B, precision="exact")
    albedo, normal = tig.forward(vox, z, poses)
    normal[:, 200, 100:108] = 0.0
    normal[:, 300, 300:308] = 0.5
    normal[1, 0, 0] = 0.5
    ldir = torch.from_numpy(light_pos(np.array([[0.4], [2.1]]), 0.7)).to(dev)
    tgt = torch.rand_like(albedo)
    loss, d_albedo, d_normal, d_light = ops.phong_recon_loss_grad(albedo, normal, tgt, ldir, torch.ones(B, 3, device=dev),
                                                                  black_background=False, with_mask=True)
    for name, t in (("loss", loss), ("d_albedo", d_albedo), ("d_normal", d_normal), ("d_light", d_light)):
        assert torch.isfinite(t).all(), name
    dvox, dtex, dpose = tig.backward(d_albedo, d_normal)
    for name, a in (("dvox", dvox), ("dtex", dtex), ("dpose", dpose)):
        assert np.isfinite(a).all(), name
    print(f"loss {loss.cpu().numpy()}, |dvox| {np.abs(dvox).max():.3e}, |dtex| {np.abs(dtex).max():.3e}, "
          f"|dpose| {np.abs(dpose).max():.3e}")
