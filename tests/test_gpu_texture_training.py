"""GPU parity of the Texture+Normal training step (RenderNet_Texture_Face_Normal.py:155-187): the new weight-gradient kernels
against float64, the gradients of all 186 variables of the full-size network against torch.autograd through the oracle chain
(float64 decoder -> device-cell resampler -> concat -> rendernet_texture, two MSEs) with the same dropout masks, two optimiser
steps against the oracle driven by the same Adam formulas, the trained weights in TextureRenderEngine, and overflow recovery."""
import contextlib
import math
import zlib

import numpy as np
import pytest
import torch

from oracle import rendernet_oracle as orc
from oracle import resample_cells as rc

from test_texture_training_host import texture_dropout

pytestmark = pytest.mark.gpu
dev = "cuda"
TE = "texture_encoder"


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape, (a.shape, b.shape)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def _rms(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.sqrt(((a - b) ** 2).mean() / max((b ** 2).mean(), 1e-300)))


def _cos(a, b):
    a, b = np.asarray(a, np.float64).ravel(), np.asarray(b, np.float64).ravel()
    return float((a * b).sum() / max(np.linalg.norm(a) * np.linalg.norm(b), 1e-300))


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("B", [1, 5, 24, 32])
def test_fully_connected_param_grad_matches_float64(B):
    """rn_fully_connected_param_grad at e_tex_fc1's size (K = 199, N = 131072), slopes of both signs: gz, dW, db and dalpha
    within 1e-6 of their scale (measured on an H100 80GB HBM3: <= 2.7e-7), and two runs bit-identical (fixed-order sums over
    b)."""
    from rendernet_b200 import ops
    rng = np.random.default_rng(B)
    K, N = 199, 32 * 32 * 32 * 4
    x = rng.standard_normal((B, K)).astype(np.float32)
    gy = rng.standard_normal((B, N)).astype(np.float32)
    z = rng.standard_normal((B, N)).astype(np.float32)
    a = rng.uniform(-0.5, 0.5, N).astype(np.float32)
    z64, gy64 = z.astype(np.float64), gy.astype(np.float64)
    gz64 = np.where(z64 > 0, gy64, gy64 * a)
    want = dict(gz=gz64, dw=x.astype(np.float64).T @ gz64, db=gz64.sum(0), da=(gy64 * z64 * (z64 < 0)).sum(0))
    d = lambda t: torch.from_numpy(t).to(dev)                                      # noqa: E731
    runs = [[t.cpu().numpy() for t in ops.fully_connected_param_grad(d(x), d(gy), d(z), d(a), want_gz=True)] for _ in range(2)]
    errs = {k: _rel(g, want[k]) for k, g in zip(("gz", "dw", "db", "da"), runs[0])}
    same = all(np.array_equal(p.view(np.uint32), q.view(np.uint32)) for p, q in zip(*runs))
    print(f"fc param grad B={B}: " + ", ".join(f"{k} {e:.2e}" for k, e in errs.items()) + f"; bit-identical rerun {same}")
    assert max(errs.values()) < 1e-6 and same
    _, dw2, db2, da2 = ops.fully_connected_param_grad(d(x), d(gy), d(z), d(a))
    assert np.array_equal(dw2.cpu().numpy(), runs[0][1]) and np.array_equal(da2.cpu().numpy(), runs[0][3])


def test_fully_connected_param_grad_rejects_what_it_cannot_run():
    from rendernet_b200 import ops
    from rendernet_b200._lib import RenderNetCudaError
    z = lambda *s: torch.zeros(s, device=dev)                                       # noqa: E731
    with pytest.raises(RenderNetCudaError):
        ops.fully_connected_param_grad(z(33, 7), z(33, 64), z(33, 64), z(64))
    with pytest.raises(RenderNetCudaError):
        ops.fully_connected_param_grad(z(2, 7), z(2, 66), z(2, 66), z(66))


@pytest.mark.parametrize("B", [1, 24])
def test_prelu_grad_f32_matches_float64(B):
    """rn_prelu_grad_f32 at the decoder's shapes (C = 4 over B*32^3 and B*64^3, C = 8 over B*64^3): gz bit-identical to
    g * (z > 0 ? 1 : alpha), db and dalpha within 5e-6 of their scale (measured on an H100 80GB HBM3: <= 1.1e-6)."""
    from rendernet_b200 import ops
    rng = np.random.default_rng(100 + B)
    for S, C in ((32, 4), (64, 8), (64, 4)):
        z = rng.standard_normal((B, S, S, S, C)).astype(np.float32)
        gy = rng.standard_normal((B, S, S, S, C)).astype(np.float32)
        a = rng.uniform(-0.5, 0.5, C).astype(np.float32)
        gz, db, da = (t.cpu().numpy() for t in ops.prelu_grad_f32(torch.from_numpy(gy).to(dev), torch.from_numpy(z).to(dev),
                                                                    torch.from_numpy(a).to(dev)))
        want_gz = np.where(z > 0, gy, gy * a)
        g64, z64 = gy.astype(np.float64).reshape(-1, C), z.astype(np.float64).reshape(-1, C)
        e_b = _rel(db, np.where(z64 > 0, g64, g64 * a).sum(0))
        e_a = _rel(da, (g64 * z64 * (z64 < 0)).sum(0))
        print(f"prelu_grad_f32 B={B} {S}^3 x {C}: db {e_b:.2e}, dalpha {e_a:.2e}")
        assert np.array_equal(gz.view(np.uint32), want_gz.view(np.uint32))
        assert e_b < 5e-6 and e_a < 5e-6


THIN_CASES = [
    # layer, transposed, filter shape, input shape (per item), stride
    ("e_tex_conv0", True, (4, 4, 4, 4, 4), (32, 32, 32, 4), 1),
    ("e_tex_conv1", True, (4, 4, 4, 8, 4), (32, 32, 32, 4), 2),
    ("e_tex_conv2", False, (4, 4, 4, 8, 4), (64, 64, 64, 8), 1),
]


@pytest.mark.parametrize("B", [1, 24])
@pytest.mark.parametrize("layer,transposed,wshape,xshape,stride", THIN_CASES)
def test_decoder_thin_weight_gradients_match_float64(layer, transposed, wshape, xshape, stride, B):
    """(4,4) and (4,8) thin correlations on fp32 operands, driven as _decoder_weight_step drives them, vs float64 autograd (on
    the device) through the oracle's conv3d / conv3d_transpose.  Measured on an H100 80GB HBM3: <= 7.4e-7."""
    from rendernet_b200 import ops
    rng = np.random.default_rng(zlib.crc32(f"{layer}{B}".encode()))
    x = torch.from_numpy(rng.standard_normal((B,) + xshape).astype(np.float32)).to(dev)
    w = torch.tensor(rng.standard_normal(wshape) * 0.05, device=dev, requires_grad=True)
    s3 = (stride,) * 3
    y = orc.conv3d_transpose(x, w, None, s3, dtype=torch.float64) if transposed else orc.conv3d(x, w, None, s3, dtype=torch.float64)
    G = torch.from_numpy(rng.standard_normal(tuple(y.shape)).astype(np.float32)).to(dev)
    (y * G.double()).sum().backward()
    ks = wshape[:3]
    if transposed:
        pad = tuple(ops.same_pad_before(xshape[i] * stride, ks[i], stride) for i in range(3))
        got = ops.conv_weight_grad_direct(x, G, ks, s3, pad, Ca=wshape[4], Cb=wshape[3])
    else:
        pad = tuple(ops.same_pad_before(xshape[i], ks[i], stride) for i in range(3))
        got = ops.conv_weight_grad_direct(G, x, ks, s3, pad, Ca=wshape[4], Cb=wshape[3])
    e = _rel(got.permute(0, 1, 2, 4, 3).cpu().numpy(), w.grad.cpu().numpy())
    print(f"{layer} weight gradient B={B}: err {e:.2e}")
    assert e < 5e-6


@pytest.mark.parametrize("B", [1, 24])
def test_e_conv1_weight_gradient_matches_float64(B):
    """(8,5): e_conv1 of the Texture+Normal network (5^3 s2 over the 128^3 x 5 grid, fp32) from a 16-bit, loss-scaled g in both
    formats, vs float64 autograd on the device.  Measured on an H100 80GB HBM3: exact <= 1.5e-6, fast <= 3.0e-4."""
    from rendernet_b200 import ops
    rng = np.random.default_rng(200 + B)
    q = torch.from_numpy(rng.random((B, 128, 128, 128, 5), dtype=np.float32)).to(dev)
    w = torch.tensor(rng.standard_normal((5, 5, 5, 5, 8)) * 0.05, device=dev, requires_grad=True)
    y = orc.conv3d(q, w, None, (2, 2, 2), dtype=torch.float64)
    G = torch.from_numpy(rng.standard_normal(tuple(y.shape)).astype(np.float32)).to(dev)
    (y * G.double()).sum().backward()
    want = w.grad.cpu().numpy()
    pad = tuple(ops.same_pad_before(128, 5, 2) for _ in range(3))
    for fmt, tol in ((2, 5e-6), (0, 2e-3)):
        g16 = ops.cast_to_16(G * 64.0, fmt=fmt)
        got = ops.conv_weight_grad_direct(g16, q, (5, 5, 5), (2, 2, 2), pad, Ca=8, Cb=5, scale=1 / 64.0).permute(0, 1, 2, 4, 3)
        e = _rel(got.cpu().numpy(), want)
        print(f"e_conv1 (8,5) weight gradient B={B} fmt {fmt}: err {e:.2e}")
        assert e < tol


# ------------------------------------------------------------------------------------------------ whole network
def _scene(B, seed):
    rng = np.random.default_rng(seed)
    vox = ((rng.random((B, 64, 64, 64, 1)) < 0.25) * rng.uniform(0.5, 1.0, (B, 64, 64, 64, 1))).astype(np.float32)
    z = rng.standard_normal((B, 199)).astype(np.float32)
    poses = np.concatenate([orc.compute_pose_param(*p) for p in ((45.0, 30.0, 2.5), (130.0, 75.0, 3.0))[:B]]).astype(np.float32)
    t_img = rng.random((B, 512, 512, 3)).astype(np.float32)
    t_nrm = rng.random((B, 512, 512, 3)).astype(np.float32)
    return vox, z, poses, t_img, t_nrm


def _minv(poses):
    R, S = orc.rotation_around_grid_centroid(poses)
    return orc.inverse_total_matrix(R, S, 64, 128)


def _decoder(z, Wt, masks):
    """float64 texture decoder through the oracle's layers; masks {alpha name: z > 0} freezes the PReLU branches (None: plain)."""
    d = torch.float64

    def pr(t, name):
        a = Wt[f"{TE}/{name}/alpha"].double()
        if masks is None:
            return orc.prelu(t, a, d)
        return torch.where(torch.as_tensor(masks[f"{TE}/{name}/alpha"]).reshape(t.shape), t, a * t)
    h = pr(orc.fully_connected(z, Wt[f"{TE}/e_tex_fc1/fully_connected/weights"], Wt[f"{TE}/e_tex_fc1/fully_connected/biases"],
                               dtype=d), "e_tex_fc1").reshape(z.shape[0], 32, 32, 32, 4)
    for name, s, tr in (("e_tex_conv0", 1, True), ("e_tex_conv1", 2, True), ("e_tex_conv2", 1, False)):
        pre = f"{TE}/{name}/{'conv3d_transpose' if tr else 'conv3d'}"
        op = orc.conv3d_transpose if tr else orc.conv3d
        h = pr(op(h, Wt[pre + "/weights"], Wt[pre + "/biases"], (s, s, s), dtype=d), name)
    return h


def _oracle_step(vox, z, poses, Wt, t_img, t_nrm, keep, seed, masks=None, grads=True):
    """Oracle chain with the library's dropout masks (restated on the host) -> (loss, image, {name: dL/dvariable})."""
    from rendernet_b200 import ops
    from oracle.frozen_kinks import prelu_kinks

    def drop(call, t):
        m = ops.dropout_mask_host(t.numel(), keep, seed, call).reshape(tuple(t.shape)).astype(np.float32)
        return t * torch.from_numpy(m) / keep

    mt = torch.from_numpy(_minv(poses).astype(np.float64))
    with torch.set_grad_enabled(grads):
        tex = _decoder(torch.from_numpy(z.astype(np.float64)), Wt, masks)
        x = torch.cat([rc.resample(torch.from_numpy(vox.astype(np.float64)), mt, 128), rc.resample(tex, mt, 128)], -1).float()
        with contextlib.ExitStack() as stack:
            if masks is not None:
                stack.enter_context(prelu_kinks(Wt, masks=masks))
            if keep < 1.0:
                stack.enter_context(texture_dropout(Wt, drop))
            img, nrm = orc.rendernet_texture(x, Wt)
        loss = ((img - torch.from_numpy(t_img)) ** 2).mean() + ((nrm - torch.from_numpy(t_nrm)) ** 2).mean()
    if not grads:
        return float(loss), img.numpy(), None
    names = sorted(Wt)
    g = torch.autograd.grad(loss, [Wt[n] for n in names])
    return float(loss.detach()), img.detach().numpy(), {n: gi.numpy() for n, gi in zip(names, g)}


def _compare_gradients(tag, tr, grads, g_ref, g_f, cos_bar, ratio_bar, rms_bar, max_bar, dec_cos_bar=None):
    assert set(grads) == set(g_ref) and len(grads) == 186
    rows = sorted((_cos(grads[n].cpu().numpy(), g_ref[n]),
                   float(np.linalg.norm(grads[n].cpu().numpy()) / max(np.linalg.norm(g_ref[n]), 1e-30)), n) for n in g_ref)
    for c, r, n in rows[:4]:
        print(f"[{tag}]   lowest cosine: {n} cos {c:.5f} norm ratio {r:.4f}")
    errs = sorted(((_rms(grads[n].cpu().numpy(), g_f[n]), _rel(grads[n].cpu().numpy(), g_f[n]), n) for n in g_f), reverse=True)
    for e, m, n in errs[:4]:
        print(f"[{tag}]   largest frozen-kink error: {n} rel-rms {e:.2e} max {m:.2e}")
    dec = [e for e in errs if e[2].startswith(TE)]
    print(f"[{tag}] {len(rows)} variables: cosine min {rows[0][0]:.5f}, norm ratio {min(r for _, r, _ in rows):.4f}.."
          f"{max(r for _, r, _ in rows):.4f}; frozen kinks rel-rms max {errs[0][0]:.2e}, max-err max {max(e[1] for e in errs):.2e}"
          f" (decoder: {max(e[0] for e in dec):.2e} / {max(e[1] for e in dec):.2e})")
    dec_cos_bar = cos_bar if dec_cos_bar is None else dec_cos_bar
    assert all(c > (dec_cos_bar if n.startswith(TE) else cos_bar) for c, _, n in rows), rows[:3]
    assert all(abs(r - 1) < ratio_bar for _, r, _ in rows), [x for x in rows if abs(x[1] - 1) >= ratio_bar][:3]
    assert errs[0][0] < rms_bar and max(e[1] for e in errs) < max_bar, errs[:3]


def _weights(seed):
    return orc.init_texture_weights(seed=seed, alpha_range=(-0.1, 0.3), bias_jitter=0.02)


@pytest.mark.parametrize("precision", ["exact", "fast"])
def test_gradients_of_every_variable_match_oracle_autograd(precision):
    """Full size, B = 1, keep 0.75: loss and dL/d(variable) of all 186 variables (decoder included) vs torch.autograd through
    the oracle chain with the same dropout masks -- per variable cosine and norm ratio against the plain oracle, element by
    element against the frozen-kink oracle (decoder kinks included).
    Measured on an H100 80GB HBM3: exact -- cosine >= 0.99998 (lowest: e_tex_fc1), norm ratio 0.9996..1.0003, frozen kinks
    rel-rms <= 1.24e-4 and max <= 1.41e-4 (decoder 9.7e-5); fast -- render-net cosine >= 0.9985's bar, decoder cosine 0.99766
    (e_tex_fc1) .. 0.99997, norm ratio 0.9990..1.0022, frozen kinks rel-rms <= 1.9e-3, max <= 2.2e-3 (both at e_tex_fc1).  The
    fast decoder's lower cosine against the PLAIN oracle is kink flips, not arithmetic: the fast forward moves the render net's
    pre-activations by ~1e-3, units flip, and each FC column sees only the few grid cells its texel is resampled into, so a
    flip weighs more there than in a filter summed over the whole grid; with the kinks frozen the same gradients agree to 2e-3."""
    from rendernet_b200 import tfcompat as tf
    from rendernet_b200.training import TextureTrainer
    from oracle.frozen_kinks import tape_prelu_masks
    vox, z, poses, t_img, t_nrm = _scene(1, 31)
    W = _weights(32)
    tr = TextureTrainer(W, 1, precision=precision, keep_prob=0.75, seed=5)
    loss, grads = tr.loss_and_gradients(vox, z, poses, t_img, t_nrm)
    Wt = {n: torch.tensor(v, requires_grad=True) for n, v in W.items()}
    loss_ref, img_ref, g_ref = _oracle_step(vox, z, poses, Wt, t_img, t_nrm, 0.75, tr.dropout_seed(0))
    e_img = float(np.abs(tr.albedo.cpu().numpy() - img_ref).max())
    print(f"[{precision}] training-mode forward: image max-abs err {e_img:.2e}, loss {loss:.6f} vs {loss_ref:.6f}")
    assert e_img < (1e-3 if precision == "exact" else 5e-3)
    assert abs(loss - loss_ref) < (5e-5 if precision == "exact" else 1e-3) * loss_ref
    with tf.use_store(tr.store):
        masks = tape_prelu_masks(tr.tape)
    g_f = _oracle_step(vox, z, poses, Wt, t_img, t_nrm, 0.75, tr.dropout_seed(0), masks=masks)[2]
    if precision == "exact":
        _compare_gradients(precision, tr, grads, g_ref, g_f, 0.9999, 5e-3, 6e-4, 9e-4)
    else:
        _compare_gradients(precision, tr, grads, g_ref, g_f, 0.9985, 3e-2, 4e-3, 4.5e-3, dec_cos_bar=0.995)


def test_shipped_config_batch2_gradients_match_oracle_autograd():
    """config_RenderNet_texture.json's keep_prob 1.0, B = 2 with two poses, exact precision: the same comparison.  Measured on
    an H100 80GB HBM3: cosine >= 0.99998, norm ratio 0.9995..1.0000, frozen kinks rel-rms <= 1.29e-4, max <= 1.41e-4."""
    from rendernet_b200 import tfcompat as tf
    from rendernet_b200.training import TextureTrainer
    from oracle.frozen_kinks import tape_prelu_masks
    vox, z, poses, t_img, t_nrm = _scene(2, 41)
    W = _weights(42)
    tr = TextureTrainer(W, 2, precision="exact")
    assert tr.keep_prob == 1.0 and tr.e_eta == 1e-5 and tr.decay_steps == 100000
    loss, grads = tr.loss_and_gradients(vox, z, poses, t_img, t_nrm)
    Wt = {n: torch.tensor(v, requires_grad=True) for n, v in W.items()}
    loss_ref, _, g_ref = _oracle_step(vox, z, poses, Wt, t_img, t_nrm, 1.0, 0)
    print(f"[B=2 keep 1.0] loss {loss:.6f} vs {loss_ref:.6f}")
    assert abs(loss - loss_ref) < 5e-5 * loss_ref
    with tf.use_store(tr.store):
        masks = tape_prelu_masks(tr.tape)
    g_f = _oracle_step(vox, z, poses, Wt, t_img, t_nrm, 1.0, 0, masks=masks)[2]
    _compare_gradients("B=2 keep 1.0", tr, grads, g_ref, g_f, 0.9999, 5e-3, 6e-4, 9e-4)


def test_two_adam_steps_follow_the_oracle():
    """Two optimiser steps (exact, no dropout, PReLU slopes at 0 as initialised by the reference) vs the oracle trained by the
    same TF-Adam formulas: the loss before each step and after the second, and the direction of the total update of the FC,
    decoder and head tensors.  Measured on an H100 80GB HBM3: losses 0.167357 / 0.166882 / 0.166714 against the oracle's
    0.167357 / 0.166882 / 0.166714; update cosines >= 0.9996."""
    from rendernet_b200.training import TextureTrainer
    vox, z, poses, t_img, t_nrm = _scene(1, 51)
    W = orc.init_texture_weights(seed=52)
    lr, b1, b2, eps = 2e-5, 0.5, 0.999, 1e-8
    tr = TextureTrainer(W, 1, precision="exact", learning_rate=lr)
    losses = [tr.step(vox, z, poses, t_img, t_nrm), tr.step(vox, z, poses, t_img, t_nrm)]
    final = tr.loss_and_gradients(vox, z, poses, t_img, t_nrm, training=False)[0]
    Wt = {n: torch.tensor(v, requires_grad=True) for n, v in W.items()}
    m = {n: torch.zeros_like(v) for n, v in Wt.items()}
    v2 = {n: torch.zeros_like(v) for n, v in Wt.items()}
    ref = []
    for t in (1, 2):
        l, _, g = _oracle_step(vox, z, poses, Wt, t_img, t_nrm, 1.0, 0)
        ref.append(l)
        lr_t = lr * math.sqrt(1 - b2 ** t) / (1 - b1 ** t)
        with torch.no_grad():
            for n in Wt:
                gn = torch.from_numpy(g[n])
                m[n] += (gn - m[n]) * (1 - b1)
                v2[n] += (gn * gn - v2[n]) * (1 - b2)
                Wt[n] -= lr_t * m[n] / (v2[n].sqrt() + eps)
    ref_final = _oracle_step(vox, z, poses, Wt, t_img, t_nrm, 1.0, 0, grads=False)[0]
    print(f"loss trajectory: GPU {losses + [final]} vs oracle {ref + [ref_final]}")
    assert abs(losses[0] - ref[0]) < 1e-5 * ref[0]
    drop_ref, drop = ref[0] - ref_final, losses[0] - final
    assert drop_ref > 1e-4 * ref[0], "the step size of this test should move the loss"
    assert abs(losses[1] - ref[1]) < 0.1 * abs(ref[0] - ref[1]) + 1e-5 * ref[0]
    assert abs(drop - drop_ref) < 0.1 * drop_ref
    sd = tr.state_dict()
    assert tr.global_step == 2 and set(sd) == set(W)
    for n in (f"{TE}/e_tex_fc1/fully_connected/weights", f"{TE}/e_tex_fc1/alpha", f"{TE}/e_tex_conv1/conv3d_transpose/weights",
              f"{TE}/e_tex_conv2/conv3d/biases", "encoder/e_conv1/e_conv1/weights", "encoder/res2_3/con1_3X3/weights",
              "encoder/Image/e_conv9_1/conv2d_transpose/weights", "encoder/Normal/e_conv10_2/e_conv10_2/biases"):
        du, dr = sd[n] - W[n], Wt[n].detach().numpy() - W[n]
        c = _cos(du, dr)
        print(f"  update of {n}: cosine {c:.4f}, |update| mean {np.abs(du).mean():.2e} vs {np.abs(dr).mean():.2e}")
        assert c > 0.9


def test_trained_weights_render_in_the_engine():
    """state_dict() after a step (dropout on) loads into TextureRenderEngine; its exact-mode render of the updated weights
    matches the oracle forward on the same weights within the exact-mode bar (1e-3)."""
    from rendernet_b200.engine import TextureRenderEngine
    from rendernet_b200.training import TextureTrainer
    vox, z, poses, t_img, t_nrm = _scene(1, 61)
    tr = TextureTrainer(orc.init_texture_weights(seed=62), 1, precision="exact", keep_prob=0.75, learning_rate=1e-4)
    tr.step(vox, z, poses, t_img, t_nrm)
    sd = tr.state_dict()
    eng = TextureRenderEngine(sd, 1, precision="exact", use_graph=False)
    img, nrm = eng.render(vox, z, poses)
    ref_img, ref_nrm = orc.render_forward_texture(vox, z, poses, sd)
    e = max(float(np.abs(np.asarray(img) - ref_img.numpy()).max()), float(np.abs(np.asarray(nrm) - ref_nrm.numpy()).max()))
    print(f"engine render of the trained weights vs oracle: max-abs err {e:.2e}")
    assert e < 1e-3


def test_texture_trainer_recovers_from_overflow():
    """A fixed loss scale far too high: the step overflows, the scale is halved and the step redone with the same dropout
    masks; the applied gradient matches a trainer started at the scale it settled on."""
    from rendernet_b200.training import TextureTrainer
    vox, z, poses, t_img, t_nrm = _scene(1, 71)
    W = _weights(72)

    def stepped(scale):
        tr = TextureTrainer(W, 1, precision="exact", keep_prob=0.75, seed=4, learning_rate=1e-4, loss_scale=scale)
        tr.step(vox, z, poses, t_img, t_nrm)
        assert tr.global_step == 1
        return tr

    hot = stepped(2.0 ** 40)
    print(f"fixed loss scale 2^40 -> 2^{math.log2(hot.loss_scale):.0f}")
    assert hot.loss_scale < 2.0 ** 40
    ref = stepped(hot.loss_scale)
    assert ref.loss_scale == hot.loss_scale
    worst = max(_rel(hot.m[n].cpu().numpy(), ref.m[n].cpu().numpy()) for n in ref.m if float(ref.m[n].abs().max()) > 0)
    print(f"first moments vs a trainer started at the settled scale: max rel diff {worst:.2e}")
    assert worst < 1e-4
