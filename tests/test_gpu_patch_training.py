"""GPU tests of training on random patches (RenderNet_Shader.py:150-156, RenderNet_Texture_Face_Normal.py:164-179,
tools/model_util.py:77-161): the windowed input-stage kernels bit for bit against the whole-grid kernels they generalise, the
windowed resample5 backward against float64 device-cell autograd, and both trainers on patches against torch.autograd through
the oracle on the oracle-resampled grid sliced to the window (same dropout masks).  Errors are max |error| / max |reference|
unless stated otherwise."""
import math
import os

import numpy as np
import pytest
import torch

from oracle import rendernet_oracle as orc
from oracle import resample_cells as rc

import test_gpu_texture_training as ttt
import test_gpu_training as tst

pytestmark = pytest.mark.gpu
dev = "cuda"
N = 128
POSES = {"az90": (90.0, 60.0, 3.3), "turntable": (180.0, 90.0, 3.3), "generic": (45.0, 30.0, 2.5), "clipped": (300.0, 20.0, 1.8)}


def _poses(*names):
    return np.concatenate([orc.compute_pose_param(*POSES[n]) for n in names]).astype(np.float32)


def _minv(poses):
    R, S = orc.rotation_around_grid_centroid(poses)
    return orc.inverse_total_matrix(R, S, 64, N)


def _windows(P):
    """Both corners, both edges and an interior point for a P x P patch (and one non-square window)."""
    e = N - P
    return [(0, 0, P, P), (e, e, P, P), (0, e // 2 // 16 * 16, P, P), (e // 2 // 16 * 16, e, P, P), (e // 3, e // 5, P, P)] + (
        [(e // 4, 0, P, 2 * P)] if 2 * P <= N else [])


def _inputs(B, seed):
    rng = np.random.default_rng(seed)
    vox = ((rng.random((B, 64, 64, 64, 1)) < 0.25) * rng.uniform(0.5, 1.0, (B, 64, 64, 64, 1))).astype(np.float32)
    tex = rng.random((B, 64, 64, 64, 4)).astype(np.float32)
    return torch.from_numpy(vox).to(dev), torch.from_numpy(tex).to(dev)


def _bits(t):
    from rendernet_b200 import ops
    return (t.planes if isinstance(t, ops.Split16) else t).view(torch.int16)


# ------------------------------------------------------------------------------------------------ input-stage kernels
def test_windowed_resample_is_a_slice_of_the_whole_grid():
    """rn_resample_window_f32 == rn_resample_f32(transform=1)[:, y0:y0+ph, x0:x0+pw], bit for bit, C = 1 and 4, P = 16..128,
    corners, edges, interior, a non-square window; poses include an axis-aligned turntable frame (knife-edge coordinates)."""
    from rendernet_b200 import ops
    vox, tex = _inputs(3, 1)
    minv = torch.from_numpy(_minv(_poses("turntable", "generic", "clipped"))).to(dev)
    n = 0
    for v in (vox, tex):
        full = ops.resample(v, minv, N, True)
        for P in (16, 32, 64, 128):
            for y0, x0, ph, pw in _windows(P):
                got = ops.resample(v, minv, N, True, window=(y0, x0, ph, pw))
                assert tuple(got.shape) == (3, ph, pw, N, v.shape[-1])
                assert torch.equal(got, full[:, y0:y0 + ph, x0:x0 + pw]), (v.shape[-1], y0, x0, ph, pw)
                n += 1
    print(f"{n} windows bit-identical to slices of the whole grid")


@pytest.mark.parametrize("fmt", [0, 2])
def test_windowed_fused_econv1_equals_resample_then_direct_conv(fmt):
    """Both windowed fused kernels == windowed resample -> (concat) -> rn_conv3d_direct, bit for bit, in fp16 and fp16 hi/lo;
    with the full window they equal the existing whole-grid fused entries bit for bit."""
    from rendernet_b200 import ops
    rng = np.random.default_rng(fmt)
    vox, tex = _inputs(2, 2)
    minv = torch.from_numpy(_minv(_poses("turntable", "generic"))).to(dev)
    w1 = torch.from_numpy((rng.standard_normal((5, 5, 5, 1, 8)) * 0.2).astype(np.float32)).to(dev)
    w5 = torch.from_numpy((rng.standard_normal((5, 5, 5, 5, 8)) * 0.1).astype(np.float32)).to(dev)
    b = torch.from_numpy(rng.standard_normal(8).astype(np.float32) * 0.1).to(dev)
    a = torch.from_numpy(rng.uniform(-0.2, 0.3, 8).astype(np.float32)).to(dev)
    for alpha in (a, None):
        whole1 = ops.resample_conv1(vox, minv, N, w1, b, alpha, fmt=fmt)
        whole5 = ops.resample5_conv1(vox, tex, minv, N, w5, b, alpha, fmt=fmt)
        assert torch.equal(_bits(ops.resample_conv1(vox, minv, N, w1, b, alpha, fmt=fmt, window=(0, 0, N, N))), _bits(whole1))
        assert torch.equal(_bits(ops.resample5_conv1(vox, tex, minv, N, w5, b, alpha, fmt=fmt, window=(0, 0, N, N))), _bits(whole5))
        for P in (16, 32, 64, 128):
            for win in _windows(P):
                g = ops.resample(vox, minv, N, True, window=win)
                got1 = ops.resample_conv1(vox, minv, N, w1, b, alpha, fmt=fmt, window=win)
                want1 = ops.conv3d_direct(g, w1, b, alpha, (2, 2, 2), fmt=fmt)
                assert got1.shape == want1.shape == (2, win[2] // 2, win[3] // 2, N // 2, 8)
                assert torch.equal(_bits(got1), _bits(want1)), ("resample_conv1", win)
                x5 = ops.concat_channels(g, ops.resample(tex, minv, N, True, window=win))
                got5 = ops.resample5_conv1(vox, tex, minv, N, w5, b, alpha, fmt=fmt, window=win)
                assert torch.equal(_bits(got5), _bits(ops.conv3d_direct(x5, w5, b, alpha, (2, 2, 2), fmt=fmt))), ("resample5", win)


def test_windowed_resample5_backward_matches_float64_and_the_whole_grid_kernel():
    """rn_resample5_backward_window_f32 vs autograd through the float64 device-cell resampler restricted to the window (bars of
    the whole-grid kernel: dvox / dtex 1e-6, dM^-1 4e-6 of scale), and vs rn_resample5_backward_f32 fed the window's gradient
    zero-padded to the whole grid (same scatter; dM^-1 summed in another order)."""
    from rendernet_b200 import ops
    names = ("turntable", "generic")
    B = len(names)
    minv = _minv(_poses(*names))
    vox_d, tex_d = _inputs(B, 3)
    vox, tex = vox_d.cpu().numpy(), tex_d.cpu().numpy()
    vt = torch.tensor(vox.astype(np.float64), requires_grad=True)
    tt = torch.tensor(tex.astype(np.float64), requires_grad=True)
    mt = torch.tensor(minv.astype(np.float64), requires_grad=True)
    full = torch.cat([rc.resample(vt, mt, N), rc.resample(tt, mt, N)], -1)
    md = torch.from_numpy(minv).to(dev)
    for k, (y0, x0, ph, pw) in enumerate([(48, 32, 32, 32), (0, 64, 64, 64), (112, 0, 16, 128)]):
        G = np.random.default_rng(k).standard_normal((B, ph, pw, N, 5)).astype(np.float32)
        ref = torch.autograd.grad((full[:, y0:y0 + ph, x0:x0 + pw] * torch.from_numpy(G.astype(np.float64))).sum(), (vt, tt, mt),
                                  retain_graph=True)
        Gd = torch.from_numpy(G).to(dev)
        got = [t.cpu().numpy() for t in ops.resample5_backward(vox_d, tex_d, md, Gd, window=(y0, x0, ph, pw))]
        Gf = torch.zeros((B, N, N, N, 5), device=dev)
        Gf[:, y0:y0 + ph, x0:x0 + pw] = Gd
        whole = [t.cpu().numpy() for t in ops.resample5_backward(vox_d, tex_d, md, Gf)]
        for b in range(B):
            e = [tst._rel(got[i][b], ref[i][b].numpy()) for i in range(3)]
            w = [tst._rel(got[i][b], whole[i][b]) for i in range(3)]
            print(f"window {(y0, x0, ph, pw)} {names[b]}: vs float64 dvox {e[0]:.2e} dtex {e[1]:.2e} dMinv {e[2]:.2e}; "
                  f"vs whole-grid kernel {w[0]:.2e} {w[1]:.2e} {w[2]:.2e}")
            assert e[0] < 1e-6 and e[1] < 1e-6 and e[2] < 4e-6
            assert w[0] < 1e-6 and w[1] < 1e-6 and w[2] < 4e-6
    only = ops.resample5_backward(vox_d, tex_d, md, torch.zeros((B, 32, 32, N, 5), device=dev), want_dvox=False, want_dminv=False,
                                  window=(0, 0, 32, 32))
    assert only[0] is None and only[2] is None and float(only[1].abs().max()) == 0.0


# ------------------------------------------------------------------------------------------------ Shader trainer on patches
def _shader_scene(golden_dir, B=2):
    bv = np.load(os.path.join(golden_dir, "binvox.npz"))
    chair = np.unpackbits(bv["chair_bits"]).reshape(1, 64, 64, 64, 1).astype(np.float32)
    vox = np.concatenate([chair, chair[:, ::-1].copy()], 0)[:B]
    poses = np.concatenate([orc.compute_pose_param(250.0, 60.0, 3.3), orc.compute_pose_param(40.0, 75.0, 3.0)])[:B].astype(np.float32)
    grid = orc.transform_voxel_to_match_image(orc.rotation_resampling(vox, poses)).astype(np.float32)
    sil = (grid[..., 0].sum(axis=3) > 0.5).astype(np.float32)                                       # [B,128,128]
    target = np.repeat(np.repeat(sil, 4, 1), 4, 2)[..., None] * np.array([0.9, 0.6, 0.3], np.float32)
    return vox, poses, grid, np.ascontiguousarray(target, np.float32)


def _crop(grid, target, origin, P):
    y0, x0 = origin
    return (np.ascontiguousarray(grid[:, y0:y0 + P, x0:x0 + P]),
            np.ascontiguousarray(target[:, 4 * y0:4 * (y0 + P), 4 * x0:4 * (x0 + P)]))


SHADER_ORIGIN = {32: (48, 40), 64: (32, 40)}


@pytest.mark.parametrize("P", [32, 64])
@pytest.mark.parametrize("precision", ["exact", "fast"])
def test_shader_patch_gradients_match_oracle_autograd(golden_dir, precision, P):
    """B = 2, keep 0.75, a fixed interior origin: loss, image and the gradients of all 166 variables vs torch.autograd through the
    oracle on the oracle-resampled grid sliced to the window, with the same dropout masks; test_gpu_training.py's full-size
    bars, element-wise with the kinks frozen at the device's."""
    from rendernet_b200.training import ShaderTrainer
    from oracle.frozen_kinks import kink_flips, prelu_kinks, tape_prelu_masks
    vox, poses, grid, target = _shader_scene(golden_dir)
    origin = SHADER_ORIGIN[P]
    g_p, t_p = _crop(grid, target, origin, P)
    W = orc.init_shader_weights(seed=1, alpha_range=(-0.1, 0.3), bias_jitter=0.02)
    tr = ShaderTrainer(W, 2, precision=precision, keep_prob=0.75, seed=5)
    loss, grads = tr.loss_and_gradients(vox, poses, target, patch_size=P, origin=origin)
    assert tr.last_crop == (origin, P) and tuple(tr.img.shape) == (2, 4 * P, 4 * P, 3)
    Wt = {n: torch.tensor(v, requires_grad=True) for n, v in W.items()}
    signs = {}
    with prelu_kinks(Wt, record=signs):
        loss_ref, img_ref, g_ref = tst._oracle_step(g_p, Wt, t_p, 0.75, tr.dropout_seed(0))
    e_img = float(np.abs(tr.img.cpu().numpy() - img_ref).max())
    print(f"[{precision} P={P}] image max-abs err {e_img:.2e}, loss {loss:.6f} vs {loss_ref:.6f}")
    assert e_img < (1e-3 if precision == "exact" else 5e-3)
    assert abs(loss - loss_ref) < (5e-5 if precision == "exact" else 1e-3) * loss_ref
    assert set(grads) == set(g_ref) and len(grads) == 166
    rows = sorted((tst._cos(grads[n].cpu().numpy(), g_ref[n]),
                   float(np.linalg.norm(grads[n].cpu().numpy()) / max(np.linalg.norm(g_ref[n]), 1e-30)), n) for n in g_ref)
    masks = tape_prelu_masks(tr.tape)
    flips, units = kink_flips(masks, signs)
    with prelu_kinks(Wt, masks=masks):
        g_f = tst._oracle_step(g_p, Wt, t_p, 0.75, tr.dropout_seed(0))[2]
    errs = sorted(((tst._rms(grads[n].cpu().numpy(), g_f[n]), tst._rel(grads[n].cpu().numpy(), g_f[n]), n) for n in g_f), reverse=True)
    print(f"[{precision} P={P}] cosine min {rows[0][0]:.5f} ({rows[0][2]}), norm ratio {min(r for _, r, _ in rows):.4f}.."
          f"{max(r for _, r, _ in rows):.4f}; {flips} of {units} units flipped; frozen kinks rel-rms max {errs[0][0]:.2e} "
          f"({errs[0][2]}), max-err max {max(e[1] for e in errs):.2e}")
    cos_bar, ratio_bar, rms_bar, max_bar = (0.9999, 5e-3, 6e-4, 9e-4) if precision == "exact" else (0.9985, 3e-2, 4e-3, 4.5e-3)
    assert rows[0][0] > cos_bar, rows[:3]
    assert all(abs(r - 1) < ratio_bar for _, r, _ in rows)
    assert errs[0][0] < rms_bar and max(e[1] for e in errs) < max_bar, errs[:3]


def test_shader_patch_greyscale_bce_matches_oracle_autograd(golden_dir):
    """Greyscale BCE (sum over the patch, mean over the batch; RenderNet_Shader.py:158-161) at P = 32, B = 2, exact."""
    from rendernet_b200.training import ShaderTrainer
    vox, poses, grid, _ = _shader_scene(golden_dir)
    sil = (grid[..., 0].sum(axis=3) > 0.5).astype(np.float32)
    target = np.ascontiguousarray(np.repeat(np.repeat(sil, 4, 1), 4, 2)[..., None])
    origin, P = (48, 40), 32
    g_p, t_p = _crop(grid, target, origin, P)
    W = orc.init_shader_weights(seed=3, is_greyscale=True, alpha_range=(-0.05, 0.25), bias_jitter=0.02)
    tr = ShaderTrainer(W, 2, precision="exact", is_greyscale=True)
    loss, grads = tr.loss_and_gradients(vox, poses, target, patch_size=P, origin=origin)
    Wt = {n: torch.tensor(v, requires_grad=True) for n, v in W.items()}
    img = orc.rendernet_shader(torch.from_numpy(g_p), Wt)
    t = torch.from_numpy(t_p)
    ref = (-(t * torch.log(1e-6 + img) + (1 - t) * torch.log(1e-6 + 1 - img)).sum(dim=(1, 2, 3))).mean()
    g_ref = dict(zip(sorted(Wt), torch.autograd.grad(ref, [Wt[n] for n in sorted(Wt)])))
    worst = min((tst._cos(grads[n].cpu().numpy(), g_ref[n].numpy()), n) for n in g_ref)
    ratios = [float(np.linalg.norm(grads[n].cpu().numpy()) / max(np.linalg.norm(g_ref[n].numpy()), 1e-30)) for n in g_ref]
    print(f"[greyscale BCE P=32] loss {loss:.4f} vs {float(ref):.4f}; lowest cosine {worst[0]:.5f} ({worst[1]}), "
          f"norm ratio {min(ratios):.4f}..{max(ratios):.4f}")
    assert abs(loss - float(ref)) < 5e-5 * float(ref)
    assert set(grads) == set(g_ref) and worst[0] > 0.9995 and all(abs(r - 1) < 1e-2 for r in ratios)


# ------------------------------------------------------------------------------------------------ Texture trainer on patches
def _texture_oracle_step(vox, z, poses, Wt, t_img, t_nrm, keep, seed, origin, P, masks=None):
    """test_gpu_texture_training's oracle chain (float64 decoder -> device-cell resampler -> concat) sliced to the window before
    rendernet_texture; targets cropped at 4x the origin."""
    import contextlib
    from rendernet_b200 import ops
    from oracle.frozen_kinks import prelu_kinks

    def drop(call, t):
        m = ops.dropout_mask_host(t.numel(), keep, seed, call).reshape(tuple(t.shape)).astype(np.float32)
        return t * torch.from_numpy(m) / keep
    y0, x0 = origin
    mt = torch.from_numpy(_minv(poses).astype(np.float64))
    tex = ttt._decoder(torch.from_numpy(z.astype(np.float64)), Wt, masks)
    x = torch.cat([rc.resample(torch.from_numpy(vox.astype(np.float64)), mt, N), rc.resample(tex, mt, N)], -1).float()
    x = x[:, y0:y0 + P, x0:x0 + P]
    with contextlib.ExitStack() as stack:
        if masks is not None:
            stack.enter_context(prelu_kinks(Wt, masks=masks))
        if keep < 1.0:
            stack.enter_context(ttt.texture_dropout(Wt, drop))
        img, nrm = orc.rendernet_texture(x, Wt)
    ti = torch.from_numpy(t_img[:, 4 * y0:4 * (y0 + P), 4 * x0:4 * (x0 + P)].copy())
    tn = torch.from_numpy(t_nrm[:, 4 * y0:4 * (y0 + P), 4 * x0:4 * (x0 + P)].copy())
    loss = ((img - ti) ** 2).mean() + ((nrm - tn) ** 2).mean()
    names = sorted(Wt)
    g = torch.autograd.grad(loss, [Wt[n] for n in names])
    return float(loss.detach()), img.detach().numpy(), {n: gi.numpy() for n, gi in zip(names, g)}


@pytest.mark.parametrize("P", [32, 64])
@pytest.mark.parametrize("precision", ["exact", "fast"])
def test_texture_patch_gradients_match_oracle_autograd(precision, P):
    """B = 1, keep 0.75, fixed interior origin: all 186 gradients (decoder included: dL/d(texture volume) comes from the window
    only) vs the oracle chain sliced to the window, at test_gpu_texture_training.py's bars."""
    from rendernet_b200 import tfcompat as tf
    from rendernet_b200.training import TextureTrainer
    from oracle.frozen_kinks import tape_prelu_masks
    vox, z, poses, t_img, t_nrm = ttt._scene(1, 31)
    origin = {32: (40, 56), 64: (32, 16)}[P]
    W = ttt._weights(32)
    tr = TextureTrainer(W, 1, precision=precision, keep_prob=0.75, seed=5)
    loss, grads = tr.loss_and_gradients(vox, z, poses, t_img, t_nrm, patch_size=P, origin=origin)
    assert tr.last_crop == (origin, P) and tuple(tr.albedo.shape) == (1, 4 * P, 4 * P, 3)
    Wt = {n: torch.tensor(v, requires_grad=True) for n, v in W.items()}
    loss_ref, img_ref, g_ref = _texture_oracle_step(vox, z, poses, Wt, t_img, t_nrm, 0.75, tr.dropout_seed(0), origin, P)
    e_img = float(np.abs(tr.albedo.cpu().numpy() - img_ref).max())
    print(f"[{precision} P={P}] image max-abs err {e_img:.2e}, loss {loss:.6f} vs {loss_ref:.6f}")
    assert e_img < (1e-3 if precision == "exact" else 5e-3)
    assert abs(loss - loss_ref) < (5e-5 if precision == "exact" else 1e-3) * loss_ref
    with tf.use_store(tr.store):
        masks = tape_prelu_masks(tr.tape)
    g_f = _texture_oracle_step(vox, z, poses, Wt, t_img, t_nrm, 0.75, tr.dropout_seed(0), origin, P, masks=masks)[2]
    if precision == "exact":
        ttt._compare_gradients(f"{precision} P={P}", tr, grads, g_ref, g_f, 0.9999, 5e-3, 6e-4, 9e-4)
    else:
        ttt._compare_gradients(f"{precision} P={P}", tr, grads, g_ref, g_f, 0.9985, 3e-2, 4e-3, 4.5e-3, dec_cos_bar=0.995)


# ------------------------------------------------------------------------------------------------ whole-frame equivalence
def _same_step(got, want, what):
    """The loss and the weight gradients are sums over fp32 / fp64 atomics, so two runs of one path agree to the last bits only:
    rel 1e-12 for the loss, 1e-5 of each gradient's scale (its run-to-run noise is ~1e-7)."""
    (lg, gg), (lw, gw) = got, want
    assert abs(lg - lw) <= 1e-12 * abs(lw), (what, lg, lw)
    assert set(gg) == set(gw)
    worst = max(tst._rel(gg[n].cpu().numpy(), gw[n].cpu().numpy()) for n in gw)
    print(f"{what}: loss {lg!r} vs {lw!r}, gradients max rel diff {worst:.2e}")
    assert worst < 1e-5, (what, worst)


def test_patch_size_new_size_is_the_whole_frame_path(golden_dir):
    """patch_size = new_size takes the whole-frame path, for both trainers: no window on the tape, a bit-identical image, and
    the loss and gradients of a call without patch_size (within the atomics' run-to-run noise)."""
    from rendernet_b200.training import ShaderTrainer, TextureTrainer
    vox, poses, _, target = _shader_scene(golden_dir, B=1)
    W = orc.init_shader_weights(seed=4, alpha_range=(-0.1, 0.3))
    a, b = (ShaderTrainer(W, 1, precision="fast", keep_prob=0.75, seed=2) for _ in range(2))
    ra = a.loss_and_gradients(vox, poses, target)
    rb = b.loss_and_gradients(vox, poses, target, patch_size=N)
    assert b.last_crop is None and all(r.get("window") is None for r in b.tape)
    assert torch.equal(a.img, b.img)
    _same_step(rb, ra, "Shader, patch_size = 128 vs whole frame")
    tv, tz, tp, ti, tn = ttt._scene(1, 31)
    Wt = ttt._weights(32)
    c, d = (TextureTrainer(Wt, 1, precision="exact", keep_prob=0.75, seed=2) for _ in range(2))
    rc_ = c.loss_and_gradients(tv, tz, tp, ti, tn)
    rd = d.loss_and_gradients(tv, tz, tp, ti, tn, patch_size=N)
    assert d.last_crop is None and all(r.get("window") is None for r in d.tape)
    assert torch.equal(c.albedo, d.albedo) and torch.equal(c.normal, d.normal)
    _same_step(rd, rc_, "Texture+Normal, patch_size = 128 vs whole frame")


def test_validation_ignores_the_patch_size(golden_dir):
    from rendernet_b200.training import ShaderTrainer
    vox, poses, _, target = _shader_scene(golden_dir, B=1)
    tr = ShaderTrainer(orc.init_shader_weights(seed=6), 1, precision="fast")
    full = tr.loss_and_gradients(vox, poses, target, training=False)
    img = tr.img.clone()
    val = tr.loss_and_gradients(vox, poses, target, training=False, patch_size=32)
    assert tuple(tr.img.shape) == (1, 512, 512, 3) and torch.equal(tr.img, img) and tr.last_crop is None
    _same_step(val, full, "validation with patch_size = 32 vs without")


# ------------------------------------------------------------------------------------------------ optimisation
def test_two_adam_steps_on_drawn_patches_follow_the_oracle(golden_dir):
    """Two Shader steps at P = 64 on the trainer's own drawn origins (exact, no dropout) vs the oracle trained by the same
    TF-Adam formulas on the same patches: the loss before each step, and the loss of the first patch after the second step."""
    from rendernet_b200.training import ShaderTrainer
    vox, poses, grid, target = _shader_scene(golden_dir, B=1)
    W = orc.init_shader_weights(seed=2, alpha_range=(0.0, 0.0))
    lr, b1, b2, eps, P = 2e-5, 0.5, 0.999, 1e-8, 64
    tr = ShaderTrainer(W, 1, precision="exact", learning_rate=lr, seed=9)
    origins = [tr.crop_origin(0, P), tr.crop_origin(1, P)]
    losses = []
    for s in range(2):
        losses.append(tr.step(vox, poses, target, patch_size=P))
        assert tr.last_crop == (origins[s], P)
    final = tr.loss_and_gradients(vox, poses, target, patch_size=P, origin=origins[0])[0]
    Wt = {n: torch.tensor(v, requires_grad=True) for n, v in W.items()}
    m = {n: torch.zeros_like(v) for n, v in Wt.items()}
    v2 = {n: torch.zeros_like(v) for n, v in Wt.items()}
    ref = []
    for t in (1, 2):
        g_p, t_p = _crop(grid, target, origins[t - 1], P)
        l, _, g = tst._oracle_step(g_p, Wt, t_p, 1.0, 0)
        ref.append(l)
        lr_t = lr * math.sqrt(1 - b2 ** t) / (1 - b1 ** t)
        with torch.no_grad():
            for n in Wt:
                gn = torch.from_numpy(g[n])
                m[n] += (gn - m[n]) * (1 - b1)
                v2[n] += (gn * gn - v2[n]) * (1 - b2)
                Wt[n] -= lr_t * m[n] / (v2[n].sqrt() + eps)
    g0, t0 = _crop(grid, target, origins[0], P)
    ref_final = tst._oracle_step(g0, Wt, t0, 1.0, 0)[0]
    print(f"origins {origins}; loss trajectory: GPU {losses + [final]} vs oracle {ref + [ref_final]}")
    assert abs(losses[0] - ref[0]) < 1e-5 * ref[0]
    assert abs(losses[1] - ref[1]) < 1e-4 * ref[1]
    drop_ref, drop = ref[0] - ref_final, losses[0] - final
    assert drop_ref > 0, "the step size of this test should move the loss"
    assert abs(drop - drop_ref) < 0.1 * drop_ref


def test_overflow_retry_keeps_the_crop(golden_dir):
    """A fixed loss scale far too high on a drawn patch: the step overflows and is redone at a lower scale on the same patch
    (the applied moments match a trainer started at the settled scale, which draws the same origin)."""
    from rendernet_b200.training import ShaderTrainer
    vox, poses, _, target = _shader_scene(golden_dir, B=1)
    W = orc.init_shader_weights(seed=7, alpha_range=(-0.1, 0.3))

    def stepped(scale):
        tr = ShaderTrainer(W, 1, precision="exact", keep_prob=0.75, seed=4, learning_rate=1e-4, loss_scale=scale)
        tr.step(vox, poses, target, patch_size=32)
        assert tr.global_step == 1 and tr.last_crop == (tr.crop_origin(0, 32), 32)
        return tr

    hot = stepped(2.0 ** 30)
    print(f"fixed loss scale 2^30 -> 2^{math.log2(hot.loss_scale):.0f}, crop {hot.last_crop}")
    assert hot.loss_scale < 2.0 ** 30
    ref = stepped(hot.loss_scale)
    worst = max(tst._rel(hot.m[n].cpu().numpy(), ref.m[n].cpu().numpy()) for n in ref.m if float(ref.m[n].abs().max()) > 0)
    assert worst < 1e-4


@pytest.mark.parametrize("precision", ["exact", "fast"])
def test_texture_b24_p64_step_is_finite(precision):
    """The configuration the reference ships (batch_size 24) at the later-epoch patch size: one step runs and every gradient
    is finite."""
    from rendernet_b200.training import TextureTrainer
    rng = np.random.default_rng(24)
    B = 24
    vox = ((rng.random((B, 64, 64, 64, 1)) < 0.25) * 1.0).astype(np.float32)
    z = rng.standard_normal((B, 199)).astype(np.float32)
    poses = np.concatenate([orc.compute_pose_param(15.0 * i, 30.0 + 2 * i, 3.0) for i in range(B)]).astype(np.float32)
    t = rng.random((B, 512, 512, 3)).astype(np.float32)
    tr = TextureTrainer(None, B, precision=precision)
    loss, grads = tr.loss_and_gradients(vox, z, poses, t, t, patch_size=64)
    assert math.isfinite(loss) and len(grads) == 186
    assert all(bool(torch.isfinite(g).all()) for g in grads.values())
    tr.step(vox, z, poses, t, t, patch_size=64)
    assert tr.global_step == 1 and tr.last_crop[1] == 64
