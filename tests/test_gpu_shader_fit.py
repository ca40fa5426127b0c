"""GPU tests of the Shader pose / light fit: rn_phong_composite_loss_grad (the demo's composite, differentiated), the per-item
losses of rn_image_loss_grad_items, shader_fit_gradients through the whole Shader network, ShaderPoseFit.run and the command line.

References are float64: the composite through oracle/phong_np.py (at the kernel's fp32 mask value), the network through the
oracle Shader with the device's PReLU kinks frozen (oracle/frozen_kinks.py) and the device-cell resampler
(oracle/resample_cells.py).  Errors are max |error| / max |reference| unless stated otherwise."""
import json
import math
import os

import numpy as np
import pytest
import torch

from oracle import phong_np as pn
from oracle import rendernet_oracle as orc
from oracle import resample_cells as rc

pytestmark = pytest.mark.gpu
dev = "cuda"
D64 = torch.float64


def _d(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _rel(got, want):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert got.shape == want.shape, (got.shape, want.shape)
    return float(np.abs(got - want).max() / max(np.abs(want).max(), 1e-30))


def _normals(B, H, W, seed, white):
    """Random normal maps plus pixels on n.l = 0 and on u = L (d = 1: the diffuse clip's upper bound at k_d = 1) for the light
    (0, 0, 2), exact 0 / 1 components, and a band of pixels on the mask's transition (|s| < 15).  No pixel is (0.5, 0.5, 0.5)."""
    rng = np.random.default_rng(seed)
    n = rng.random((B, H, W, 3)).astype(np.float32)
    n[:, 0, :8] = [0.75, 0.5, 0.5]                     # v = (0.25, 0, 0): v.L = 0 exactly
    n[:, 0, 8:16] = [0.5, 0.25, 0.5]
    n[:, 1, :8] = [0.5, 0.5, 0.75]                     # v / |v| = L: d = 1
    n[:, 1, 8:16] = [1.0, 0.0, 1.0]
    n[:, 2, :8] = [0.0, 1.0, 0.25]
    dirs = rng.random((B, 8, W, 3)) + 0.05
    dirs /= np.linalg.norm(dirs, axis=-1, keepdims=True)
    if white:                                          # |1 - n| around 80 / 255
        n[:, 8:16] = (1.0 - dirs * rng.uniform(0.27, 0.36, (B, 8, W, 1))).astype(np.float32)
    else:                                              # |n| around 150 / 255
        n[:, 8:16] = (dirs * rng.uniform(0.55, 0.63, (B, 8, W, 1))).astype(np.float32)
    return n


def _lights(B, seed):
    rng = np.random.default_rng(seed)
    ld = np.concatenate([[[0.0, 0.0, 2.0]], 1.7 * rng.standard_normal((B - 1, 3))]).astype(np.float32)[:B]
    return ld, rng.uniform(0.6, 1.1, (B, 3)).astype(np.float32)


def _mask32(n, white):
    """The fp32 mask phong_pixel evaluates, emulated in float64 with one rounding per operation (|a|^2 as fmaf(c, c, .) as nvcc
    contracts it, then sqrtf, 255 x - thr as one fmaf, expf, 1 / (1 + e)).  Agrees with the device to about an ulp of expf."""
    a = (1.0 - n.astype(np.float64)).astype(np.float32) if white else n
    a = a.astype(np.float64)
    f32 = lambda x: np.asarray(x, np.float64).astype(np.float32).astype(np.float64)   # noqa: E731
    s = f32(a[..., 0] * a[..., 0])
    s = f32(a[..., 1] * a[..., 1] + s)
    s = f32(a[..., 2] * a[..., 2] + s)
    arg = f32(255.0 * f32(np.sqrt(s)) - (80.0 if white else 150.0))
    with np.errstate(over="ignore"):                   # expf(-arg) overflows to inf where the mask is 0, as on the device
        return f32(1.0 / f32(1.0 + f32(np.exp(-arg))))[..., None]


def _transition(n, white):
    return np.abs(pn.np_mask_arg(torch.from_numpy(n).double(), white).numpy()[..., 0]) < 15


# ----------------------------------------------------------------------------------------- the loss kernel
@pytest.mark.parametrize("white", [False, True])
@pytest.mark.parametrize("mask", [False, True])
def test_composite_loss_is_zero_at_the_kernels_own_image(white, mask):
    """Target = rn_phong_composite's own image, lights of several lengths: loss 0, d_img 0 and d_light 0 exactly, so the image the
    loss measures is rn_phong_composite's, bit for bit (any differing value would leave a positive squared residual)."""
    from rendernet_b200 import ops
    B = 4
    n = _d(_normals(B, 64, 96, 1, white))
    ld, lc = _lights(B, 2)
    ld[2] *= 0.01
    ld, lc = _d(ld), _d(lc)
    for ambient, kd in ((0.1, 0.9), (0.0, 1.0)):
        img = ops.phong_composite(n, ld, lc, ambient, kd, background_white=white, with_mask=mask)
        loss, di, dl = ops.phong_composite_loss_grad(n, img, ld, lc, ambient, kd, white, mask)
        assert (loss == 0).all(), loss
        assert (di == 0).all(), int((di != 0).sum())
        assert (dl == 0).all(), dl


@pytest.mark.parametrize("white,mask,ambient,kd", [(False, True, 0.1, 0.9), (True, True, 0.1, 0.9), (False, False, 0.0, 1.0),
                                                   (True, True, 0.0, 1.0)])
def test_composite_loss_grad_matches_float64_autograd(white, mask, ambient, kd):
    """Loss, d_img and d_light against float64 autograd of oracle/phong_np.py at the kernel's fp32 mask value, on pixels that
    include n.l = 0, both diffuse clip bounds (d = 0 and d = 1 at k_d = 1), the composite's clips and the mask's transition.
    Bars: loss 1e-6 relative, d_img 1e-6 of its scale, d_light 1e-5 of its scale.  On the transition band (|s| < 15 for the
    mask sigmoid(s)) d_img has its own bar, 1e-5: the oracle's mask value is emulated, not read from the device, and one ulp of
    the device's expf there moves the composite by ~m (1 - m) ulp and its 255-fold derivative with it.  Measured on an H100 80GB
    HBM3: loss <= 3.0e-8, d_img <= 1.7e-7 off the band and <= 7.5e-6 on it, d_light <= 3.0e-7."""
    from rendernet_b200 import ops
    B, H, W = 3, 64, 64
    n = _normals(B, H, W, 3 + white + 2 * mask, white)
    ld, lc = _lights(B, 4)
    col = np.ones_like(lc) if kd == 1.0 else lc
    tgt = np.random.default_rng(5).random((B, H, W, 3)).astype(np.float32)
    loss, di, dl = ops.phong_composite_loss_grad(_d(n), _d(tgt), _d(ld), _d(col), ambient, kd, white, mask)
    nt = torch.tensor(n.astype(np.float64), requires_grad=True)
    lt = torch.tensor(ld.astype(np.float64), requires_grad=True)
    mv = torch.from_numpy(_mask32(n, white)) if mask else None
    ref = pn.fit_loss(nt, torch.from_numpy(tgt).double(), lt, torch.from_numpy(col).double(), ambient, kd, white, mask, mv)
    ref.sum().backward()
    edge = _transition(n, white) if mask else np.zeros(n.shape[:3], bool)
    di, gref = di.cpu().numpy().astype(np.float64), nt.grad.numpy()
    scale = np.abs(gref).max()
    e_loss = float((np.abs(loss.cpu().numpy() - ref.detach().numpy()) / ref.detach().numpy()).max())
    e_img = float(np.abs(di - gref)[~edge].max() / scale)
    e_edge = float(np.abs(di - gref)[edge].max() / scale) if edge.any() else 0.0
    e_light = _rel(dl.cpu().numpy(), lt.grad.numpy())
    on_kink = int(((n[..., 0] == 0.75) & (n[..., 1] == 0.5)).sum())
    print(f"white={white} mask={mask} ambient={ambient} k_d={kd}: loss {e_loss:.2e}, d_img {e_img:.2e} "
          f"({int(edge.sum())} transition pixels {e_edge:.2e}), d_light {e_light:.2e}; {on_kink} pixels on n.l = 0")
    assert e_loss <= 1e-6 and e_img <= 1e-6 and e_light <= 1e-5
    assert e_edge <= 1e-5
    assert not mask or edge.sum() >= B * 8 * W // 2


def test_composite_loss_grad_at_the_degenerate_normal():
    """img = (0.5, 0.5, 0.5): the forward shades it as rn_phong_composite does (loss 0 against that image) and the gradient is
    finite -- the mask term alone -- and adds nothing to d_light."""
    from rendernet_b200 import ops
    n = np.full((1, 4, 4, 3), 0.5, np.float32)
    ld, lc = _d(np.array([[0.3, 0.4, 0.8]], np.float32)), _d(np.ones((1, 3), np.float32))
    img = ops.phong_composite(_d(n), ld, lc, 0.1, 0.9)
    loss, di, dl = ops.phong_composite_loss_grad(_d(n), img, ld, lc)
    assert (loss == 0).all() and (di == 0).all()
    loss, di, dl = ops.phong_composite_loss_grad(_d(n), torch.zeros_like(img), ld, lc)
    assert torch.isfinite(di).all() and (dl == 0).all() and loss.item() > 0


# ----------------------------------------------------------------------------------------- per-item losses
@pytest.mark.parametrize("C", [1, 3])
@pytest.mark.parametrize("kind", ["mse", "bce"])
def test_per_item_losses(kind, C):
    """rn_image_loss_grad_items against NumPy float64 (loss 1e-6 relative) for B = 1..8, against the scalar kernel: the mean of
    the per-item losses is its loss, and the per-item d_img B times its gradient within two fp32 roundings."""
    from rendernet_b200 import ops
    rng = np.random.default_rng(7 + C)
    for B in range(1, 9):
        p = rng.uniform(0.001, 0.999, (B, 40, 24, C)).astype(np.float32)
        t = (rng.random((B, 40, 24, C)) < 0.3).astype(np.float32) if kind == "bce" else rng.random((B, 40, 24, C)).astype(np.float32)
        loss, di = ops.image_loss_grad_items(_d(p), _d(t), kind)
        p64, t64 = p.astype(np.float64), t.astype(np.float64)
        if kind == "mse":
            want = ((p64 - t64) ** 2).mean(axis=(1, 2, 3))
        else:
            want = -(t64 * np.log(1e-6 + p64) + (1 - t64) * np.log(1e-6 + 1 - p64)).sum(axis=(1, 2, 3))
        assert _rel(loss.cpu().numpy(), want) <= 1e-6 and loss.dtype == torch.float64
        scalar, ds = ops.image_loss_grad(_d(p), _d(t), kind)
        assert abs(float(loss.mean()) - float(scalar)) <= 1e-12 * abs(float(scalar))
        a, b = di.cpu().numpy().astype(np.float64), B * ds.cpu().numpy().astype(np.float64)
        assert (np.abs(a - b) <= 2.0 ** -22 * np.abs(a)).all(), (B, float(np.abs(a - b).max()))
        loss2, none = ops.image_loss_grad_items(_d(p), _d(t), kind, want_grad=False)
        assert none is None and torch.allclose(loss2, loss, rtol=1e-12, atol=0)


# ----------------------------------------------------------------------------------------- the whole chain
def _chair(B):
    bv = np.load(os.path.join(os.path.dirname(__file__), "golden", "binvox.npz"))
    vox = np.unpackbits(bv["chair_bits"]).reshape(1, 64, 64, 64, 1).astype(np.float32)
    vox = vox * 0.75 + 0.125 * (np.random.default_rng(2).random(vox.shape) < 0.02)
    return np.ascontiguousarray(np.repeat(vox, B, 0))


def _hypotheses():
    from rendernet_b200.Reconstruct_RenderNet_Face import create_param_center
    p = create_param_center(250, 60, 60, 30)
    lights = np.stack([np.linspace(230, 320, 5) * math.pi / 180, np.full(5, math.radians(60.0))], 1)
    return p, lights


def _oracle_pose_grads(vox, poses, W, masks, Gs):
    """dL/dview_params of the frozen-kink oracle for each image gradient in Gs (one forward, one backward each)."""
    from oracle.frozen_kinks import prelu_kinks
    from rendernet_b200.backward import pose_matrix_jacobian_vjp
    minv = orc.inverse_total_matrix(*orc.rotation_around_grid_centroid(poses), 64, 128)
    mt = torch.tensor(minv.astype(np.float64), requires_grad=True)
    grid = rc.resample(torch.from_numpy(vox.astype(np.float64)), mt, 128)
    with prelu_kinks(W, masks=masks):
        img = orc.rendernet_shader(grid.float(), W)
    out = []
    for k, G in enumerate(Gs):
        g, = torch.autograd.grad(img, mt, torch.from_numpy(np.asarray(G, np.float32)), retain_graph=k + 1 < len(Gs))
        out.append(pose_matrix_jacobian_vjp(poses, g.numpy()))
    return out


@pytest.mark.parametrize("network", ["rgb", "grey"])
@pytest.mark.parametrize("precision", ["exact", "fast"])
def test_full_size_fit_gradients_match_frozen_kink_oracle(precision, network):
    """shader_fit_gradients at B = 5 (the search's five hypotheses, full size): "phong" and "mse" on the RGB network, "bce" on the
    greyscale one.  The objective in float64 at the device's image (phong: at its fp32 mask value), pushed through the oracle
    Shader with the device's kinks frozen and the device-cell resampler: dL/dpose within the face reconstruction's bars (exact
    3e-4, fast 6e-3), loss 1e-6 and dL/dlight 1e-5 relative.  dL/dlight also against a central difference of the loss kernel
    (step 1e-3 rad, bar 1e-3: the step carries pixels across n.l = 0 and the clips).  Measured on an H100 80GB HBM3: dL/dpose
    1.1e-4 to 1.2e-4 exact and 1.0e-3 to 2.5e-3 fast, loss <= 8.7e-8, dL/dlight 2.3e-7 (central difference 4.5e-4 / 5.8e-4)."""
    from rendernet_b200 import ops, tfcompat as tf
    from rendernet_b200.backward import ShaderInputGradients
    from rendernet_b200.shader_fit import light_dir, shader_fit_gradients
    from oracle.frozen_kinks import tape_prelu_masks
    B = 5
    grey = network == "grey"
    W = orc.init_shader_weights(seed=1, is_greyscale=grey, alpha_range=(0.05, 0.3), bias_jitter=0.02)
    vox, (poses, lights) = _chair(B), _hypotheses()
    ig = ShaderInputGradients(W, B, precision=precision, is_greyscale=grey)
    rng = np.random.default_rng(8)
    objectives = ("bce",) if grey else ("phong", "mse")
    C = 1 if grey else 3
    results, Gs = {}, []
    for obj in objectives:
        tgt = (rng.random((B, 512, 512, C)) < 0.3).astype(np.float32) if obj == "bce" else rng.random((B, 512, 512, C)).astype(np.float32)
        loss, g = shader_fit_gradients(ig, vox, poses, tgt, obj, light=lights if obj == "phong" else None)
        img = ig.img.cpu().numpy()
        with tf.use_store(ig.store):
            masks = tape_prelu_masks(ig.tape)
        x = torch.tensor(img.astype(np.float64), requires_grad=True)
        t64 = torch.from_numpy(tgt).double()
        lt = torch.tensor(lights, requires_grad=True)
        if obj == "phong":
            ref = pn.fit_loss(x, t64, pn.generate_light_pos(lt), torch.ones(B, 3, dtype=D64), 0.1, 0.9, False, True,
                              torch.from_numpy(_mask32(img, False)))
        elif obj == "mse":
            ref = ((x - t64) ** 2).mean(dim=(1, 2, 3))
        else:
            ref = -(t64 * torch.log(1e-6 + x) + (1 - t64) * torch.log(1e-6 + 1 - x)).sum(dim=(1, 2, 3))
        ref.sum().backward()
        Gs.append(x.grad.numpy())
        results[obj] = dict(loss=loss, g=g, ref=ref.detach().numpy(), dlight=lt.grad.numpy() if obj == "phong" else None,
                            img=img, tgt=tgt)
    for obj, dpose_f in zip(objectives, _oracle_pose_grads(vox, poses, W, masks, Gs)):
        r = results[obj]
        e = dict(loss=float((np.abs(r["loss"] - r["ref"]) / r["ref"]).max()), pose=_rel(r["g"]["pose"], dpose_f))
        if obj == "phong":
            e["light"] = _rel(r["g"]["light"], r["dlight"])
            # central difference of the loss kernel in the light angles, at the device's image
            h, cd = 1e-3, np.zeros((B, 2))
            for k in range(2):
                lp, lm = lights.copy(), lights.copy()
                lp[:, k] += h
                lm[:, k] -= h
                f = [ops.phong_composite_loss_grad(_d(r["img"]), _d(r["tgt"]), _d(light_dir(L)), (1.0, 1.0, 1.0), 0.1, 0.9)[0]
                     .cpu().numpy() for L in (lp, lm)]
                cd[:, k] = (f[0] - f[1]) / (2 * h)
            e["light_cd"] = _rel(r["g"]["light"], cd)
        print(f"[{precision}] {obj} B=5 vs frozen-kink oracle: " + ", ".join(f"{k} {v:.2e}" for k, v in e.items()))
        bar = 3e-4 if precision == "exact" else 6e-3
        assert e["loss"] < 1e-6 and e["pose"] < bar, (obj, e)
        if obj == "phong":
            assert e["light"] < 1e-5 and e["light_cd"] < 1e-3, e


def test_batch_of_five_equals_five_single_calls():
    """shader_fit_gradients at B = 5 equals five B = 1 calls: the loss to its double atomics' order (1e-12), dL/dpose and
    dL/dlight within the noise of the resampler's fp32 atomics (1e-5 of scale)."""
    from rendernet_b200.backward import ShaderInputGradients
    from rendernet_b200.shader_fit import shader_fit_gradients
    W = orc.init_shader_weights(seed=1, alpha_range=(0.05, 0.3), bias_jitter=0.02)
    vox, (poses, lights) = _chair(5), _hypotheses()
    tgt = np.random.default_rng(9).random((5, 512, 512, 3)).astype(np.float32)
    ig5 = ShaderInputGradients(W, 5)
    loss5, g5 = shader_fit_gradients(ig5, vox, poses, tgt, "phong", light=lights)
    del ig5
    torch.cuda.empty_cache()
    ig1 = ShaderInputGradients(W, 1)
    for b in range(5):
        loss1, g1 = shader_fit_gradients(ig1, vox[b:b + 1], poses[b:b + 1], tgt[b:b + 1], "phong", light=lights[b:b + 1])
        ep, el = _rel(g1["pose"][0], g5["pose"][b]), _rel(g1["light"][0], g5["light"][b])
        print(f"item {b}: loss {loss1[0]:.9e} vs {loss5[b]:.9e}, dpose {ep:.2e}, dlight {el:.2e}")
        assert abs(loss1[0] - loss5[b]) <= 1e-12 * loss5[b] and ep < 1e-5 and el < 1e-5


# ----------------------------------------------------------------------------------------- the search and the command line
def _true_case():
    from rendernet_b200.RenderNet_demo import compute_pose_param
    pose = compute_pose_param(262.0, 54.0, 3.3)[0].astype(np.float32)
    light = np.array([math.radians(280.0), math.radians(60.0)], np.float32)
    return pose, light


def test_short_run_decreases_the_loss():
    """run() with two epochs of three steps, seeded weights, on a target rendered at a known pose and light inside the first
    window: the best loss falls below every first-step loss, the selection is the argmin of the re-evaluated losses, and the
    selected pose lies in the last searched window."""
    from rendernet_b200.RenderNet_demo import compute_pose_param
    from rendernet_b200.shader_fit import ShaderPoseFit, in_window
    fit = ShaderPoseFit(None, _chair(1), objective="phong", inner_step=3, max_epochs=2)
    pose, light = _true_case()
    target = fit.render(dict(pose=np.tile(pose, (5, 1)), light=np.tile(light, (5, 1))))["shaded"]
    seen = []
    out = fit.run(target, init=dict(pose=compute_pose_param(250.0, 60.0, 3.3)[0], light_elevation=math.radians(60.0)),
                  callback=lambda e, i, s, loss, sel: seen.append((np.asarray(loss).copy(), None if sel is None else sel.copy())))
    first = seen[0][0]
    sel = [s[1] for s in seen if s[1] is not None]
    print("first-step losses", first, "best loss per epoch", out["best_loss"], "selected", out["best_index"], "pose", out["pose"],
          "light", out["light"], "windows", out["windows"])
    assert len(seen) == 6 and len(sel) == 2
    assert out["best_loss"][-1] < first.min()
    assert out["best_index"] == int(np.argmin(sel[-1])) and out["best_loss"][-1] == sel[-1].min()
    assert in_window(out["pose"], out["windows"][-1])
    assert out["pose"][2] == np.float32(1.0) and out["light"].shape == (2,)


def _write_binvox(path, vox):
    """A #binvox 1 file of a 64^3 occupancy grid (x-z-y run-length order, binvox_rw's fix_coords inverse)."""
    flat = np.ascontiguousarray(np.asarray(vox, bool).reshape(64, 64, 64).transpose(0, 2, 1)).ravel().astype(np.uint8)
    runs, i = [], 0
    while i < flat.size:
        j = i
        while j < flat.size and j - i < 255 and flat[j] == flat[i]:
            j += 1
        runs += [flat[i], j - i]
        i = j
    with open(path, "wb") as f:
        f.write(b"#binvox 1\ndim 64 64 64\ntranslate 0 0 0\nscale 1\ndata\n" + bytes(runs))


@pytest.mark.parametrize("objective", ["phong", "bce"])
def test_command_line_fits_a_rendered_target(tmp_path, objective):
    """python -m rendernet_b200.shader_fit on a target rendered with the seeded weights at a known pose (and light): the JSON's
    pose lies in the searched window, its loss below the starting loss, and the PNG is the fitted render."""
    from PIL import Image
    from rendernet_b200 import binvox_rw
    from rendernet_b200.shader_fit import ShaderPoseFit, in_window, main
    vox = (_chair(1)[0, ..., 0] > 0.5)
    _write_binvox(tmp_path / "chair.binvox", vox)
    with open(tmp_path / "chair.binvox", "rb") as f:
        assert np.array_equal(binvox_rw.read_as_3d_array(f).data, vox)
    grey = objective == "bce"
    fit = ShaderPoseFit(None, vox.astype(np.float32), objective=objective, is_greyscale=grey)
    pose, light = _true_case()
    state = dict(pose=np.tile(pose, (5, 1)), light=np.tile(light, (5, 1)))
    img = fit.render(state)
    u8 = img["shaded_u8"][0] if objective == "phong" else img["image_u8"][0, ..., 0]
    Image.fromarray(u8).save(tmp_path / "target.png")
    del fit
    torch.cuda.empty_cache()
    argv = ["--voxel_path", str(tmp_path / "chair.binvox"), "--target", str(tmp_path / "target.png"), "--model",
            str(tmp_path / "none.pb"), "--objective", objective, "--inner_step", "2", "--max_epochs", "2", "--out_dir",
            str(tmp_path / "fit")] + (["--is_greyscale"] if grey else [])
    res = main(argv)
    with open(tmp_path / "fit" / "chair_fit.json") as f:
        saved = json.load(f)
    assert saved == json.loads(json.dumps(res))
    print(objective, {k: v for k, v in saved.items() if k != "windows"})
    assert in_window(np.array(saved["pose"]), saved["windows"][-1])
    assert saved["best_loss"][-1] < min(saved["first_step_loss"])
    assert ("light_azimuth" in saved) == (objective == "phong")
    png = np.asarray(Image.open(tmp_path / "fit" / "chair_fit.png"))
    assert png.shape == ((512, 512, 3) if objective == "phong" else (512, 512))
