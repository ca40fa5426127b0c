"""GPU tests of the face-reconstruction shape decoder (Reconstruct_RenderNet_Face.decoder_3d_pretrained, backward.ShapeDecoderGradients),
its kernels (rn_conv3d_f32, rn_act_backward_f32) and the reconstruction driver (FaceReconstruction.step / run).

References are float64: oracle/shape_decoder.py's decoder (run on the device in float64), float64 autograd, and for the whole
reconstruction step the oracle chain float64 decoder -> device-cell resampler (oracle/resample_cells.py) -> rendernet_texture with
the device's PReLU / ReLU kinks frozen (oracle/frozen_kinks.py).  Errors are max |error| / max |reference| unless stated otherwise.
"""
import math

import numpy as np
import pytest
import torch

from oracle import rendernet_oracle as orc
from oracle import resample_cells as rc
from oracle.shape_decoder import CONV_LAYERS, decoder_3d, init_shape_decoder_weights

pytestmark = pytest.mark.gpu
dev = "cuda"
TE = "texture_encoder"
D64 = torch.float64


def _rel(got, want):
    got = got.detach().double().cpu().numpy() if isinstance(got, torch.Tensor) else np.asarray(got, np.float64)
    want = want.detach().double().cpu().numpy() if isinstance(want, torch.Tensor) else np.asarray(want, np.float64)
    assert got.shape == want.shape, (got.shape, want.shape)
    return float(np.abs(got - want).max() / max(np.abs(want).max(), 1e-300))


def _in_shape(name, B):
    """input grid of each decoder layer: 4^3 x 256 -> ... -> 64^3 x 16 (g_conv5 keeps 64^3)."""
    shape = {n: sh for n, sh, _ in CONV_LAYERS}[name]
    side = {256: 4, 128: 8, 64: 16, 32: 32, 16: 64}[shape[4]]
    return (B, side, side, side, shape[4])


# ----------------------------------------------------------------------------------------- rn_conv3d_f32, layer by layer
@pytest.mark.parametrize("B", [1, 5, 32])
@pytest.mark.parametrize("name", [n for n, _, _ in CONV_LAYERS])
def test_layer_forward_and_data_gradient_match_float64(name, B):
    """Each decoder layer at its own shape: conv3d_transpose + bias (forward) against float64, and its data gradient -- conv3d
    of dL/dy on the same filter array, stride 2 for g_conv1..4, stride 1 from 1 to 16 channels for g_conv5 -- against float64
    autograd.  Two runs are bit-identical (split-K layers sum their slices in a fixed order)."""
    from rendernet_b200 import ops
    W = init_shape_decoder_weights(seed=11)
    s = dict((n, st) for n, _, st in CONV_LAYERS)[name]
    w, b = torch.from_numpy(W[name + "_weights"]).to(dev), torch.from_numpy(W[name + "_biases"]).to(dev)
    g = torch.Generator(device=dev).manual_seed(B * 100 + len(name))
    x = torch.randn(_in_shape(name, B), device=dev, generator=g)
    y = ops.conv3d_f32(x, w, b, s, True)
    xr = x.double().requires_grad_(True)
    yr = orc.conv3d_transpose(xr, w.double(), b.double(), (s, s, s), dtype=D64)
    G = torch.randn(tuple(yr.shape), device=dev, generator=g)
    (yr * G.double()).sum().backward()
    dx = ops.conv3d_f32(G, w, None, s, False)
    e_f, e_b = _rel(y, yr), _rel(dx, xr.grad)
    same = torch.equal(y, ops.conv3d_f32(x, w, b, s, True)) and torch.equal(dx, ops.conv3d_f32(G, w, None, s, False))
    print(f"{name} B={B}: forward {e_f:.2e}, data gradient {e_b:.2e}, bit-identical rerun {same}")
    # measured on an H100 80GB HBM3 (400 W): forward 3.0e-7 .. 1.7e-6, data gradient 3.4e-7 .. 2.3e-6 (K up to 8192 fp32 terms)
    assert e_f < 7e-6 and e_b < 7e-6 and same


def test_conv3d_f32_rejects_what_it_cannot_run():
    from rendernet_b200 import ops
    from rendernet_b200._lib import RenderNetCudaError
    w = torch.zeros((4, 4, 4, 16, 32), device=dev)
    with pytest.raises(RenderNetCudaError):             # B > 32
        ops.conv3d_f32(torch.zeros((33, 4, 4, 4, 32), device=dev), w, None, 2, True)
    with pytest.raises(ValueError):                     # channel mismatch
        ops.conv3d_f32(torch.zeros((1, 4, 4, 4, 16), device=dev), w, None, 2, True)
    with pytest.raises(ValueError):
        ops.conv3d_f32(torch.zeros((1, 4, 4, 4, 32), device=dev), w, None, 2, True, act="prelu")


# ----------------------------------------------------------------------------------------- ELU / sigmoid at the boundaries
_Z = np.array([0.0, 1e-30, -1e-30, -1e-7, -0.5, -20.0, -100.0, -1e30, 2.5, 1e30], np.float32)


def _identity_filter():
    """conv3d_transpose s1 filter whose only non-zero tap passes channel 0 through (o = i): the output is the input exactly."""
    w = torch.zeros((4, 4, 4, 16, 16), device=dev)
    for c in range(16):
        w[1, 1, 1, c, c] = 1.0
    return w


def test_elu_and_sigmoid_forward_at_boundary_values():
    """The fused epilogues on exact pre-activations: ELU = exp(z) - 1 below zero (-1e-30 -> +0, -100 -> -1 exactly), z itself at
    and above zero; sigmoid in fp32.  Against float64 within the rounding of exp."""
    from rendernet_b200 import ops
    z = np.zeros((1, 4, 4, 4, 16), np.float32)
    z.reshape(-1)[:_Z.size] = _Z
    x = torch.from_numpy(z).to(dev)
    w = _identity_filter()
    assert torch.equal(ops.conv3d_f32(x, w, None, 1, True), x)
    elu = ops.conv3d_f32(x, w, None, 1, True, act="elu").cpu().numpy().reshape(-1)[:_Z.size]
    sig = ops.conv3d_f32(x, w, None, 1, True, act="sigmoid").cpu().numpy().reshape(-1)[:_Z.size]
    z64 = _Z.astype(np.float64)
    want_elu = np.where(z64 < 0, np.exp(z64) - 1, z64)
    print("elu:", elu, "sigmoid:", sig)
    assert np.all(np.abs(elu - want_elu) <= 1.2e-7 * np.maximum(1, np.abs(want_elu)))
    assert elu[1] == np.float32(1e-30) and elu[2] == 0.0 and not np.signbit(elu[2]) and elu[6] == -1.0 and elu[7] == -1.0
    assert elu[8] == 2.5 and elu[9] == np.float32(1e30)
    assert np.abs(sig - 1 / (1 + np.exp(-z64))).max() < 2e-7 and sig[7] == 0.0 and sig[9] == 1.0


def test_act_backward_f32_bit_identical_to_tf_rules():
    """EluGrad from the output, y < 0 ? g (y + 1) : g, and SigmoidGrad g y (1 - y), on outputs at the boundaries: y = 0, -0
    (ELU of -0), ELU of tiny negative z (y = +0 or -1e-7 ...), y = -1 (large negative z), and random values."""
    from rendernet_b200 import ops
    rng = np.random.default_rng(3)
    y_elu = np.concatenate([np.array([0.0, -0.0, -1.1920929e-07, -5.9604645e-08, -1.0, -0.99999994, 1e-30, 3.0], np.float32),
                            np.where(rng.standard_normal(4088) < 0, np.expm1(rng.standard_normal(4088) * -2), 1).astype(np.float32)])
    y_sig = np.concatenate([np.array([0.0, 1.0, 0.5, 1e-30, 0.99999994, 5.9604645e-08, 0.25, 0.75], np.float32),
                            rng.random(4088).astype(np.float32)])
    g = rng.standard_normal(4096).astype(np.float32)
    g[::17] = 0.0
    for act, y, want in (("elu", y_elu, np.where(y_elu < 0, g * (y_elu + np.float32(1)), g)),
                         ("sigmoid", y_sig, g * y_sig * (np.float32(1) - y_sig))):
        got = ops.act_backward_f32(torch.from_numpy(g).to(dev), torch.from_numpy(y).to(dev), act).cpu().numpy()
        assert want.dtype == np.float32 and np.array_equal(got.view(np.uint32), want.view(np.uint32)), act
    got = ops.act_backward_f32(torch.from_numpy(g[:8]).to(dev), torch.from_numpy(y_elu[:8]).to(dev), "elu").cpu().numpy()
    assert got[0] == g[0] and got[1] == g[1] and got[4] == 0.0        # y = 0 and -0 pass g; y = -1 stops it


# ----------------------------------------------------------------------------------------- the whole decoder
@pytest.mark.parametrize("B", [1, 5])
def test_whole_decoder_forward_and_latent_gradient_match_float64(B):
    """decoder_3d_pretrained through ShapeDecoderGradients: the voxels against the float64 oracle, dL/dlatent element by element
    against float64 autograd (ELU and sigmoid are C^1: no kinks to freeze).  Reproducible bit for bit."""
    from rendernet_b200.backward import ShapeDecoderGradients
    W = init_shape_decoder_weights(seed=5)
    z = np.random.default_rng(B).standard_normal((B, 200)).astype(np.float32)
    z[0] = 0.5
    G = np.random.default_rng(B + 1).standard_normal((B, 64, 64, 64, 1)).astype(np.float32)
    sdg = ShapeDecoderGradients(W, B)
    vox = sdg.forward(z)
    dz = sdg.backward(G)
    assert sorted(r["op"] for r in sdg.tape) == ["conv_f32"] * 5 + ["fc"]
    zr = torch.tensor(z.astype(np.float64), device=dev, requires_grad=True)
    Wd = {k: torch.from_numpy(v).to(dev) for k, v in W.items()}
    ref = decoder_3d(zr, Wd, dtype=D64)
    (ref * torch.from_numpy(G).to(dev).double()).sum().backward()
    e_f = _rel(vox, ref)
    e_b = max(_rel(dz[b], zr.grad[b]) for b in range(B))
    vox2, dz2 = sdg.forward(z).clone(), sdg.backward(G)
    same = torch.equal(vox, vox2) and np.array_equal(dz.view(np.uint32), dz2.view(np.uint32))
    print(f"shape decoder B={B}: voxels {e_f:.2e}, dL/dlatent (worst item) {e_b:.2e}, bit-identical rerun {same}")
    # measured on an H100 80GB HBM3 (400 W): voxels 4.7e-7 / 7.0e-7, dL/dlatent 8.5e-7 / 1.7e-6 at B = 1 / 5
    assert e_f < 3e-6 and e_b < 5e-6 and same
    # a device tensor gradient is taken as it is
    assert np.array_equal(sdg.backward(torch.from_numpy(G).to(dev)), dz)


def test_decoder_variable_names_and_missing_key():
    """The variables decoder_3d_pretrained creates carry the reference's scopes; a missing npz key raises KeyError."""
    from rendernet_b200.backward import ShapeDecoderGradients
    W = init_shape_decoder_weights(seed=1)
    sdg = ShapeDecoderGradients(W, 1)
    sdg.forward(np.full((1, 200), 0.5, np.float32))
    want = ["g_conv1/g_conv1/biases", "g_conv1/g_conv1/weights", "g_conv2/g_conv2/biases", "g_conv2/g_conv2/weights",
            "g_conv3/g_conv3/biases", "g_conv3/g_conv3/weights", "g_conv4/g_conv4/biases", "g_conv4/g_conv4/weights",
            "g_conv5/biases", "g_conv5/weights", "g_zP/g_gc1/biases", "g_zP/g_gc1/weights"]
    assert sorted(sdg.store.vars) == want
    for k in ("g_conv3_g_conv3_weights", "g_conv5_biases", "g_zP_g_gc1_weights"):
        Wm = dict(W)
        del Wm[k]
        with pytest.raises(KeyError):
            ShapeDecoderGradients(Wm, 1).forward(np.zeros((1, 200), np.float32))


# ----------------------------------------------------------------------------------------- FaceReconstruction
def _texture_weights(seed):
    """Texture weights with mixed-sign PReLU slopes, residual slopes zero (model="pretrained" uses ReLU there)."""
    W = orc.init_texture_weights(seed=seed, alpha_range=(-0.3, 0.3), bias_jitter=0.02)
    for k in list(W):
        if k.endswith("/alpha") and "/res" in k:
            W[k] = np.zeros_like(W[k])
    return W


def _tex_decoder64(z, W, masks):
    """float64 texture decoder with the PReLU branches `masks`."""
    def pr(t, name):
        a = torch.from_numpy(W[f"{TE}/{name}/alpha"].astype(np.float64))
        return torch.where(torch.as_tensor(masks[f"{TE}/{name}/alpha"]).reshape(t.shape), t, a * t)
    h = pr(orc.fully_connected(z, W[f"{TE}/e_tex_fc1/fully_connected/weights"], W[f"{TE}/e_tex_fc1/fully_connected/biases"],
                               dtype=D64), "e_tex_fc1").reshape(z.shape[0], 32, 32, 32, 4)
    for name, s, tr in (("e_tex_conv0", 1, True), ("e_tex_conv1", 2, True), ("e_tex_conv2", 1, False)):
        pre = f"{TE}/{name}/{'conv3d_transpose' if tr else 'conv3d'}"
        h = pr((orc.conv3d_transpose if tr else orc.conv3d)(h, W[pre + "/weights"], W[pre + "/biases"], (s, s, s), dtype=D64), name)
    return h


def _setup(seed=61):
    from rendernet_b200.Reconstruct_RenderNet_Face import pretrained_dict_from_texture_weights
    W = _texture_weights(seed)
    Wd = init_shape_decoder_weights(seed + 1)
    return W, pretrained_dict_from_texture_weights(W), Wd


@pytest.mark.parametrize("precision", ["exact", "fast"])
def test_face_reconstruction_step_matches_frozen_kink_oracle(precision):
    """One FaceReconstruction.step at full size, B = 5: the loss and dL/d(latent, texture, pose, light azimuth) of sum_b loss[b]
    against the oracle chain (float64 shape decoder -> device-cell resampler -> rendernet_texture with the device's kinks frozen;
    the objective in float64 at the device's images, as its own kinks are frozen that way).  The update is var - eta * grad in
    float32.  The forward from the decoder's device tensor equals the NumPy-input forward bit for bit."""
    from rendernet_b200 import tfcompat as tf
    from rendernet_b200.backward import TextureInputGradients, pose_matrix_jacobian_vjp
    from rendernet_b200.Reconstruct_RenderNet_Face import FaceReconstruction, create_param_center
    from oracle import phong_tf as pt
    from oracle.frozen_kinks import prelu_kinks, tape_prelu_masks
    B = 5
    W, Wp, Wd = _setup()
    rec = FaceReconstruction(Wp, Wd, batch=B, precision=precision)
    rng = np.random.default_rng(62)
    state = dict(latent=(0.5 + 0.3 * rng.standard_normal((B, 200))).astype(np.float32),
                 pose=create_param_center(270, 60, 90, 30),
                 texture=rng.standard_normal((B, 199)).astype(np.float32),
                 light=np.linspace(230, 320, 5).reshape(B, 1).astype(np.float32) * np.float32(math.pi / 180))
    target = rng.random((B, 512, 512, 3)).astype(np.float32)
    new, loss, grads = rec.step(state, target)
    for k in state:
        want = (state[k] - np.float32(rec.eta[k]) * grads[k].astype(np.float32)).astype(np.float32)
        assert new[k].dtype == np.float32 and np.array_equal(new[k], want), k

    # the device's images and kinks; the forward from the device voxel tensor vs from NumPy
    vox = rec.sdg.forward(state["latent"])
    a1, n1 = (t.clone() for t in rec.tig.forward(vox, state["texture"], state["pose"]))
    a2, n2 = rec.tig.forward(vox.cpu().numpy(), state["texture"], state["pose"])
    same = torch.equal(a1, a2) and torch.equal(n1, n2)
    tigT = TextureInputGradients(W, B, precision=precision)             # the same network under TF variable names
    at, nt = tigT.forward(vox, state["texture"], state["pose"])
    same_t = torch.equal(at, a1) and torch.equal(nt, n1)
    with tf.use_store(tigT.store):
        masks = tape_prelu_masks(tigT.tape)

    # the objective in float64 at the device's images
    el = rec.elevation
    a_ = torch.tensor(a1.cpu().numpy().astype(np.float64), requires_grad=True)
    n_ = torch.tensor(n1.cpu().numpy().astype(np.float64), requires_grad=True)
    az = torch.tensor(state["light"].astype(np.float64), requires_grad=True)
    ref = pt.recon_loss(a_, n_, torch.from_numpy(target).double(), pt.tf_generate_light_pos(az, el), torch.ones(B, 3, dtype=D64))
    ref.sum().backward()
    # ... pushed through the frozen-kink network to the voxels, the texture vector and M^-1, then the decoder and the pose map
    minv = orc.inverse_total_matrix(*orc.rotation_around_grid_centroid(state["pose"]), 64, 128)
    vt = torch.tensor(vox.cpu().numpy().astype(np.float64), requires_grad=True)
    zt = torch.tensor(state["texture"].astype(np.float64), requires_grad=True)
    mt = torch.tensor(minv.astype(np.float64), requires_grad=True)
    x = torch.cat([rc.resample(vt, mt, 128), rc.resample(_tex_decoder64(zt, W, masks), mt, 128)], -1)
    with prelu_kinks(W, masks=masks):
        img, nrm = orc.rendernet_texture(x.float(), W)
    (img * a_.grad.float() + nrm * n_.grad.float()).sum().backward()
    lat = torch.tensor(state["latent"].astype(np.float64), device=dev, requires_grad=True)
    Wdd = {k: torch.from_numpy(v).to(dev) for k, v in Wd.items()}
    (decoder_3d(lat, Wdd, dtype=D64) * vt.grad.to(dev)).sum().backward()
    dpose_f = pose_matrix_jacobian_vjp(state["pose"], mt.grad.numpy())
    errs = dict(loss=_rel(loss, ref), latent=_rel(grads["latent"], lat.grad), texture=_rel(grads["texture"], zt.grad),
                pose=_rel(grads["pose"], dpose_f), light=_rel(grads["light"], az.grad))
    print(f"[{precision}] FaceReconstruction.step B=5 vs frozen-kink oracle: " + ", ".join(f"{k} {v:.2e}" for k, v in errs.items())
          + f"; forward from the device voxels bit-identical {same}, pretrained == texture-model forward {same_t}")
    assert same and same_t
    # Measured on an H100 80GB HBM3 (400 W): exact loss 1.5e-9, latent 2.2e-4, texture 2.5e-4, pose 1.2e-4, light 1.0e-6; fast
    # 1.9e-9, 2.0e-3, 2.4e-3, 2.1e-3, 6.8e-7.  The bars are those of the Texture+Normal input-gradient tests.
    bar = 3e-4 if precision == "exact" else 6e-3
    assert errs["loss"] < 1e-6 and errs["light"] < 1e-5
    for k in ("latent", "texture", "pose"):
        assert errs[k] < bar, (k, errs[k])


def test_face_reconstruction_short_run_decreases_the_loss():
    """run() with max_epochs = 2, inner_step = 3 on a target rendered from a known latent / texture / pose / light: the best loss
    falls from epoch to epoch and below every first-step loss, and the selected hypothesis is the argmin of the re-evaluated
    losses the callback saw."""
    from rendernet_b200.Reconstruct_RenderNet_Face import FaceReconstruction
    from oracle import phong_tf as pt
    B = 5
    _, Wp, Wd = _setup(71)
    rec = FaceReconstruction(Wp, Wd, batch=B, precision="exact", inner_step=3, max_epochs=2, seed=3)
    rng = np.random.default_rng(72)
    z_true = np.tile((0.5 + 0.2 * rng.standard_normal(200)).astype(np.float32), (B, 1))
    t_true = np.tile(np.random.default_rng(3).standard_normal((B, 199))[2].astype(np.float32) * 0.5, (B, 1))
    pose_true = np.tile(np.array([[math.radians(272), math.radians(3), 1.0]], np.float32), (B, 1))
    light_true = np.full((B, 1), math.radians(280), np.float32)
    albedo, normal = rec.tig.forward(rec.sdg.forward(z_true), t_true, pose_true)
    ld = pt.tf_generate_light_pos(torch.from_numpy(light_true.astype(np.float64)), rec.elevation)
    shade = pt.tf_phong_composite(normal.double().cpu(), ld, torch.ones(B, 3, dtype=D64), 0.0, 1.0)
    target = (albedo.double().cpu() * shade).float().numpy()
    seen = []
    out = rec.run(target, callback=lambda e, i, s, loss, sel: seen.append((e, i, np.asarray(loss).copy(),
                                                                            None if sel is None else np.asarray(sel).copy())))
    first = seen[0][2]
    sel = [s for s in seen if s[3] is not None]
    print("first-step losses", first, "best loss per epoch", out["best_loss"], "selected", out["best_index"])
    assert len(seen) == 6 and len(sel) == 2
    assert out["best_loss"][1] < out["best_loss"][0] < first.min()
    assert out["best_index"] == int(np.argmin(sel[-1][3])) and out["best_loss"][-1] == sel[-1][3].min()
    assert out["voxels"].shape == (64, 64, 64) and out["latent"].shape == (200,) and out["texture"].shape == (199,)
    assert out["pose"].shape == (3,) and out["light"].shape == (1,)
