"""GPU tests of fine-tuning the face-reconstruction shape decoder: the weight-gradient kernels (rn_conv3d_f32_weight_grad, the
no-activation case of rn_fully_connected_param_grad), ShapeDecoderGradients.backward(want_weight_grads=True) and
nn.ShapeDecoder(trainable=True), alone and composed with the pretrained Texture+Normal network and the Phong composite.

References are float64: oracle/shape_decoder.py's decoder and orc.conv3d_transpose in float64 autograd on the device, and for
the composed objective the chain float64 decoder -> device-cell resampler (oracle/resample_cells.py) -> rendernet_texture with
the device's PReLU / ReLU kinks frozen (oracle/frozen_kinks.py).  Errors are max |error| / max |reference|.
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
D64 = torch.float64
TE = "texture_encoder"
# npz prefix -> TF scope of each decoder layer
TF_PREFIX = {"g_zP_g_gc1": "g_zP/g_gc1", "g_conv1_g_conv1": "g_conv1/g_conv1", "g_conv2_g_conv2": "g_conv2/g_conv2",
             "g_conv3_g_conv3": "g_conv3/g_conv3", "g_conv4_g_conv4": "g_conv4/g_conv4", "g_conv5": "g_conv5"}


def _rel(got, want):
    got = got.detach().double().cpu().numpy() if isinstance(got, torch.Tensor) else np.asarray(got, np.float64)
    want = want.detach().double().cpu().numpy() if isinstance(want, torch.Tensor) else np.asarray(want, np.float64)
    assert got.shape == want.shape, (got.shape, want.shape)
    return float(np.abs(got - want).max() / max(np.abs(want).max(), 1e-300))


def _in_shape(name, B):
    shape = {n: sh for n, sh, _ in CONV_LAYERS}[name]
    side = {256: 4, 128: 8, 64: 16, 32: 32, 16: 64}[shape[4]]
    return (B, side, side, side, shape[4])


def _bits_equal(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


# ----------------------------------------------------------------------------------------- the kernels, layer by layer
@pytest.mark.parametrize("B", [1, 5, 32])
@pytest.mark.parametrize("name", [n for n, _, _ in CONV_LAYERS])
def test_conv_weight_grad_matches_float64(name, B):
    """dw [4,4,4,Cout,Cin] and db of each decoder conv at its own shape, for random x and gz = dL/d(pre-activation), against
    float64 autograd of orc.conv3d_transpose; two runs are bit-identical.  g_conv5 (16 -> 1, s1) runs the direct kernel, the
    others the 8-phase split-K GEMM.  Measured on an H100 80GB HBM3 (700 W): dw 3.6e-7 .. 2.2e-6, db 1.9e-7 .. 2.3e-6 over
    the 15 cases (K up to 32 x 64^3 fp32 terms), every rerun bit-identical."""
    from rendernet_b200 import ops
    s = dict((n, st) for n, _, st in CONV_LAYERS)[name]
    g = torch.Generator(device=dev).manual_seed(B * 1000 + len(name))
    x = torch.randn(_in_shape(name, B), device=dev, generator=g)
    cout = {n: sh for n, sh, _ in CONV_LAYERS}[name][3]
    side = x.shape[1] * s
    gz = torch.randn((B, side, side, side, cout), device=dev, generator=g)
    dw, db = ops.conv3d_f32_weight_grad(x, gz, s, True)
    dw2, db2 = ops.conv3d_f32_weight_grad(x, gz, s, True)
    same = _bits_equal(dw, dw2) and _bits_equal(db, db2)
    w = torch.zeros(tuple(dw.shape), device=dev, dtype=D64, requires_grad=True)
    b = torch.zeros(cout, device=dev, dtype=D64, requires_grad=True)
    y = orc.conv3d_transpose(x.double(), w, b, (s, s, s), dtype=D64)
    (y * gz.double()).sum().backward()
    del y
    e_w, e_b = _rel(dw, w.grad), _rel(db, b.grad)
    print(f"{name} B={B}: dw {e_w:.2e}, db {e_b:.2e}, bit-identical rerun {same}")
    assert e_w < 2e-5 and e_b < 2e-5 and same


@pytest.mark.parametrize("B", [1, 5, 32])
def test_fc_weight_grad_without_activation_matches_float64(B):
    """g_gc1 (200 -> 16384, no activation): rn_fully_connected_param_grad with z = alpha = NULL gives dW = x^T gy and db = sum_b
    gy; float64 reference, bit-identical rerun.  Measured on an H100 80GB HBM3 (700 W): dW <= 2.3e-7, db <= 2.1e-7."""
    from rendernet_b200 import ops
    g = torch.Generator(device=dev).manual_seed(B)
    x = torch.randn((B, 200), device=dev, generator=g)
    gy = torch.randn((B, 16384), device=dev, generator=g)
    gz, dw, db, da = ops.fully_connected_param_grad(x, gy, None, None, want_gz=True)
    _, dw2, db2, _ = ops.fully_connected_param_grad(x, gy, None, None)
    assert gz is gy and da is None
    e_w, e_b = _rel(dw, x.double().T @ gy.double()), _rel(db, gy.double().sum(0))
    same = _bits_equal(dw, dw2) and _bits_equal(db, db2)
    print(f"g_gc1 B={B}: dW {e_w:.2e}, db {e_b:.2e}, bit-identical rerun {same}")
    assert e_w < 2e-5 and e_b < 2e-5 and same


def test_weight_grad_edges():
    """An all-zero gz gives exactly zero dw and db on both paths; what the kernel cannot run is refused before the launch
    (ValueError) or by the C entry (an error code)."""
    from rendernet_b200 import ops
    from rendernet_b200._lib import RenderNetCudaError
    for name, s in (("g_conv2_g_conv2", 2), ("g_conv5", 1)):
        x = torch.randn(_in_shape(name, 2), device=dev)
        cout = {n: sh for n, sh, _ in CONV_LAYERS}[name][3]
        side = x.shape[1] * s
        dw, db = ops.conv3d_f32_weight_grad(x, torch.zeros((2, side, side, side, cout), device=dev), s, True)
        assert not dw.any() and not db.any(), name
    _, dw, db, _ = ops.fully_connected_param_grad(torch.randn(3, 200, device=dev), torch.zeros(3, 16384, device=dev), None, None)
    assert not dw.any() and not db.any()
    x = torch.zeros((33, 4, 4, 4, 256), device=dev)
    with pytest.raises(ValueError):                                    # B > 32
        ops.conv3d_f32_weight_grad(x, torch.zeros((33, 8, 8, 8, 128), device=dev), 2, True)
    with pytest.raises(ValueError):                                    # gz not on the layer's output grid
        ops.conv3d_f32_weight_grad(x[:2], torch.zeros((2, 4, 4, 4, 128), device=dev), 2, True)
    with pytest.raises(ValueError):                                    # batch mismatch
        ops.conv3d_f32_weight_grad(x[:2], torch.zeros((3, 8, 8, 8, 128), device=dev), 2, True)
    with pytest.raises(ValueError):                                    # more than 512 channels
        ops.conv3d_f32_weight_grad(torch.zeros((1, 4, 4, 4, 520), device=dev), torch.zeros((1, 8, 8, 8, 8), device=dev), 2,
                                   True)
    with pytest.raises(RenderNetCudaError):                           # the 7-bit row coordinates: grids up to 127 a side
        ops.conv3d_f32_weight_grad(torch.zeros((1, 128, 1, 1, 16), device=dev), torch.zeros((1, 128, 1, 1, 16), device=dev), 1,
                                   True)
    with pytest.raises(ValueError):
        ops.fully_connected_param_grad(x[0, 0, 0], torch.zeros(4, 8, device=dev), torch.zeros(4, 8, device=dev), None)


# ----------------------------------------------------------------------------------------- the whole decoder walk
def _decoder64(W, lat):
    """float64 leaves of the 12 decoder variables (npz keys) and the decoder's output at `lat`."""
    Wl = {k: torch.from_numpy(v).to(dev).double().requires_grad_(True) for k, v in W.items()}
    return Wl, decoder_3d(lat, Wl, dtype=D64)


def _tf_name(npz_key):
    for p, t in TF_PREFIX.items():
        if npz_key.startswith(p + "_"):
            return t + "/" + npz_key[len(p) + 1:]
    raise KeyError(npz_key)


@pytest.mark.parametrize("B", [1, 5])
def test_whole_decoder_weight_gradients_match_float64(B):
    """ShapeDecoderGradients.backward(G, want_weight_grads=True): the 12 gradients against float64 autograd of decoder_3d with
    random G; dL/dlatent bit-identical to the call without weight gradients; reruns bit-identical; want_dlatent=False skips the
    latent and keeps the weight gradients.  Measured on an H100 80GB HBM3 (700 W): worst variable 1.2e-6 (B = 1), 1.6e-6
    (B = 5); dL/dlatent 1.0e-6 / 1.6e-6."""
    from rendernet_b200.backward import ShapeDecoderGradients
    W = init_shape_decoder_weights(seed=5)
    z = np.random.default_rng(B).standard_normal((B, 200)).astype(np.float32)
    G = np.random.default_rng(B + 1).standard_normal((B, 64, 64, 64, 1)).astype(np.float32)
    sdg = ShapeDecoderGradients(W, B)
    sdg.forward(z)
    dz0 = sdg.backward(G)
    dz = sdg.backward(G, want_weight_grads=True)
    wg = dict(sdg.weight_grads)
    assert len(wg) == 12
    dz2 = sdg.backward(G, want_weight_grads=True)
    same = np.array_equal(dz.view(np.uint32), dz0.view(np.uint32))
    rerun = np.array_equal(dz2.view(np.uint32), dz.view(np.uint32)) and all(_bits_equal(wg[k], sdg.weight_grads[k]) for k in wg)
    assert sdg.backward(G, want_weight_grads=True, want_dlatent=False) is None
    rerun = rerun and all(_bits_equal(wg[k], sdg.weight_grads[k]) for k in wg)
    lat = torch.tensor(z.astype(np.float64), device=dev, requires_grad=True)
    Wl, ref = _decoder64(W, lat)
    (ref * torch.from_numpy(G).to(dev).double()).sum().backward()
    errs = {k: _rel(wg[_tf_name(k)], Wl[k].grad) for k in W}
    e_lat = _rel(dz, lat.grad)
    worst = max(errs, key=errs.get)
    print(f"shape decoder weight gradients B={B}: worst {worst} {errs[worst]:.2e}, dL/dlatent {e_lat:.2e}; "
          f"dL/dlatent bit-identical to the latent-only walk {same}, reruns bit-identical {rerun}")
    assert same and rerun
    assert max(errs.values()) < 2e-5 and e_lat < 5e-6


# ----------------------------------------------------------------------------------------- nn.ShapeDecoder(trainable=True)
def test_trainable_module_matches_the_gradient_object():
    """Parameter gradients equal ShapeDecoderGradients' bit for bit (one walk gives them and dL/dlatent); 12 parameters keyed
    params.<tf name>; trainable=False records no parameters and gives the latent gradient of today; no_grad records nothing."""
    from rendernet_b200.backward import ShapeDecoderGradients
    from rendernet_b200.nn import ShapeDecoder
    B = 2
    W = init_shape_decoder_weights(seed=7)
    z = np.random.default_rng(8).standard_normal((B, 200)).astype(np.float32)
    G = torch.from_numpy(np.random.default_rng(9).standard_normal((B, 64, 64, 64, 1)).astype(np.float32)).to(dev)
    dec = ShapeDecoder(W, trainable=True)
    keys = sorted(dec.state_dict())
    assert keys == sorted("params." + _tf_name(k) for k in W) and len(keys) == 12
    lat = torch.from_numpy(z).to(dev).requires_grad_()
    (dec(lat) * G).sum().backward()
    sdg = ShapeDecoderGradients(W, B)
    sdg.forward(z)
    dz = sdg.backward(G, want_weight_grads=True, on_device=True)
    for n, p in dec.params.items():
        assert _bits_equal(p.grad, sdg.weight_grads[n]), n
    assert _bits_equal(lat.grad, dz)
    # only the parameters: no latent gradient
    dec.zero_grad()
    (dec(torch.from_numpy(z).to(dev)) * G).sum().backward()
    assert all(_bits_equal(p.grad, sdg.weight_grads[n]) for n, p in dec.params.items())
    # trainable=False: as before
    frozen = ShapeDecoder(W)
    assert len(list(frozen.parameters())) == 0
    lat2 = torch.from_numpy(z).to(dev).requires_grad_()
    (frozen(lat2) * G).sum().backward()
    assert _bits_equal(lat2.grad, torch.from_numpy(sdg.backward(G)).to(dev))
    with torch.no_grad():
        v = dec(lat)
    assert v.grad_fn is None and not v.requires_grad


def test_trainable_module_fits_voxels_and_reports_in_place_edits():
    """A few Adam steps fitting voxels to a fixed target lower the BCE loss; after the steps the forward uses the new weights
    (equal bit for bit to a fresh ShapeDecoder(dec.decoder_weight_dict())); an in-place edit between a forward and its backward
    raises.  Measured on an H100 80GB HBM3 (700 W): BCE 0.701 -> 0.518 after six steps at lr 1e-3."""
    from rendernet_b200.nn import ShapeDecoder
    B = 2
    W = init_shape_decoder_weights(seed=3)
    Wt = init_shape_decoder_weights(seed=4)
    lat = torch.from_numpy(np.random.default_rng(5).standard_normal((B, 200)).astype(np.float32)).to(dev)
    with torch.no_grad():
        target = (ShapeDecoder(Wt)(lat) > 0.5).float()
    dec = ShapeDecoder(W, trainable=True)
    opt = torch.optim.Adam(dec.parameters(), lr=1e-3)
    losses = []
    for _ in range(6):
        opt.zero_grad()
        loss = torch.nn.functional.binary_cross_entropy(dec(lat), target)
        loss.backward()
        opt.step()
        losses.append(float(loss))
    with torch.no_grad():
        final = float(torch.nn.functional.binary_cross_entropy(dec(lat), target))
    print(f"Adam fit of the decoder, BCE per step: {', '.join(f'{v:.4f}' for v in losses)}, final {final:.4f}")
    assert final < 0.9 * losses[0]
    Wn = dec.decoder_weight_dict()
    assert sorted(Wn) == sorted(W) and all(Wn[k].shape == W[k].shape for k in W)
    with torch.no_grad():
        assert torch.equal(dec(lat), ShapeDecoder(Wn)(lat))
    v = dec(lat)
    with torch.no_grad():
        dec.params["g_conv3/g_conv3/weights"].mul_(1.0)
    with pytest.raises(RuntimeError, match="inplace"):
        v.sum().backward()


# ----------------------------------------------------------------------------------------- composed fine-tuning
def _face_setup(seed=61):
    from rendernet_b200.Reconstruct_RenderNet_Face import pretrained_dict_from_texture_weights
    W = orc.init_texture_weights(seed=seed, alpha_range=(-0.3, 0.3), bias_jitter=0.02)
    for k in list(W):
        if k.endswith("/alpha") and "/res" in k:
            W[k] = np.zeros_like(W[k])
    return W, pretrained_dict_from_texture_weights(W), init_shape_decoder_weights(seed + 1)


def _tex_decoder64(z, W, masks):
    def pr(t, name):
        a = torch.from_numpy(W[f"{TE}/{name}/alpha"].astype(np.float64))
        return torch.where(torch.as_tensor(masks[f"{TE}/{name}/alpha"]).reshape(t.shape), t, a * t)
    h = pr(orc.fully_connected(z, W[f"{TE}/e_tex_fc1/fully_connected/weights"], W[f"{TE}/e_tex_fc1/fully_connected/biases"],
                               dtype=D64), "e_tex_fc1").reshape(z.shape[0], 32, 32, 32, 4)
    for name, s, tr in (("e_tex_conv0", 1, True), ("e_tex_conv1", 2, True), ("e_tex_conv2", 1, False)):
        pre = f"{TE}/{name}/{'conv3d_transpose' if tr else 'conv3d'}"
        h = pr((orc.conv3d_transpose if tr else orc.conv3d)(h, W[pre + "/weights"], W[pre + "/biases"], (s, s, s), dtype=D64), name)
    return h


@pytest.mark.parametrize("precision", ["exact", "fast"])
def test_composed_fine_tuning_matches_frozen_kink_oracle(precision):
    """ShapeDecoder(trainable=True) -> TextureRenderer(model="pretrained") -> phong_shade(composite="tf", white background,
    ambient 0, k_diffuse 1) -> per-item MSE summed, at B = 5: the 12 decoder parameter gradients and dL/dlatent of the same walk
    against the float64 chain (float64 decoder with its weights as leaves -> device-cell resampler -> rendernet_texture with the
    device's kinks frozen; the objective in float64 at the device's images).  Bars: those of dL/dlatent in
    test_face_reconstruction_step_matches_frozen_kink_oracle, 3e-4 exact, 6e-3 fast.  Measured on an H100 80GB HBM3 (700 W):
    exact worst variable 6.5e-5 (g_gc1's filter), dL/dlatent 5.8e-5; fast 1.8e-3, 1.4e-3."""
    from rendernet_b200 import tfcompat as tf
    from rendernet_b200.Reconstruct_RenderNet_Face import create_param_center
    from rendernet_b200.backward import TextureInputGradients
    from rendernet_b200.nn import ShapeDecoder, TextureRenderer, phong_shade
    from oracle import phong_tf as pt
    from oracle.frozen_kinks import prelu_kinks, tape_prelu_masks
    B = 5
    W, Wp, Wd = _face_setup()
    rng = np.random.default_rng(62)
    latent = (0.5 + 0.3 * rng.standard_normal((B, 200))).astype(np.float32)
    pose = create_param_center(270, 60, 90, 30).astype(np.float32)
    texture = rng.standard_normal((B, 199)).astype(np.float32)
    light = np.linspace(230, 320, 5).reshape(B, 1).astype(np.float32) * np.float32(math.pi / 180)
    target = rng.random((B, 512, 512, 3)).astype(np.float32)
    el = float(np.float32(105.0 * math.pi / 180))                      # FaceReconstruction's default light elevation
    az = torch.from_numpy(light)
    elt = torch.tensor(np.float32(el))
    ld = torch.cat([torch.sin(elt) * torch.cos(az), torch.sin(elt) * torch.sin(az), torch.cos(elt).expand(B, 1)], 1).to(dev)

    dec = ShapeDecoder(Wd, trainable=True)
    ren = TextureRenderer(Wp, precision=precision, model="pretrained")
    lat = torch.from_numpy(latent).to(dev).requires_grad_()
    tex = torch.from_numpy(texture).to(dev).requires_grad_()
    vox = dec(lat)
    albedo, normal = ren(vox, tex, pose)
    compos = phong_shade(normal, ld, albedo=albedo, composite="tf", background_white=True, ambient=0.0, k_diffuse=1.0)
    loss = ((compos.double() - torch.from_numpy(target).to(dev).double()) ** 2).mean(dim=(1, 2, 3))
    loss.sum().backward()
    pgrads = {n: p.grad.clone() for n, p in dec.params.items()}
    glat = lat.grad.clone()
    vox_d, a1 = vox.detach().clone(), albedo.detach().clone()
    del dec, ren, vox, albedo, normal, compos
    torch.cuda.empty_cache()

    # the device's kinks, from the same network under TF variable names on the same voxels
    tigT = TextureInputGradients(W, B, precision=precision)
    at, nt = tigT.forward(vox_d, texture, pose)
    same_t = torch.equal(at, a1)
    with tf.use_store(tigT.store):
        masks = tape_prelu_masks(tigT.tape)
    a_ = torch.tensor(at.cpu().numpy().astype(np.float64), requires_grad=True)
    n_ = torch.tensor(nt.cpu().numpy().astype(np.float64), requires_grad=True)
    ref = pt.recon_loss(a_, n_, torch.from_numpy(target).double(), pt.tf_generate_light_pos(az.double(), el),
                        torch.ones(B, 3, dtype=D64), with_black_background=False)
    ref.sum().backward()
    del tigT
    torch.cuda.empty_cache()
    minv = orc.inverse_total_matrix(*orc.rotation_around_grid_centroid(pose), 64, 128)
    vt = torch.tensor(vox_d.cpu().numpy().astype(np.float64), requires_grad=True)
    zt = torch.tensor(texture.astype(np.float64))
    mt = torch.tensor(minv.astype(np.float64))
    x = torch.cat([rc.resample(vt, mt, 128), rc.resample(_tex_decoder64(zt, W, masks), mt, 128)], -1)
    with prelu_kinks(W, masks=masks):
        img, nrm = orc.rendernet_texture(x.float(), W)
    (img * a_.grad.float() + nrm * n_.grad.float()).sum().backward()
    latr = torch.tensor(latent.astype(np.float64), device=dev, requires_grad=True)
    Wl, vref = _decoder64(Wd, latr)
    (vref * vt.grad.to(dev)).sum().backward()
    errs = {k: _rel(pgrads[_tf_name(k)], Wl[k].grad) for k in Wd}
    e_lat = _rel(glat, latr.grad)
    worst = max(errs, key=errs.get)
    print(f"[{precision}] composed fine-tuning B=5 vs frozen-kink oracle: worst variable {worst} {errs[worst]:.2e}, "
          f"dL/dlatent {e_lat:.2e}; module forward == texture-model forward {same_t}")
    assert same_t
    bar = 3e-4 if precision == "exact" else 6e-3
    assert e_lat < bar
    for k, e in errs.items():
        assert e < bar, (k, e)
