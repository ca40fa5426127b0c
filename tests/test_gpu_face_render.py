"""GPU tests of the shaded, relit face: rn_phong_shade (the demo's NumPy composite and TensorFlow's composite, times an albedo),
TextureRenderEngine(phong=..., model=...) with a per-step light, and FaceReconstruction.render.

The TensorFlow composite is held to tests/golden/phong_tf.npz (the reference's own tools/Phong_shading.py over the NumPy shim of
TF-1) and, bit for bit, to the image rn_phong_recon_loss_grad measures; the NumPy composite to rn_phong_composite bit for bit and
to tests/golden/phong.npz."""
import math
import os

import numpy as np
import pytest
import torch

from oracle import rendernet_oracle as orc

pytestmark = pytest.mark.gpu
dev = "cuda"


def _d(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _normals(B, H, W, seed):
    """Random normal maps in [0,1] plus black (0) and white (1) background pixels, exact 0 / 1 components, pixels on the kinks
    of light (0,0,2) (u.L = 1 and u.L = 0), mask transitions and n = (0.5, 0.5, 0.5), which is shaded as unlit."""
    rng = np.random.default_rng(seed)
    n = rng.random((B, H, W, 3)).astype(np.float32)
    n[:, 0, :8] = 0.0
    n[:, 1, :8] = 1.0
    n[:, 2, :8] = [0.0, 1.0, 0.5]
    n[:, 2, 8:16] = [1.0, 0.0, 1.0]
    n[:, 3, :8] *= 0.05
    n[:, 4, :8] = 0.97 + 0.03 * n[:, 4, :8]
    n[:, 5, 0:8] = [0.5, 0.5, 0.75]
    n[:, 5, 8:16] = [0.75, 0.5, 0.5]
    n[:, 6, :8] = 0.5
    return n


def _lights(B, seed):
    rng = np.random.default_rng(seed)
    ld = np.concatenate([[[0.0, 0.0, 2.0]], rng.standard_normal((B - 1, 3))]).astype(np.float32)[:B]
    return ld, rng.uniform(0.5, 1.2, (B, 3)).astype(np.float32)


def _u8(x):
    return np.clip(np.float32(255) * np.asarray(x, np.float32), 0, 255).astype(np.uint8)


# ----------------------------------------------------------------------------------------- the NumPy composite
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("white", [False, True])
@pytest.mark.parametrize("mask", [False, True])
def test_numpy_composite_is_rn_phong_composite(B, white, mask):
    """No albedo: shade, compos and uint8 equal rn_phong_composite bit for bit.  With an albedo: compos is the fp32 product of the
    albedo and the kernel's own shading, and the uint8 image its clip(255 x) truncation."""
    from rendernet_b200 import ops
    n = _d(_normals(B, 32, 48, 1 + B))
    ld, lc = (_d(a) for a in _lights(B, 2))
    ref, ref8 = ops.phong_composite(n, ld, lc, 0.1, 0.9, background_white=white, with_mask=mask, want_u8=True)
    shade, compos, u8 = ops.phong_shade(n, ld, lc, 0.1, 0.9, composite="numpy", background_white=white, with_mask=mask)
    assert torch.equal(shade, ref) and compos is shade and torch.equal(u8, ref8)
    a = np.random.default_rng(3).random((B, 32, 48, 3)).astype(np.float32)
    s2, c2, u2 = (t.cpu().numpy() for t in ops.phong_shade(n, ld, lc, 0.1, 0.9, albedo=_d(a), composite="numpy",
                                                           background_white=white, with_mask=mask))
    assert np.array_equal(s2, ref.cpu().numpy())
    assert np.array_equal(c2, a * s2)
    assert np.array_equal(u2, _u8(c2))


def test_numpy_composite_matches_reference_golden(golden_dir):
    """compos against the reference's float64 np_phong_composite (tests/golden/phong.npz) times the albedo: <= 1e-6 wherever
    the mask is saturated.  Where it is not (|s| < 15 for the mask sigmoid(s), s = 255 |n| - 150 or 255 |1 - n| - 80), the fp32
    arithmetic of phong_pixel multiplies the rounding of |n| by 255: measured on an H100 80GB HBM3, 3.2e-6 there; bar 5e-6."""
    from rendernet_b200 import ops
    g = np.load(os.path.join(golden_dir, "phong.npz"))
    nm = g["normal_map"].astype(np.float64)
    a = np.random.default_rng(4).random(g["normal_map"].shape).astype(np.float32)
    for key, white in (("composite", False), ("composite_white", True)):
        _, c, u8 = ops.phong_shade(_d(g["normal_map"]), g["light"], (1.0, 1.0, 1.0), 0.1, 0.9, albedo=_d(a), composite="numpy",
                                   background_white=white, with_mask=True)
        err = np.abs(c.cpu().numpy().astype(np.float64) - a * g[key]).max(axis=-1)
        s = 255 * np.linalg.norm(1 - nm, axis=-1) - 80 if white else 255 * np.linalg.norm(nm, axis=-1) - 150
        edge = np.abs(s) < 15
        e_sat, e_edge = float(err[~edge].max()), float(err[edge].max()) if edge.any() else 0.0
        print(f"numpy composite ({key}) x albedo vs float64 reference: saturated mask {e_sat:.2e}, "
              f"{int(edge.sum())} transition pixels {e_edge:.2e}")
        assert e_sat <= 1e-6 and e_edge <= 5e-6 and edge.mean() < 0.2
        assert np.array_equal(u8.cpu().numpy(), _u8(c.cpu().numpy()))


# ----------------------------------------------------------------------------------------- the TensorFlow composite
def test_tf_composite_matches_reference_golden(golden_dir):
    """rn_phong_shade(composite="tf") and Phong_shading.tf_phong_composite (NumPy in -> NumPy out, CUDA in -> CUDA out) against
    the reference's TensorFlow composite: max abs < 2e-6, and the clip boundary exact_light_k1 hits comes out as exactly 1.0."""
    from rendernet_b200 import Phong_shading
    d = np.load(os.path.join(golden_dir, "phong_tf.npz"))
    nm, light, col, amb, kd = d["normal_map"], d["light"], d["light_col"], float(d["ambient"]), float(d["k_diffuse"])
    for name, black, mask in (("white_mask", False, True), ("black_mask", True, True), ("no_mask", False, False)):
        got = Phong_shading.tf_phong_composite(nm, light, col, amb, kd, with_black_background=black, with_mask=mask)
        assert isinstance(got, np.ndarray) and got.dtype == np.float32
        on_dev = Phong_shading.tf_phong_composite(_d(nm), light, col, amb, kd, with_black_background=black, with_mask=mask)
        assert on_dev.is_cuda and np.array_equal(on_dev.cpu().numpy(), got)
        e = float(np.abs(got.astype(np.float64) - d[name]).max())
        print(f"tf composite {name} vs reference: {e:.2e}")
        assert e < 2e-6, name
    got = Phong_shading.tf_phong_composite(nm, light, np.ones((1, 3)), 0.0, 1.0, with_mask=False)
    e = float(np.abs(got.astype(np.float64) - d["exact_light_k1"]).max())
    print(f"tf composite exact_light_k1 vs reference: {e:.2e}")
    assert e < 2e-6
    ones = d["exact_light_k1"] == 1.0
    assert ones.sum() >= 4 and (got[ones] == 1.0).all()


@pytest.mark.parametrize("black,mask,ambient,kd", [(False, True, 0.0, 1.0), (True, True, 0.1, 0.9), (False, False, 0.0, 1.0),
                                                   (False, False, 0.1, 0.9)])
def test_tf_shading_is_the_image_the_loss_measures(black, mask, ambient, kd):
    """Albedo 1 and target = the kernel's tf shading: rn_phong_recon_loss_grad returns loss 0 and d_normal 0 at every pixel
    (bit-identical images).  A random albedo against target 0: the loss is the float64 mean of compos^2 (1e-6 relative)."""
    from rendernet_b200 import ops
    B = 2
    n = _d(_normals(B, 64, 64, 12))
    ld, lc = (_d(a) for a in _lights(B, 13))
    shade, _, _ = ops.phong_shade(n, ld, lc, ambient, kd, composite="tf", background_white=not black, with_mask=mask,
                                  want_compos=False, want_u8=False)
    loss, _, dn, _ = ops.phong_recon_loss_grad(torch.ones_like(n), n, shade, ld, lc, ambient, kd, black, mask)
    assert (loss == 0).all(), loss
    assert (dn == 0).all(), int((dn != 0).sum())
    a = _d(np.random.default_rng(14).random((B, 64, 64, 3)).astype(np.float32))
    _, compos, _ = ops.phong_shade(n, ld, lc, ambient, kd, albedo=a, composite="tf", background_white=not black, with_mask=mask)
    loss, *_ = ops.phong_recon_loss_grad(a, n, torch.zeros_like(n), ld, lc, ambient, kd, black, mask)
    want = (compos.double() ** 2).mean(dim=(1, 2, 3))
    e = float(((loss - want).abs() / want).max())
    print(f"loss vs float64 mean of compos^2: {e:.2e}")
    assert e <= 1e-6


def test_light_rows_and_u8():
    """One light row stands for the batch; the uint8 image is clip(255 compos) truncated."""
    from rendernet_b200 import ops
    B = 3
    n = _d(_normals(B, 16, 16, 15))
    a = _d(np.random.default_rng(16).random((B, 16, 16, 3)).astype(np.float32))
    one = np.array([[0.3, -0.2, 0.9]], np.float32)
    s1, c1, u1 = ops.phong_shade(n, one, (1.0, 0.9, 0.8), 0.05, 0.95, albedo=a)
    s3, c3, u3 = ops.phong_shade(n, np.repeat(one, B, 0), np.repeat([[1.0, 0.9, 0.8]], B, 0), 0.05, 0.95, albedo=a)
    assert torch.equal(s1, s3) and torch.equal(c1, c3) and torch.equal(u1, u3)
    assert np.array_equal(u1.cpu().numpy(), _u8(c1.cpu().numpy()))


def test_malformed_input_raises():
    from rendernet_b200 import ops
    n = torch.rand(3, 8, 8, 3, device=dev)
    with pytest.raises(ValueError):
        ops.phong_shade(n, torch.ones(2, 3))
    with pytest.raises(ValueError):
        ops.phong_shade(n, torch.ones(1, 3), light_col=torch.ones(2, 3))
    with pytest.raises(ValueError):
        ops.phong_shade(n, torch.ones(1, 3), composite="opengl")
    with pytest.raises(ValueError):
        ops.phong_shade(n, torch.ones(1, 3), albedo=torch.rand(3, 8, 4, 3, device=dev))


# ----------------------------------------------------------------------------------------- TextureRenderEngine(phong=...)
PHONG = dict(light_dir=np.array([[0.4, 0.5, 0.77]], np.float32), light_col=(1.0, 0.95, 0.9), ambient=0.05, k_diffuse=0.9)


@pytest.fixture(scope="module")
def bench_case():
    import bench
    vox, poses = bench.synthetic_batch(24)
    return vox, bench.synthetic_texture(24), poses, {}


def _equal(got, want, label):
    got, want = torch.as_tensor(np.asarray(got)), torch.as_tensor(np.asarray(want))
    d = got != want
    if d.any():
        print(f"{label}: {int(d.sum())} values differ, items {sorted({int(i) for i in d.nonzero()[:, 0]})}")
    assert not d.any(), label


@pytest.mark.parametrize("composite", ["tf", "numpy"])
@pytest.mark.parametrize("precision", ["exact", "fast"])
def test_engine_phong_b24(bench_case, precision, composite):
    """On the bench's inputs (B = 24, seeded weights): albedo and normal equal an engine without phong bit for bit; compos and
    compos_u8 equal ops.phong_shade on those maps; B = 24 equals three B = 8 shards and B = 1 renders; submit/result ships the
    uint8 image of render; the step is the unshaded step plus one launch."""
    from rendernet_b200 import ops
    from rendernet_b200.engine import TextureRenderEngine
    vox, tex, poses, cache = bench_case
    if precision not in cache:
        eng = TextureRenderEngine(None, 24, precision=precision)
        cache[precision] = ([t.clone() for t in eng.render(vox, tex, poses)], eng.launches_per_step)
        del eng
        torch.cuda.empty_cache()
    (plain_a, plain_n), plain_launches = cache[precision]
    phong = dict(PHONG, composite=composite)
    eng = TextureRenderEngine(None, 24, precision=precision, phong=phong)
    assert eng.launches_per_step == plain_launches + 1
    out = [t.clone() for t in eng.render(vox, tex, poses)]
    assert len(out) == 4 and out[3].dtype == torch.uint8
    _equal(out[0], plain_a, "albedo vs unshaded engine")
    _equal(out[1], plain_n, "normal vs unshaded engine")
    _, c, u8 = ops.phong_shade(_d(out[1]), phong["light_dir"], phong["light_col"], phong["ambient"], phong["k_diffuse"],
                               albedo=_d(out[0]), composite=composite, background_white=True, with_mask=True)
    _equal(out[2], c.cpu(), "compos vs ops.phong_shade")
    _equal(out[3], u8.cpu(), "compos_u8 vs ops.phong_shade")
    _equal(eng.result(eng.submit(vox, tex, poses)), out[3], "submit/result uint8")
    del eng
    torch.cuda.empty_cache()
    for Bs, items in ((8, [slice(0, 8), slice(8, 16), slice(16, 24)]), (1, [slice(0, 1), slice(9, 10), slice(23, 24)])):
        eng = TextureRenderEngine(None, Bs, precision=precision, phong=phong)
        for sl in items:
            got = eng.render(vox[sl], tex[sl], poses[sl])
            for k, name in enumerate(("albedo", "normal", "compos", "compos_u8")):
                _equal(got[k], out[k][sl], f"B={Bs} {sl} {name}")
        del eng
        torch.cuda.empty_cache()


def test_engine_per_step_light():
    """Two lights alternated over four steps, synchronously (render / upload + step_device) and through submit/result with two
    steps in flight: each step equals a freshly built engine with that light, bit for bit; light_dir=None is the engine's own."""
    from rendernet_b200.engine import TextureRenderEngine
    B = 2
    rng = np.random.default_rng(21)
    vox = (rng.random((B, 64, 64, 64, 1)) < 0.2).astype(np.float32)
    tex = rng.standard_normal((B, 199)).astype(np.float32)
    poses = np.array([orc.compute_pose_param(30.0, 60.0, 3.3)[0], orc.compute_pose_param(200.0, 40.0, 3.0)[0]], np.float32)
    lights = [np.array([[0.4, 0.5, 0.77], [-0.3, 0.8, 0.2]], np.float32), np.array([[-0.9, 0.1, 0.3]], np.float32)]
    refs = []
    for L in lights:
        eng = TextureRenderEngine(None, B, precision="fast", phong=dict(light_dir=L))
        refs.append([t.clone() for t in eng.render(vox, tex, poses)])
        del eng
    assert not torch.equal(refs[0][3], refs[1][3])
    eng = TextureRenderEngine(None, B, precision="fast", phong=dict(light_dir=lights[0]))
    for i in range(4):
        got = eng.render(vox, tex, poses, light_dir=lights[i % 2])
        for k in range(4):
            _equal(got[k], refs[i % 2][k], f"sync step {i} output {k}")
    eng.upload(vox, tex, poses)                                 # None: the light given at construction
    eng.step_device()
    _equal(eng.out[2].cpu(), refs[0][2], "light_dir=None")
    tickets, got = [], {}
    for i in range(4):
        tickets.append(eng.submit(vox, tex, poses, light_dir=lights[i % 2]))
        if i >= 1:
            got[i - 1] = eng.result(tickets[i - 1]).clone()
    got[3] = eng.result(tickets[3]).clone()
    for i in range(4):
        _equal(got[i], refs[i % 2][3], f"pipelined step {i}")
    with pytest.raises(ValueError):
        eng.render(vox, tex, poses, light_dir=np.ones((3, 3), np.float32))


@pytest.mark.parametrize("precision", ["exact", "fast"])
def test_engine_pretrained_model(precision):
    """model="pretrained" on the npz-keyed re-keying of W equals model="texture" on W bit for bit, on all four outputs (W with
    zero residual-block slopes: the pretrained network uses ReLU there)."""
    from rendernet_b200.engine import TextureRenderEngine
    from rendernet_b200.Reconstruct_RenderNet_Face import pretrained_dict_from_texture_weights
    B = 2
    W = orc.init_texture_weights(seed=31, alpha_range=(-0.3, 0.3), bias_jitter=0.02)
    for k in list(W):
        if k.endswith("/alpha") and "/res" in k:
            W[k] = np.zeros_like(W[k])
    rng = np.random.default_rng(32)
    vox = (rng.random((B, 64, 64, 64, 1)) < 0.2).astype(np.float32)
    tex = rng.standard_normal((B, 199)).astype(np.float32)
    poses = np.array([orc.compute_pose_param(120.0, 50.0, 3.3)[0], orc.compute_pose_param(300.0, 70.0, 2.8)[0]], np.float32)
    phong = dict(light_dir=np.array([[0.2, 0.9, 0.4]], np.float32))
    a = TextureRenderEngine(W, B, precision=precision, phong=phong)
    ref = [t.clone() for t in a.render(vox, tex, poses)]
    del a
    b = TextureRenderEngine(pretrained_dict_from_texture_weights(W), B, precision=precision, model="pretrained", phong=phong)
    got = b.render(vox, tex, poses)
    for k, name in enumerate(("albedo", "normal", "compos", "compos_u8")):
        _equal(got[k], ref[k], f"pretrained vs texture {name}")


# ----------------------------------------------------------------------------------------- FaceReconstruction.render
def test_face_reconstruction_render():
    """At a state: albedo and normal equal tig.forward, the per-item mean((target - compos)^2) equals rec.loss (1e-6 relative),
    compos = albedo * shading.  At a novel pose and light: equals TextureRenderEngine(model="pretrained", phong=...) bit for bit."""
    from rendernet_b200.engine import TextureRenderEngine
    from rendernet_b200.Reconstruct_RenderNet_Face import (FaceReconstruction, create_param_center, light_pos,
                                                            pretrained_dict_from_texture_weights)
    from oracle.shape_decoder import init_shape_decoder_weights
    B = 5
    W = orc.init_texture_weights(seed=61, alpha_range=(-0.3, 0.3), bias_jitter=0.02)
    for k in list(W):
        if k.endswith("/alpha") and "/res" in k:
            W[k] = np.zeros_like(W[k])
    Wp, Wd = pretrained_dict_from_texture_weights(W), init_shape_decoder_weights(62)
    rec = FaceReconstruction(Wp, Wd, batch=B)
    rng = np.random.default_rng(63)
    state = dict(latent=(0.5 + 0.3 * rng.standard_normal((B, 200))).astype(np.float32), pose=create_param_center(270, 60, 90, 30),
                 texture=rng.standard_normal((B, 199)).astype(np.float32),
                 light=np.linspace(230, 320, 5).reshape(B, 1).astype(np.float32) * np.float32(math.pi / 180))
    out = rec.render(state)
    assert set(out) == {"albedo", "normal", "shading", "compos", "compos_u8", "voxels"}
    assert out["voxels"].shape == (B, 64, 64, 64) and out["compos_u8"].dtype == np.uint8
    vox = rec.sdg.forward(state["latent"])
    a, n = rec.tig.forward(vox, state["texture"], state["pose"])
    assert np.array_equal(out["albedo"], a.cpu().numpy()) and np.array_equal(out["normal"], n.cpu().numpy())
    assert np.array_equal(out["compos"], out["albedo"] * out["shading"])
    assert np.array_equal(out["compos_u8"], _u8(out["compos"]))
    target = rng.random((B, 512, 512, 3)).astype(np.float32)
    loss = rec.loss(state, target)
    mse = ((target.astype(np.float64) - out["compos"]) ** 2).mean(axis=(1, 2, 3))
    e = float((np.abs(mse - loss) / loss).max())
    print(f"render: mean((target - compos)^2) vs rec.loss: {e:.2e}")
    assert e <= 1e-6

    vp = np.array([orc.compute_pose_param(az, 70.0, 3.3)[0] for az in (10, 80, 150, 220, 290)], np.float32)
    laz = np.linspace(0.3, 2.5, B).reshape(B, 1).astype(np.float32)
    nov = rec.render(state, view_params=vp, light_azimuth=laz)
    assert not np.array_equal(nov["albedo"], out["albedo"])
    eng = TextureRenderEngine(Wp, B, precision="exact", model="pretrained",
                              phong=dict(light_dir=light_pos(laz, rec.elevation)))
    got = eng.render(nov["voxels"][..., None], state["texture"], vp)
    for k, name in enumerate(("albedo", "normal", "compos", "compos_u8")):
        _equal(got[k], nov[name], f"render vs engine {name}")
