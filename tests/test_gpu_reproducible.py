"""GPU tests of reproducible inverse rendering under torch.use_deterministic_algorithms(True) (DESIGN §8b): the fixed-order
twins of the resampler backward and of the four image objectives against the float64 device-cell oracle and the atomic kernels,
their invariance to the batch an item is part of and to the run, a NumPy emulation of the fixed-point scatter, non-finite
propagation, the modules and fits end to end, the exact forward under the flag, and the training paths raising or warning.

Every test runs under the flag with CUBLAS_WORKSPACE_CONFIG removed (a device einsum or matmul would then raise) and restores
the flag afterwards.  Bars and poses of the resampler come from tests/test_gpu_resample_backward.py."""
import contextlib
import math
import os

import numpy as np
import pytest
import torch

from oracle import rendernet_oracle as orc
from oracle import resample_cells as rc

pytestmark = pytest.mark.gpu
dev = "cuda"

BAR_DVOX, BAR_DMINV, BAR_DPOSE = 1.2e-6, 5e-6, 2.7e-5
POSES = {"suite": (250.0, 60.0, 3.3), "az0": (0.0, 60.0, 3.3), "az90": (90.0, 60.0, 3.3), "clipped": (300.0, 20.0, 1.8),
         "generic": (45.0, 30.0, 2.5)}


@pytest.fixture(autouse=True)
def deterministic(monkeypatch):
    monkeypatch.delenv("CUBLAS_WORKSPACE_CONFIG", raising=False)
    was, warn_only = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(was, warn_only=warn_only)


@contextlib.contextmanager
def _default_path():
    """The atomic kernels, as without the flag."""
    torch.use_deterministic_algorithms(False)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(True)


def _d(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _rel(got, want):
    got = got.detach().double().cpu().numpy() if isinstance(got, torch.Tensor) else np.asarray(got, np.float64)
    want = want.detach().double().cpu().numpy() if isinstance(want, torch.Tensor) else np.asarray(want, np.float64)
    return float(np.abs(got - want).max() / max(np.abs(want).max(), 1e-300))


def _poses(*names):
    return np.concatenate([orc.compute_pose_param(*POSES[n]) for n in names]).astype(np.float32)


def _minv(poses, size=64, new=128):
    R, S = orc.rotation_around_grid_centroid(poses)
    return orc.inverse_total_matrix(R, S, size, new)


def _chair(B=1):
    bv = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "binvox.npz"))
    vox = np.unpackbits(bv["chair_bits"]).reshape(1, 64, 64, 64, 1).astype(np.float32)
    rng = np.random.default_rng(2)
    return (vox * 0.75 + 0.125 * (rng.random((B, 64, 64, 64, 1)) < 0.02)).astype(np.float32)


def _field(kind, shape, seed):
    rng = np.random.default_rng(seed)
    g = rng.standard_normal(shape)
    if kind == "sparse":
        g *= rng.random(shape) < 0.05
    elif kind == "binades":
        g *= np.exp2(rng.integers(-20, 21, shape))
    return g.astype(np.float32)


def _check_resample(label, poses, got, ref):
    from rendernet_b200.backward import pose_matrix_jacobian_vjp
    dp_got, dp_ref = pose_matrix_jacobian_vjp(poses, got[-1]), pose_matrix_jacobian_vjp(poses, ref[-1])
    for b in range(len(poses)):
        errs = [_rel(g[b], r[b]) for g, r in zip(got[:-1], ref[:-1])]
        e_m, e_p = _rel(got[-1][b], ref[-1][b]), _rel(dp_got[b], dp_ref[b])
        print(f"{label} item {b}: d(vox|tex) {', '.join(f'{e:.2e}' for e in errs)}, dMinv {e_m:.2e}, dpose {e_p:.2e}")
        assert max(errs) < BAR_DVOX and e_m < BAR_DMINV and e_p < BAR_DPOSE, (label, b, errs, e_m, e_p)


def _resample_ref(vox, minv, G, transform=True):
    vt = torch.tensor(vox.astype(np.float64), requires_grad=True)
    mt = torch.tensor(minv.astype(np.float64), requires_grad=True)
    (rc.resample(vt, mt, G.shape[1], transform) * torch.from_numpy(G.astype(np.float64))).sum().backward()
    return vt.grad.numpy(), mt.grad.numpy()


def _resample_twin(vox, minv, G, transform=True):
    from rendernet_b200 import ops
    dv, dm = ops.resample_backward(_d(vox), _d(minv), _d(G), transform)
    return dv.cpu().numpy(), dm.cpu().numpy()


def _resample5_ref(vox, tex, minv, G):
    vt = torch.tensor(vox.astype(np.float64), requires_grad=True)
    tt = torch.tensor(tex.astype(np.float64), requires_grad=True)
    mt = torch.tensor(minv.astype(np.float64), requires_grad=True)
    out = torch.cat([rc.resample(vt, mt, G.shape[1]), rc.resample(tt, mt, G.shape[1])], -1)
    (out * torch.from_numpy(G.astype(np.float64))).sum().backward()
    return vt.grad.numpy(), tt.grad.numpy(), mt.grad.numpy()


def _resample5_twin(vox, tex, minv, G):
    from rendernet_b200 import ops
    return tuple(t.cpu().numpy() for t in ops.resample5_backward(_d(vox), _d(tex), _d(minv), _d(G)))


# ----------------------------------------------------------------------------------------- accuracy against float64
@pytest.mark.parametrize("names,kind", [(("az0", "suite"), "white"), (("clipped",), "sparse"), (("az90", "generic"), "binades")])
def test_resample_twin_matches_float64(names, kind):
    poses = _poses(*names)
    minv, vox = _minv(poses), _chair(len(names))
    G = _field(kind, (len(names), 128, 128, 128, 1), 21)
    _check_resample(f"C=1 {kind}", poses, _resample_twin(vox, minv, G), _resample_ref(vox, minv, G))


def test_resample_twin_four_channels_untransformed():
    poses = _poses("generic")
    minv = _minv(poses)
    vox = np.random.default_rng(13).random((1, 64, 64, 64, 4)).astype(np.float32)
    G = _field("white", (1, 128, 128, 128, 4), 14)
    _check_resample("C=4 transform=0", poses, _resample_twin(vox, minv, G, False), _resample_ref(vox, minv, G, False))


def test_resample5_twin_matches_float64():
    poses = _poses("suite", "az90")
    minv, vox = _minv(poses), _chair(2)
    tex = np.random.default_rng(15).standard_normal((2, 64, 64, 64, 4)).astype(np.float32)
    G = _field("white", (2, 128, 128, 128, 5), 16)
    G[..., 1:] *= 0.01                                          # texture channels far smaller than geometry: own scales
    _check_resample("C=5", poses, _resample5_twin(vox, tex, minv, G), _resample5_ref(vox, tex, minv, G))


# ----------------------------------------------------------------------------------------- fixed-point scatter in NumPy
def test_fixed_point_scatter_matches_numpy_bit_for_bit():
    """16^3 -> 32^3, one item: the sample cells (oracle/resample_cells.py's fp32 emulation), the fp32 weights, w g in fp32,
    scaled by 2^k in double and rounded half-even to int64, summed, and converted back: dvox equal bit for bit."""
    from rendernet_b200._lib import lib
    S, N = 16, 32
    R, Sc = orc.rotation_around_grid_centroid(_poses("generic"))
    minv = orc.inverse_total_matrix(R, Sc, S, N)
    vox = np.random.default_rng(31).random((1, S, S, S, 1)).astype(np.float32)
    G = _field("binades", (1, N, N, N, 1), 32)
    got = _resample_twin(vox, minv, G)[0].reshape(-1)
    c = rc.sample_coords(minv, rc.output_grid(N))[0]                                # [3, P] fp32
    g = G.reshape(-1)
    inside = ((c >= 0) & (c < np.float32(S - 1))).all(0) & (g != 0)
    x, y, z = c[:, inside]
    g = g[inside]
    x0, y0, z0 = np.floor(x), np.floor(y), np.floor(z)
    one = np.float32(1)
    bx, by, bz = x - x0, y - y0, z - z0
    ax, ay, az = (x0 + one) - x, (y0 + one) - y, (z0 + one) - z
    k = lib.rn_fixed_point_exponent(float(np.abs(G).max()), N)
    acc = np.zeros(S ** 3, np.int64)
    i000 = ((z0.astype(np.int64) * S + y0.astype(np.int64)) * S + x0.astype(np.int64))
    for off, wx, wy, wz in ((0, ax, ay, az), (S, ax, by, az), (1, bx, ay, az), (S + 1, bx, by, az), (S * S, ax, ay, bz),
                            (S * S + S, ax, by, bz), (S * S + 1, bx, ay, bz), (S * S + S + 1, bx, by, bz)):
        v = ((wx * wy) * wz) * g                                                      # fp32, the kernel's order
        np.add.at(acc, i000 + off, np.rint(v.astype(np.float64) * 2.0 ** k).astype(np.int64))
    want = (acc.astype(np.float64) * 2.0 ** -k).astype(np.float32)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), int((got != want).sum())


# ----------------------------------------------------------------------------------------- objective twins vs atomic kernels
def _phong_inputs(B, seed, H=128, W=96):
    rng = np.random.default_rng(seed)
    n = rng.random((B, H, W, 3)).astype(np.float32)
    n[:, :2, :2] = 0.5                                                 # the degenerate normal
    a, t, g = (rng.random((B, H, W, 3)).astype(np.float32) for _ in range(3))
    ld = rng.standard_normal((B, 3)).astype(np.float32) + np.float32([0, 0, 2])
    return [_d(v) for v in (a, n, t, g, ld)]


def _objectives(a, n, t, g, ld):
    """{name: outputs} of the six objective calls (per-pixel outputs first, then loss / d_light)."""
    from rendernet_b200 import ops
    lc = torch.ones_like(ld)
    out = {}
    loss, da, dn, dl = ops.phong_recon_loss_grad(a, n, t, ld, lc)
    out["recon"] = ((da, dn), (loss, dl))
    loss, di, dl = ops.phong_composite_loss_grad(n, t, ld)
    out["composite"] = ((di,), (loss, dl))
    for comp in ("tf", "numpy"):
        dn, da, dl = ops.phong_shade_backward(n, g, ld, albedo=a, composite=comp)
        out[f"shade_{comp}"] = ((dn, da), (dl,))
    for kind in ("mse", "bce"):
        loss, di = ops.image_loss_grad_items(a, t, kind)
        out[f"items_{kind}"] = ((di,), (loss,))
    return out


def test_objective_twins_match_the_atomic_kernels():
    """Per-pixel outputs bit-identical; loss and d_light to round-off (loss 1e-12; d_light 1e-4 of scale: the atomic kernel
    sums block partials in fp32 in any order, the twin in double in block order)."""
    args = _phong_inputs(3, 41)
    got = _objectives(*args)
    with _default_path():
        ref = _objectives(*args)
    for name in got:
        for a, b in zip(got[name][0], ref[name][0]):
            assert torch.equal(a, b), name
        for a, b in zip(got[name][1], ref[name][1]):
            e = _rel(a, b)
            print(f"{name}: reduction vs atomic kernel {e:.2e}")
            assert e <= (1e-12 if a.dtype == torch.float64 else 1e-4), (name, e)


# ----------------------------------------------------------------------------------------- invariance
def _batch_invariance(call, make_item, label):
    """call(list of items) -> tuple of per-item tensors [B, ...]; an item alone and at positions 0 and 2 of a batch of three
    (the others different) gives the same bits; so do two calls in a row."""
    x, o1, o2 = make_item(0), make_item(1), make_item(2)
    alone = call([x])
    first = call([x, o1, o2])
    last = call([o1, o2, x])
    again = call([o1, o2, x])
    for i, (s, f, l_, r) in enumerate(zip(alone, first, last, again)):
        assert torch.equal(s[0], f[0]) and torch.equal(s[0], l_[2]), (label, i)
        assert torch.equal(l_, r), (label, i)


def _stack(items, j):
    return torch.stack([it[j] for it in items]).contiguous()


def test_twins_are_batch_and_run_invariant():
    from rendernet_b200 import ops
    rng = np.random.default_rng(51)
    vox1 = [_d(_chair(1)[0] * rng.random()) for _ in range(3)]
    for kind, (C, S, N) in {"resample C=1": (1, 64, 128), "resample C=4": (4, 32, 64)}.items():
        def make(i, C=C, S=S, N=N):
            r = np.random.default_rng(60 + i)
            vox = _d(r.random((S, S, S, C)).astype(np.float32)) if C == 4 else vox1[i]
            minv = _d(_minv(_poses(("suite", "az0", "clipped")[i]), S, N)[0])
            return vox, minv, _d(_field(("white", "binades", "sparse")[i], (N, N, N, C), 70 + i))
        _batch_invariance(lambda its: ops.resample_backward(_stack(its, 0), _stack(its, 1), _stack(its, 2), True), make, kind)

    def make5(i):
        r = np.random.default_rng(80 + i)
        return (vox1[i], _d(r.standard_normal((64, 64, 64, 4)).astype(np.float32)),
                _d(_minv(_poses(("generic", "az90", "suite")[i]))[0]), _d(_field("white", (128, 128, 128, 5), 90 + i)))
    _batch_invariance(lambda its: ops.resample5_backward(*(_stack(its, j) for j in range(4))), make5, "resample5")

    def makep(i):
        return [t[0] for t in _phong_inputs(1, 100 + i)]
    for name in _objectives(*_phong_inputs(1, 99)):
        def call(its, name=name):
            out = _objectives(*(_stack(its, j) for j in range(5)))[name]
            return tuple(out[0]) + tuple(out[1])
        _batch_invariance(call, makep, name)


# ----------------------------------------------------------------------------------------- non-finite G
def test_nonfinite_gradient_poisons_its_item_only():
    from rendernet_b200 import ops
    poses = _poses("suite", "az0", "generic")
    minv, vox = _d(_minv(poses)), _d(_chair(3))
    G = _field("white", (3, 128, 128, 128, 1), 111)
    G[1, 0, 0, 0, 0] = np.inf                                         # a corner point: may lie outside the cube
    dv, dm = ops.resample_backward(vox, minv, _d(G), True)
    tex = _d(np.random.default_rng(112).standard_normal((3, 64, 64, 64, 4)).astype(np.float32))
    G5 = _field("white", (3, 128, 128, 128, 5), 113)
    G5[1, 64, 64, 64, 3] = np.nan
    outs5 = ops.resample5_backward(vox, tex, minv, _d(G5))
    for t in (dv, dm) + tuple(outs5):
        assert not bool(torch.isfinite(t[1]).any())
        assert bool(torch.isfinite(t[0]).all()) and bool(torch.isfinite(t[2]).all())


def test_overflowing_walk_still_retries_and_recovers():
    """The adaptive loss scale sees the twin's NaN and walks again 16x lower, as it does with the atomic kernels."""
    from rendernet_b200.backward import LOSS_SCALE_TARGET, ShaderInputGradients
    vox, poses = _chair(1), _poses("suite")
    G = _d(np.random.default_rng(5).standard_normal((1, 512, 512, 3)).astype(np.float32))
    ig = ShaderInputGradients(orc.init_shader_weights(seed=5, alpha_range=(0.05, 0.3), bias_jitter=0.02), 1)
    ig.forward(vox, poses)
    ig.backward(G)
    sane = ig.last_loss_scale
    ig.scale_target = 2.0 ** 24
    out = ig.backward(G)
    assert ig.last_loss_scale <= 2.0 ** 24 / 16 * sane / LOSS_SCALE_TARGET
    assert all(np.isfinite(a).all() for a in out)


# ----------------------------------------------------------------------------------------- end to end
def _twice_equal(fn):
    a, b = fn(), fn()
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    return a


@pytest.mark.parametrize("precision", ["exact", "fast"])
def test_shader_renderer_through_phong_shade(precision):
    """Voxel, pose and light gradients: equal over two runs, and within the module test's bars of the default path (dvox 2e-6,
    dpose 1e-5 of scale; the light 1e-5)."""
    from rendernet_b200.nn import ShaderRenderer, phong_shade
    B = 2
    m = ShaderRenderer(orc.init_shader_weights(seed=31, alpha_range=(0.05, 0.3), bias_jitter=0.02), precision=precision)
    vox_np, vp_np = _chair(B), _poses("suite", "az90")
    G = _d(np.random.default_rng(3).standard_normal((B, 512, 512, 3)).astype(np.float32))

    def run():
        vox = _d(vox_np).reshape(B, 64, 64, 64).requires_grad_()
        vp = torch.from_numpy(vp_np).requires_grad_()
        ld = torch.tensor([[0.3, 0.5, 1.0], [-0.2, 0.4, 1.0]], device=dev, requires_grad=True)
        (phong_shade(m(vox, vp), ld, composite="numpy", ambient=0.1, k_diffuse=0.9) * G).sum().backward()
        return vox.grad, vp.grad, ld.grad
    got = _twice_equal(run)
    with _default_path():
        ref = run()
    errs = [_rel(a, b) for a, b in zip(got, ref)]
    print(f"[{precision}] fixed-order vs atomic: dvox {errs[0]:.2e}, dpose {errs[1]:.2e}, dlight {errs[2]:.2e}")
    assert errs[0] <= 2e-6 and errs[1] <= 1e-5 and errs[2] <= 1e-5


def _face_setup(seed=61):
    from oracle.shape_decoder import init_shape_decoder_weights
    from rendernet_b200.Reconstruct_RenderNet_Face import pretrained_dict_from_texture_weights
    W = orc.init_texture_weights(seed=seed, alpha_range=(-0.3, 0.3), bias_jitter=0.02)
    for k in list(W):
        if k.endswith("/alpha") and "/res" in k:
            W[k] = np.zeros_like(W[k])
    return pretrained_dict_from_texture_weights(W), init_shape_decoder_weights(seed + 1)


def test_face_chain_through_phong_shade():
    """ShapeDecoder -> TextureRenderer(model="pretrained") -> phong_shade: latent, texture, pose and light gradients equal over
    two runs, within 1e-5 of scale of the default path (tests/test_gpu_nn.py's exact-mode bar)."""
    from rendernet_b200.nn import ShapeDecoder, TextureRenderer, phong_shade
    B = 3
    Wp, Wd = _face_setup()
    dec, ren = ShapeDecoder(Wd), TextureRenderer(Wp, precision="exact", model="pretrained")
    rng = np.random.default_rng(62)
    z, tx = (0.5 + 0.3 * rng.standard_normal((B, 200))).astype(np.float32), rng.standard_normal((B, 199)).astype(np.float32)
    pose = np.array([[math.radians(270 + 10 * i), math.radians(5), 1.0] for i in range(B)], np.float32)
    G = _d(rng.standard_normal((B, 512, 512, 3)).astype(np.float32))

    def run():
        lat, tex = _d(z).requires_grad_(), _d(tx).requires_grad_()
        ps = torch.from_numpy(pose).requires_grad_()
        ld = torch.tensor([[0.3, 0.5, 1.0]] * B, device=dev, requires_grad=True)
        albedo, normal = ren(dec(lat), tex, ps)
        (phong_shade(normal, ld, albedo=albedo, composite="tf", background_white=True) * G).sum().backward()
        return lat.grad, tex.grad, ps.grad, ld.grad
    got = _twice_equal(run)
    with _default_path():
        ref = run()
    errs = [_rel(a, b) for a, b in zip(got, ref)]
    print("face chain fixed-order vs atomic: " + ", ".join(f"{e:.2e}" for e in errs))
    assert max(errs) <= 1e-5


def test_trainable_shape_decoder_is_reproducible():
    from oracle.shape_decoder import init_shape_decoder_weights
    from rendernet_b200.nn import ShapeDecoder
    dec = ShapeDecoder(init_shape_decoder_weights(seed=7), trainable=True)
    z = _d(np.random.default_rng(8).standard_normal((2, 200)).astype(np.float32))
    G = _d(np.random.default_rng(9).standard_normal((2, 64, 64, 64, 1)).astype(np.float32))

    def run():
        dec.zero_grad(set_to_none=True)
        lat = z.clone().requires_grad_()
        (dec(lat) * G).sum().backward()
        return [lat.grad] + [p.grad.clone() for p in dec.params.values()]
    got = _twice_equal(run)
    assert len(got) == 13
    with _default_path():
        ref = run()
    for a, b in zip(got, ref):
        assert torch.equal(a, b)


def test_fits_are_reproducible():
    """A few steps of ShaderPoseFit.run, ShaderShapeFit.run and a shortened FaceReconstruction.run, each twice: every output
    equal."""
    from rendernet_b200.Reconstruct_RenderNet_Face import FaceReconstruction
    from rendernet_b200.RenderNet_demo import compute_pose_param
    from rendernet_b200.shader_fit import ShaderPoseFit
    from rendernet_b200.shape_fit import ShaderShapeFit

    def same(a, b, where="out"):
        if isinstance(a, dict):
            assert a.keys() == b.keys(), where
            for k in a:
                same(a[k], b[k], f"{where}[{k!r}]")
        elif isinstance(a, (list, tuple)):
            assert len(a) == len(b), where
            for i, (x, y) in enumerate(zip(a, b)):
                same(x, y, f"{where}[{i}]")
        else:
            x = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
            y = b.detach().cpu().numpy() if isinstance(b, torch.Tensor) else np.asarray(b)
            assert np.array_equal(x, y, equal_nan=x.dtype.kind == "f"), where

    pose = compute_pose_param(262.0, 54.0, 3.3)[0].astype(np.float32)
    light = np.array([math.radians(280.0), math.radians(60.0)], np.float32)
    fit = ShaderPoseFit(None, _chair(1), objective="phong", inner_step=2, max_epochs=1)
    target = fit.render(dict(pose=np.tile(pose, (5, 1)), light=np.tile(light, (5, 1))))["shaded"]
    init = dict(pose=compute_pose_param(250.0, 60.0, 3.3)[0], light_elevation=math.radians(60.0))
    same(fit.run(target, init=init), fit.run(target, init=init))

    V = 4
    poses = np.concatenate([compute_pose_param(360.0 * k / V, 60.0, 3.3) for k in range(V)]).astype(np.float32)
    lights = np.stack([np.linspace(240, 310, V) * math.pi / 180, np.full(V, math.radians(60.0))], 1)
    sfit = ShaderShapeFit(None, poses, light=lights, batch=V)
    starget = sfit.render(_chair(1).reshape(64, 64, 64))["shaded"]
    same(sfit.run(starget, steps=3), sfit.run(starget, steps=3))

    B = 5
    Wp, Wd = _face_setup(71)
    rec = FaceReconstruction(Wp, Wd, batch=B, precision="exact", inner_step=2, max_epochs=1, seed=3)
    ftarget = np.random.default_rng(72).random((B, 512, 512, 3)).astype(np.float32)
    same(rec.run(ftarget), rec.run(ftarget))


# ----------------------------------------------------------------------------------------- exact forward under the flag
def test_exact_forward_under_the_flag():
    """The exact forward, whose Winograd filter transforms run a float64 einsum on the device the first time each trunk layer is
    used, does not raise under the flag without CUBLAS_WORKSPACE_CONFIG and equals the default forward bit for bit."""
    from rendernet_b200.nn import ShaderRenderer
    W = orc.init_shader_weights(seed=5, alpha_range=(0.05, 0.3), bias_jitter=0.02)
    vox, vp = _d(_chair(1)), _poses("suite")
    img = ShaderRenderer(W, precision="exact")(vox, vp)
    with _default_path():
        ref = ShaderRenderer(W, precision="exact")(vox, vp)
    assert torch.equal(img, ref)


# ----------------------------------------------------------------------------------------- training paths
def test_training_paths_raise_or_warn():
    from rendernet_b200.nn import ShaderRenderer, TextureRenderer
    from rendernet_b200.training import ShaderTrainer, TextureTrainer
    Ws = orc.init_shader_weights(seed=7, alpha_range=(0.05, 0.3), bias_jitter=0.02)
    Wt = orc.init_texture_weights(seed=12, alpha_range=(0.05, 0.3), bias_jitter=0.02)
    vox, vp = _chair(1), _poses("suite")
    rng = np.random.default_rng(14)
    tex = rng.standard_normal((1, 199)).astype(np.float32)
    ti, tn = (rng.random((1, 512, 512, 3)).astype(np.float32) for _ in range(2))
    cases = {
        "ShaderTrainer.step": lambda: ShaderTrainer(Ws, 1, keep_prob=1.0).step(vox, vp, ti),
        "TextureTrainer.step": lambda: TextureTrainer(Wt, 1, keep_prob=1.0).step(vox, tex, vp, ti, tn),
        "ShaderRenderer(trainable=True)": lambda: ShaderRenderer(Ws, trainable=True)(_d(vox), vp).sum().backward(),
        "TextureRenderer(trainable=True)": lambda: sum(t.sum() for t in TextureRenderer(Wt, trainable=True)(
            _d(vox), _d(tex), vp)).backward(),
    }
    for name, fn in cases.items():
        with pytest.raises(RuntimeError, match="deterministic"):
            fn()
        torch.use_deterministic_algorithms(True, warn_only=True)
        with pytest.warns(UserWarning, match="deterministic"):
            fn()
        torch.use_deterministic_algorithms(True)
        torch.cuda.empty_cache()
