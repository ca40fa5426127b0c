"""Host tests of the shading-parameter gradients (light colour and ambient term), no GPU:
  - the float64 reference (tests/phong_params_ref.py) repeats oracle/phong_vjp.py's results and its d_light_col / d_ambient
    match central differences of its own float64 forward, for both composites, mask on and off, black and white backgrounds;
  - which C entry point each ops wrapper calls and with what (a recording stand-in for the library, as
    test_reproducible_host.py does), and how the wrappers and nn.phong_shade refuse malformed colour / ambient arguments;
  - with fit_shading off, ShaderPoseFit.step / pose_search and FaceReconstruction.step / reconstruction_loop build exactly the
    states and calls they built before the option existed; with it on, the colour and ambient join the state, descend with
    their own eta and are projected onto colour >= 0, 0 <= ambient <= 1."""
import math

import numpy as np
import pytest
import torch

from oracle import phong_vjp
from rendernet_b200 import ops
from phong_params_ref import np_vjp64, tf_vjp64

RNG = np.random.default_rng(7)


def _pixels(B=3, H=6, W=7):
    return RNG.uniform(0.02, 0.98, (B, H, W, 3))


# ------------------------------------------------------------------------------------------------ the float64 reference
CASES = [(comp, mask, bg) for comp in ("tf", "numpy") for mask in (False, True) for bg in (False, True)]


def _vjp(comp, n, ld, lc, amb, kd, bg, mask, g, albedo):
    if comp == "tf":                        # tf_vjp64 takes `black`, the kernels' !white
        return tf_vjp64(n, ld, lc, amb, kd, not bg, mask, g, albedo)
    return np_vjp64(n, ld, lc, amb, kd, bg, mask, g, albedo)


@pytest.mark.parametrize("comp,mask,bg", CASES)
def test_reference_repeats_the_oracle(comp, mask, bg):
    n, g, alb = _pixels(), RNG.standard_normal((3, 6, 7, 3)), _pixels()
    ld, lc = np.array([[0.3, 0.8, 0.5]]), np.array([[0.8, 0.6, 0.5]])
    old = (phong_vjp.tf_vjp64(n, ld, lc, 0.2, 0.9, not bg, mask, g, alb) if comp == "tf" else
           phong_vjp.np_vjp64(n, ld, lc, 0.2, 0.9, bg, mask, g, alb))
    new = _vjp(comp, n, ld, lc, 0.2, 0.9, bg, mask, g, alb)
    for a, b in zip(old, new[:4]):
        np.testing.assert_array_equal(a, b)
    per_item = _vjp(comp, n, ld, lc, np.full(3, 0.2), 0.9, bg, mask, g, alb)       # [B] ambient: the same numbers
    for a, b in zip(new, per_item):
        np.testing.assert_array_equal(a, b)


@pytest.mark.parametrize("comp,mask,bg", CASES)
def test_reference_matches_central_differences(comp, mask, bg):
    """L = sum g * compos as a function of (light_col, ambient), per item; pixels within 1e-3 of a clip edge or of d = 0 get
    g = 0, so no difference straddles a kink (h = 1e-6).  Relative agreement 1e-7 of the gradient's scale."""
    B = 3
    n, alb = _pixels(B, 16, 16), _pixels(B, 16, 16)
    ld = np.array([[0.3, 0.8, 0.5], [-0.4, 0.7, 0.6], [0.1, 0.2, 0.9]])
    lc = np.array([[0.8, 0.6, 0.5], [1.0, 1.0, 1.0], [0.5, 0.9, 0.7]])
    amb = np.array([0.2, 0.05, 0.4])
    kd = 0.9

    def fwd(lc_, amb_, g_):
        shade = _vjp(comp, n, ld, lc_, amb_, kd, bg, mask, g_, None)[0]
        return (g_ * alb * shade).sum(axis=(1, 2, 3))

    # keep pixels away from the kinks the parameters move across
    L = ld / np.linalg.norm(ld, axis=1, keepdims=True)
    v = n - 0.5
    d = (v / np.linalg.norm(v, axis=-1, keepdims=True) * L[:, None, None, :]).sum(-1, keepdims=True)
    pre = kd * np.maximum(d, 0) * lc[:, None, None, :]
    far = (np.abs(d) > 1e-3) & (np.abs(pre - 1) > 1e-3).all(-1, keepdims=True)
    shade = _vjp(comp, n, ld, lc, amb, kd, bg, mask, np.ones_like(n), None)[0]
    far &= ((shade > 1e-3) & (shade < 1 - 1e-3)).all(-1, keepdims=True)
    g = RNG.uniform(-0.5, 1.5, n.shape) * far                                  # biased: the sums do not cancel
    assert far.mean() > 0.3
    got = _vjp(comp, n, ld, lc, amb, kd, bg, mask, g * alb, None)
    d_col, d_amb = got[4], got[5]
    h = 1e-6
    fd_col = np.zeros((B, 3))
    for c in range(3):
        e = np.zeros((B, 3))
        e[:, c] = h
        fd_col[:, c] = (fwd(lc + e, amb, g) - fwd(lc - e, amb, g)) / (2 * h)
    fd_amb = (fwd(lc, amb + h, g) - fwd(lc, amb - h, g)) / (2 * h)
    scale = np.abs(g).sum(axis=(1, 2, 3))
    assert np.abs(d_col - fd_col).max() < 1e-7 * scale.max()
    assert np.abs(d_amb - fd_amb).max() < 1e-7 * scale.max()
    assert np.abs(d_amb).min() > 1e-2 * scale.min() and np.abs(d_col).max() > 1e-2 * scale.min()     # not vacuous


# ------------------------------------------------------------------------------------------------ which entry point runs
class _Spy:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def fn(*args):
            self.calls.append((name, args))
            return 64 if name.endswith("_workspace") else 0
        return fn

    def names(self):
        return [n for n, _ in self.calls]


@pytest.fixture
def spy(monkeypatch):
    s = _Spy()
    monkeypatch.setattr(ops, "lib", s)
    monkeypatch.setattr(ops, "_cuda", lambda t, dtype=None: t.contiguous())
    monkeypatch.setattr(ops, "_stream", lambda: 0)
    return s


@pytest.fixture
def flag():
    was, warn_only = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    yield torch.use_deterministic_algorithms
    torch.use_deterministic_algorithms(was, warn_only=warn_only)


def _t(*shape):
    return torch.rand(shape, dtype=torch.float32)


def _calls(amb, want):
    n, a, tgt, g = _t(2, 4, 8, 3), _t(2, 4, 8, 3), _t(2, 4, 8, 3), _t(2, 4, 8, 3)
    light = torch.tensor([[0.3, 0.4, 1.0]])
    kw = dict(want_shading_grad=True) if want else {}
    return dict(recon=ops.phong_recon_loss_grad(a, n, tgt, light, torch.ones(1, 3), amb, **kw),
                composite=ops.phong_composite_loss_grad(a, tgt, light, ambient=amb, **kw),
                shade=ops.phong_shade_backward(n, g, light, ambient=amb, albedo=a, **kw),
                fwd=ops.phong_shade(n, light, ambient=amb, albedo=a))


def test_float_ambient_without_keyword_calls_todays_entries(spy, flag):
    flag(False)
    r = _calls(0.25, False)
    assert spy.names() == ["rn_phong_recon_loss_grad", "rn_phong_composite_loss_grad", "rn_phong_shade_backward", "rn_phong_shade"]
    assert [len(r[k]) for k in ("recon", "composite", "shade", "fwd")] == [4, 3, 3, 3]


@pytest.mark.parametrize("fixed", [False, True])
def test_keyword_calls_the_params_entries(spy, flag, fixed):
    flag(fixed)
    r = _calls(0.25, True)
    suffix = "_fixed" if fixed else ""
    names = [n for n in spy.names() if not n.endswith("_workspace")]
    assert names == ["rn_phong_recon_loss_grad_params" + suffix, "rn_phong_composite_loss_grad_params" + suffix,
                     "rn_phong_shade_backward_params" + suffix, "rn_phong_shade"]
    args = dict(spy.calls)
    loss, da, dn, dl, dcol, damb = r["recon"]
    ra = args["rn_phong_recon_loss_grad_params" + suffix]
    assert ra[6:9] == (1.0, 0, 1) and ra[9:15] == (loss.data_ptr(), da.data_ptr(), dn.data_ptr(), dl.data_ptr(), dcol.data_ptr(),
                                                   damb.data_ptr())
    assert dcol.shape == (2, 3) and damb.shape == (2,)
    assert not fixed or args["rn_phong_recon_loss_grad_params_fixed_workspace"] == (2, 4, 8)
    if not fixed:
        assert not dcol.any() and not damb.any()                               # accumulated into: zeroed first
    loss, dimg, dl, dcol, damb = r["composite"]
    ca = args["rn_phong_composite_loss_grad_params" + suffix]
    assert ca[5:8] == (pytest.approx(0.9), 0, 1) and ca[8:13] == (loss.data_ptr(), dimg.data_ptr(), dl.data_ptr(),
                                                                  dcol.data_ptr(), damb.data_ptr())
    dn, da, dl, dcol, damb = r["shade"]
    sa = args["rn_phong_shade_backward_params" + suffix]
    assert sa[5:9] == (1.0, 1, 1, 1) and sa[10:15] == (dn.data_ptr(), da.data_ptr(), dl.data_ptr(), dcol.data_ptr(), damb.data_ptr())


def test_ambient_array_holds_the_float_or_the_rows(spy, flag, monkeypatch):
    flag(False)
    seen = []
    real = ops._ambient_array
    monkeypatch.setattr(ops, "_ambient_array", lambda *a: seen.append(real(*a)) or seen[-1])
    _calls(0.25, True)
    assert all(torch.equal(a, torch.full((2,), 0.25)) for a in seen) and len(seen) == 3
    spy.calls.clear()
    r = _calls(torch.tensor([0.3]), False)                                    # a tensor: the per-item entries, today's tuples
    assert spy.names() == ["rn_phong_recon_loss_grad_params", "rn_phong_composite_loss_grad_params",
                           "rn_phong_shade_backward_params", "rn_phong_shade_ambient"]
    assert [len(r[k]) for k in ("recon", "composite", "shade", "fwd")] == [4, 3, 3, 3]
    assert all(a[13:15] == (None, None) for n, a in spy.calls if n == "rn_phong_shade_backward_params")
    assert ops._ambient_rows(torch.tensor([0.1, 0.2]), 2, "cpu").tolist() == pytest.approx([0.1, 0.2])
    assert ops._ambient_rows(torch.tensor(0.5, dtype=torch.float64), 2, "cpu").tolist() == [0.5, 0.5]


def test_wrappers_refuse_malformed_ambient(spy):
    n = _t(2, 4, 8, 3)
    for bad in (torch.ones(3), torch.ones(2, 1), torch.ones(1, 2)):
        with pytest.raises(ValueError, match="ambient"):
            ops.phong_shade_backward(n, n, (0, 0, 1), ambient=bad, want_shading_grad=True)
        with pytest.raises(ValueError, match="ambient"):
            ops.phong_composite_loss_grad(n, n, (0, 0, 1), ambient=bad)
        with pytest.raises(ValueError, match="ambient"):
            ops.phong_shade(n, (0, 0, 1), ambient=bad)
    with pytest.raises(TypeError, match="ambient"):
        ops.phong_recon_loss_grad(n, n, n, torch.ones(1, 3), torch.ones(1, 3), torch.ones(2, dtype=torch.int32))
    with pytest.raises(ValueError, match="light_col"):
        ops.phong_shade_backward(n, n, (0, 0, 1), light_col=torch.ones(3, 3), want_shading_grad=True)
    assert spy.calls == []


def test_nn_phong_shade_refuses_malformed_shading():
    from rendernet_b200.nn import phong_shade
    n = torch.rand(2, 4, 4, 3)                                                 # CPU: the checks below come first
    ld = torch.ones(1, 3)
    for kw in (dict(light_col=torch.ones(3, 3)), dict(light_col=torch.ones(2, 4)), dict(light_col=torch.ones(3)),
               dict(ambient=torch.ones(3)), dict(ambient=torch.ones(2, 1))):
        with pytest.raises(ValueError):
            phong_shade(n, ld, **kw)
    with pytest.raises(TypeError, match="light_col"):
        phong_shade(n, ld, light_col=torch.ones(1, 3, dtype=torch.int64))
    with pytest.raises(TypeError, match="ambient"):
        phong_shade(n, ld, ambient=torch.ones(2, dtype=torch.int32))
    with pytest.raises(TypeError, match="normal"):                             # well formed: the normal map must be on CUDA
        phong_shade(n, ld, light_col=torch.ones(2, 3, requires_grad=True), ambient=torch.zeros(1, requires_grad=True))


def test_c_entries_check_their_arguments():
    from rendernet_b200._lib import lib
    f = 256                                                                    # never dereferenced: the checks come first
    assert lib.rn_phong_shade_ambient(f, None, f, f, None, 1.0, 1, 1, 1, f, None, None, 1, 4, 4, None) == -1
    assert lib.rn_phong_shade_backward_params(f, None, f, f, None, 1.0, 1, 1, 1, f, f, None, None, None, None, 1, 4, 4, None) == -1
    assert lib.rn_phong_shade_backward_params(f, None, f, f, f, 1.0, 2, 1, 1, f, f, None, None, None, None, 1, 4, 4, None) == -1
    assert lib.rn_phong_recon_loss_grad_params(f, f, f, f, f, None, 1.0, 0, 1, f, f, f, None, None, None, 1, 4, 4, None) == -1
    assert lib.rn_phong_composite_loss_grad_params(f, f, f, f, None, 0.9, 0, 1, f, f, None, None, None, 1, 4, 4, None) == -1
    assert lib.rn_phong_composite_loss_grad_params(f, f, f, f, f, 0.9, 0, 1, f, f, None, None, None, 0, 4, 4, None) == -1
    for q in (lib.rn_phong_recon_loss_grad_params_fixed_workspace, lib.rn_phong_composite_loss_grad_params_fixed_workspace,
              lib.rn_phong_shade_backward_params_fixed_workspace):
        assert q(2, 512, 512) == 8 * 2 * 1024 * 8 and q(0, 4, 4) < 0
    # a workspace smaller than the query: -4, before any launch
    assert lib.rn_phong_composite_loss_grad_params_fixed(f, f, f, f, f, 0.9, 0, 1, f, f, None, f, None, 2, 16, 16, f, 64,
                                                         None) == -4
    assert lib.rn_phong_shade_backward_params_fixed(f, None, f, f, f, 1.0, 1, 1, 1, f, f, None, None, None, f, 2, 16, 16, f, 8,
                                                    None) == -4


# ------------------------------------------------------------------------------------------------ the fits
def _shader_fit(fit_shading, monkeypatch, record):
    from rendernet_b200 import shader_fit as sf
    fit = sf.ShaderPoseFit.__new__(sf.ShaderPoseFit)                           # no device: the gradients are a stand-in
    fit.B, fit.objective, fit.fit_scale, fit.voxels, fit.ig, fit.device = 5, "phong", False, None, None, "cpu"
    fit.eta = dict(pose=0.01, light=0.4)
    fit.fit_shading = fit_shading
    if fit_shading:
        fit.eta["shading"] = 0.5
    fit.phong = dict(light_col=sf.PHONG_DEFAULTS["light_col"], ambient=0.1, k_diffuse=0.9, background_white=False,
                     with_mask=True)
    fit._target = None

    def grads(ig, voxels, pose, target, objective, **kw):
        record.append(kw)
        g = dict(pose=np.full((5, 3), 0.5), light=np.full((5, 2), 0.25), voxels=None)
        if kw.get("want_shading_grad"):
            g.update(light_col=np.tile([[-0.3, 2.0, 0.1]], (5, 1)), ambient=np.array([-5.0, 5.0, 0.1, -0.1, 0.0]))
        return np.arange(5.0), g
    monkeypatch.setattr(sf, "shader_fit_gradients", grads)
    return fit


def test_shader_fit_without_shading_is_unchanged(monkeypatch):
    from rendernet_b200.shader_fit import PHONG_DEFAULTS, ShaderPoseFit
    record = []
    fit = _shader_fit(False, monkeypatch, record)
    state = dict(pose=np.zeros((5, 3), np.float32), light=np.ones((5, 2), np.float32))
    new, loss, g = fit.step(state, torch.zeros(1))
    assert set(new) == {"pose", "light"} and set(g) == {"pose", "light", "voxels"}
    (kw,) = record                                                            # today's call: the constants, no new keyword
    assert set(kw) == {"light", *fit.phong} and kw["light"] is state["light"]
    assert all(kw[k] == v for k, v in fit.phong.items())
    assert fit.initial_shading() is None
    import inspect
    sig = inspect.signature(ShaderPoseFit.__init__).parameters
    assert sig["fit_shading"].default is False and PHONG_DEFAULTS["ambient"] == 0.1


def test_shader_fit_with_shading_projects(monkeypatch):
    record = []
    fit = _shader_fit(True, monkeypatch, record)
    state = dict(pose=np.zeros((5, 3), np.float32), light=np.ones((5, 2), np.float32), **fit.initial_shading())
    assert state["light_col"].shape == (5, 3) and np.all(state["light_col"] == 1) and np.all(state["ambient"] == np.float32(0.1))
    new, _, _ = fit.step(state, torch.zeros(1))
    kw = record[0]
    assert kw["want_shading_grad"] is True and kw["light_col"].shape == (5, 3) and tuple(kw["ambient"].shape) == (5,)
    want_col = np.maximum(np.float32(1) - np.float32(0.5) * np.float32([-0.3, 2.0, 0.1]), 0).astype(np.float32)
    np.testing.assert_array_equal(new["light_col"], np.tile(want_col, (5, 1)))
    want_amb = np.clip(np.float32(0.1) - np.float32(0.5) * np.float32([-5.0, 5.0, 0.1, -0.1, 0.0]), 0, 1)
    np.testing.assert_array_equal(new["ambient"], want_amb)
    assert new["ambient"][0] == 1 and new["ambient"][1] == 0 and new["light_col"][0, 1] == 0


def test_shader_fit_refuses_shading_without_phong():
    from rendernet_b200.shader_fit import ShaderPoseFit
    with pytest.raises(ValueError, match="fit_shading"):
        ShaderPoseFit(None, np.zeros((64, 64, 64), np.float32), objective="mse", fit_shading=True)


class _Bowl:
    """Plain descent on a quadratic bowl in every state entry; records the states it is handed."""

    def __init__(self, keys):
        self.keys, self.calls = keys, []

    def loss(self, state, target):
        return sum(((np.asarray(state[k], np.float64).reshape(5, -1) - 0.3) ** 2).sum(1) for k in self.keys if k in state)

    def step(self, state, target):
        self.calls.append({k: np.array(v) for k, v in state.items()})
        new = {k: (np.asarray(v, np.float32) - np.float32(0.1) * (np.asarray(v, np.float32) - np.float32(0.3))).astype(np.float32)
               for k, v in state.items()}
        return new, self.loss(state, target), {}


def test_pose_search_carries_the_shading_only_when_given():
    from rendernet_b200.shader_fit import pose_search
    lights = np.tile([[4.0, 1.0]], (5, 1)).astype(np.float32)
    init = [math.radians(262.0), math.radians(36.0), 1.0]
    a, b = _Bowl(["pose", "light"]), _Bowl(["pose", "light", "light_col", "ambient"])
    out_a = pose_search(a.step, a.loss, None, init, light=lights, max_epochs=2, inner_step=2)
    assert set(out_a) == {"pose", "light", "best_param", "best_index", "best_loss", "windows", "state"}
    assert all(set(c) == {"pose", "light"} for c in a.calls)
    shading = dict(light_col=np.tile([[1.0, 0.5, 0.2]], (5, 1)), ambient=np.linspace(0.0, 0.4, 5))
    out_b = pose_search(b.step, b.loss, None, init, light=lights, max_epochs=2, inner_step=2, shading=shading)
    np.testing.assert_array_equal(b.calls[0]["light_col"], shading["light_col"].astype(np.float32))
    j = out_b["best_index"]
    sel_amb = out_b["state"]["ambient"][j]
    assert out_b["ambient"] == sel_amb and np.array_equal(out_b["light_col"], out_b["state"]["light_col"][j])
    assert np.all(b.calls[2]["ambient"] == b.calls[2]["ambient"][0])            # epoch 2 restarts all five from one value
    for k in ("pose", "light"):                                                 # the shading leaves the rest untouched
        np.testing.assert_array_equal(b.calls[0][k], a.calls[0][k])


def _face(fit_shading, monkeypatch, record):
    from rendernet_b200 import Reconstruct_RenderNet_Face as rf
    rec = rf.FaceReconstruction.__new__(rf.FaceReconstruction)
    rec.B, rec.device, rec.elevation, rec._target = 5, "cpu", 0.3, None
    rec.eta = dict(latent=0.8, pose=0.01, texture=0.8, light=0.4)
    rec.fit_shading = fit_shading
    if fit_shading:
        rec.eta["shading"] = 0.5

    class _Sdg:
        def forward(self, latent):
            return "vox"

        def backward(self, dvox):
            return np.full((5, 200), 0.1)
    rec.sdg, rec.tig = _Sdg(), None

    def grads(tig, vox, texture, pose, light, target, elevation, **kw):
        record.append(kw)
        out = (np.arange(5.0), None, np.full((5, 199), 0.1), np.full((5, 3), 0.1), np.full((5, 1), 0.1))
        if kw.get("want_shading_grad"):
            out += (np.tile([[0.4, -0.2, 3.0]], (5, 1)), np.full(5, -0.5))
        return out
    monkeypatch.setattr(rf, "reconstruction_gradients", grads)
    return rec


def _face_state():
    return dict(latent=np.zeros((5, 200), np.float32), pose=np.zeros((5, 3), np.float32), texture=np.zeros((5, 199), np.float32),
                light=np.zeros((5, 1), np.float32))


def test_face_reconstruction_without_shading_is_unchanged(monkeypatch):
    record = []
    rec = _face(False, monkeypatch, record)
    new, _, g = rec.step(_face_state(), torch.zeros(1))
    assert set(new) == {"latent", "pose", "texture", "light"} and set(g) == set(new)
    assert record == [dict(dvox_on_device=True)]                             # today's call: the reference's shading
    assert rec.initial_shading() is None


def test_face_reconstruction_with_shading_projects(monkeypatch):
    record = []
    rec = _face(True, monkeypatch, record)
    state = dict(_face_state(), **rec.initial_shading())
    assert np.all(state["light_col"] == 1) and np.all(state["ambient"] == 0)     # the reference's white light, ambient 0
    new, _, g = rec.step(state, torch.zeros(1))
    assert record[0]["want_shading_grad"] is True and tuple(record[0]["ambient"].shape) == (5,)
    np.testing.assert_array_equal(new["light_col"], np.tile(np.maximum(np.float32(1) - np.float32(0.5) *
                                                                       np.float32([0.4, -0.2, 3.0]), 0), (5, 1)))
    np.testing.assert_array_equal(new["ambient"], np.full(5, 0.25, np.float32))


def test_reconstruction_loop_carries_the_shading_only_when_given():
    from rendernet_b200.Reconstruct_RenderNet_Face import reconstruction_loop
    a, b = _Bowl(["pose", "light"]), _Bowl(["pose", "light", "light_col", "ambient"])
    out_a = reconstruction_loop(a.step, a.loss, None, max_epochs=2, inner_step=2)
    assert set(out_a) == {"latent", "texture", "light", "pose", "best_param", "best_index", "best_loss", "state"}
    assert all(set(c) == {"latent", "pose", "texture", "light"} for c in a.calls)
    shading = dict(light_col=np.ones((5, 3)), ambient=np.zeros(5))
    out_b = reconstruction_loop(b.step, b.loss, None, max_epochs=2, inner_step=2, shading=shading)
    for k in ("latent", "pose", "texture", "light"):
        np.testing.assert_array_equal(b.calls[0][k], a.calls[0][k])
    j = out_b["best_index"]
    assert out_b["ambient"] == out_b["state"]["ambient"][j] and out_b["light_col"].shape == (3,)
    assert np.all(b.calls[2]["light_col"] == b.calls[2]["light_col"][0])
