"""CPU tests of the face-reconstruction pieces that need no GPU: the float32 / float64 shape-decoder oracle against the reference's
own decoder (tests/golden/shape_decoder.npz), and the outer / inner optimisation loop (Reconstruct_RenderNet_Face.py:304-318,
:455-537) driven by a stub step function against a line-by-line restatement of the reference's loop."""
import math
import os

import numpy as np
import pytest
import torch

from oracle.shape_decoder import decoder_3d, init_shape_decoder_weights

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "shape_decoder.npz")


def test_shape_decoder_oracle_matches_reference_fixture():
    """The oracle's decoder_3d (float32 and float64) against the reference's decoder_3d_pretrained run over the TF-1 shim.
    Measured: float32 3.0e-7, float64 1.7e-7 max abs on outputs in (0.1, 0.9); full-grid sums agree to 4e-9 relative."""
    g = np.load(GOLDEN)
    W = init_shape_decoder_weights(int(g["seed"]))
    assert sorted(k.replace("/", "_") for k in g["var_names"]) == sorted(W)
    for dtype, bar in ((torch.float32, 1e-6), (torch.float64, 6e-7)):
        y = decoder_3d(g["latents"], W, dtype=dtype).numpy()
        assert y.shape == (2, 64, 64, 64, 1)
        e = float(np.abs(y[:, ::3, ::3, ::3] - g["voxels_sub"]).max())
        es = float(np.abs(y.sum(axis=(1, 2, 3, 4), dtype=np.float64) - g["voxels_sum"]).max() / g["voxels_sum"].max())
        ea = float(np.abs(np.abs(y - 0.5).sum(axis=(1, 2, 3, 4), dtype=np.float64) - g["voxels_abs_dev"]).max()
                   / g["voxels_abs_dev"].max())
        print(f"decoder_3d {dtype}: sample max abs err {e:.2e}, sum rel err {es:.2e}, |y - 0.5| sum rel err {ea:.2e}")
        assert e < bar and es < 1e-7 and ea < 1e-6


def test_elu_oracle_boundary_values():
    """TF-1's ELU: exp(x) - 1 below zero (not expm1), the input itself at and above zero (-0 stays -0)."""
    from oracle.shape_decoder import elu
    x = torch.tensor([0.0, -0.0, -1e-30, -1e-7, -100.0, 3.0], dtype=torch.float32)
    y = elu(x).numpy()
    want = np.where(x.numpy() < 0, np.exp(x.numpy().astype(np.float64)) - 1, x.numpy())
    # exp(-1e-7) rounds to 1 - 1 ulp or 1 - 2 ulp depending on the libm: only the rounding of exp may differ
    assert np.abs(y - want).max() <= 1.2e-7
    assert np.signbit(y[1]) and y[0] == 0.0 and not np.signbit(y[2]) and y[2] == 0.0 and y[4] == -1.0 and y[5] == 3.0


# ----------------------------------------------------------------------------------------- the optimisation loop
def _reference_create_param_center(phi_mid=90, phi_range=240, theta_mid=90, theta_range=120, batch_size=5):
    """:304-318, line by line (cfg['batch_size'] -> batch_size)."""
    phi_min = ((phi_mid - phi_range * 0.5) % 360) * math.pi / 180.0
    phi_max = ((phi_mid + phi_range * 0.5) % 360) * math.pi / 180.0
    theta_min = (90 - (theta_mid - theta_range * 0.5)) * math.pi / 180.0
    theta_max = (90 - (theta_mid + theta_range * 0.5)) * math.pi / 180.0
    phi_mid = phi_mid * math.pi / 180.0
    theta_mid = (90 - theta_mid) * math.pi / 180.0
    params = np.zeros(shape=[batch_size, 3], dtype=np.float32)
    params[0] = np.array([phi_min, theta_min, 1.0], dtype=np.float32)
    params[1] = np.array([phi_min, theta_max, 1.0], dtype=np.float32)
    params[2] = np.array([phi_mid, theta_mid, 1.0], dtype=np.float32)
    params[3] = np.array([phi_max, theta_min, 1.0], dtype=np.float32)
    params[4] = np.array([phi_max, theta_max, 1.0], dtype=np.float32)
    return params


class _StubSession:
    """A deterministic stand-in for the TF graph: variables (latent, pose, texture, light), a loss that depends on all four, and a
    train op that moves each variable by a fixed fraction toward a per-item optimum."""

    def __init__(self, seed):
        rng = np.random.default_rng(seed)
        self.opt = dict(latent=rng.standard_normal((5, 200)).astype(np.float32), pose=rng.uniform(0, 3, (5, 3)).astype(np.float32),
                        texture=rng.standard_normal((5, 199)).astype(np.float32), light=rng.uniform(3, 6, (5, 1)).astype(np.float32))

    def loss(self, v):
        return sum(((np.asarray(v[k], np.float64) - self.opt[k]) ** 2).reshape(5, -1).mean(1) * w
                   for k, w in (("latent", 1.0), ("pose", 3.0), ("texture", 0.5), ("light", 2.0)))

    def train(self, v):
        return {k: (v[k] - np.float32(0.3) * (v[k] - self.opt[k])).astype(np.float32) for k in v}


def _reference_loop(sess, max_epochs, inner_step, tex_first, log):
    """:451-537, line by line, with the stub session in place of sess.run; tex_first = the first epoch's texture draw."""
    best_param = np.zeros(shape=(3))
    best_vector = np.zeros(shape=(200))
    best_tex = np.zeros(shape=(199))
    best_light = None
    phi_range = 60
    theta_range = 30
    for i in range(max_epochs):
        if i == 0:
            params_batch = _reference_create_param_center(phi_mid=270, phi_range=phi_range, theta_mid=90, theta_range=theta_range)
            vector_batch = np.ones((5, 200)) * 0.5
            tex_batch = tex_first
            light_batch = np.expand_dims((np.linspace(230, 320, num=5) * math.pi / 180.0), axis=0).T
        else:
            phi_range /= 2
            theta_range /= 2
            params_batch = _reference_create_param_center(phi_mid=best_param[0], phi_range=phi_range, theta_mid=best_param[1],
                                                          theta_range=theta_range)
            vector_batch = np.tile(best_vector[np.newaxis, :], (5, 1))
            tex_batch = np.tile(best_tex[np.newaxis, :], (5, 1))
            light_batch = np.tile(best_light[np.newaxis, :], (5, 1))
        for idx in range(inner_step):
            if idx == 0:                     # assign ops: float32 variables
                v = dict(latent=vector_batch.astype(np.float32), pose=params_batch.astype(np.float32),
                         texture=tex_batch.astype(np.float32), light=light_batch.astype(np.float32))
                log.append(("assign", i, {k: a.copy() for k, a in v.items()}))
            v = sess.train(v)
            if idx == (inner_step - 1):
                recon_loss_out = sess.loss(v)
                z_out, param_out, tex_out, light_out = v["latent"], v["pose"], v["texture"], v["light"]
                best_vector = z_out[np.argmin(recon_loss_out)]
                best_tex = tex_out[np.argmin(recon_loss_out)]
                best_light = light_out[np.argmin(recon_loss_out)]
                best_param = param_out[np.argmin(recon_loss_out)] * 180. / math.pi
                best_param = np.array([best_param[0], 90 - best_param[1], 1])
                log.append(("best", i, int(np.argmin(recon_loss_out)), best_param.copy()))
    return best_vector, best_tex, best_light, best_param


@pytest.mark.parametrize("seed,max_epochs,inner_step", [(0, 3, 2), (1, 10, 1), (7, 4, 5)])
def test_reconstruction_loop_matches_reference_restatement(seed, max_epochs, inner_step):
    """Hypotheses, first-epoch initialisation, best-of-batch selection, degree / radian conversions and range halving of
    reconstruction_loop against the reference's loop restated line by line, both driven by the same stub session."""
    from rendernet_b200.Reconstruct_RenderNet_Face import create_param_center, reconstruction_loop
    sess = _StubSession(100 + seed)
    target = object()
    seen = []

    def step_fn(state, tgt):
        assert tgt is target
        if not seen or seen[-1][0] == "best":
            seen.append(("assign", {k: a.copy() for k, a in state.items()}))
        return sess.train(state), sess.loss(state), None

    def loss_fn(state, tgt):
        return sess.loss(state)

    calls = []

    def callback(epoch, idx, state, loss, sel):
        calls.append((epoch, idx, sel))
        if sel is not None:
            seen.append(("best", int(np.argmin(sel))))

    out = reconstruction_loop(step_fn, loss_fn, target, max_epochs=max_epochs, inner_step=inner_step, seed=seed, callback=callback)
    log = []
    tex_first = np.random.default_rng(seed).standard_normal((5, 199))
    bv, bt, bl, bp = _reference_loop(sess, max_epochs, inner_step, tex_first, log)

    assigns = [e for e in log if e[0] == "assign"]
    bests = [e for e in log if e[0] == "best"]
    got_assigns = [e[1] for e in seen if e[0] == "assign"]
    got_bests = [e[1] for e in seen if e[0] == "best"]
    assert len(assigns) == len(got_assigns) == max_epochs and len(calls) == max_epochs * inner_step
    for (_, i, want), got in zip(assigns, got_assigns):
        for k in want:
            assert got[k].dtype == np.float32 and np.array_equal(got[k], want[k]), (i, k)
    assert got_bests == [b[2] for b in bests]
    assert np.array_equal(out["latent"], bv) and np.array_equal(out["texture"], bt) and np.array_equal(out["light"], bl)
    assert np.array_equal(out["best_param"], bp) and out["best_index"] == bests[-1][2]
    assert len(out["best_loss"]) == max_epochs
    # the first epoch's hypotheses: azimuth 240..300 degrees, elevation +-15 degrees, scale 1
    p0 = assigns[0][2]["pose"]
    assert np.allclose(np.degrees(p0[:, 0]), [240, 240, 270, 300, 300], atol=1e-4)
    assert np.allclose(np.degrees(p0[:, 1]), [15, -15, 0, 15, -15], atol=1e-4) and np.all(p0[:, 2] == 1)
    assert np.allclose(np.degrees(assigns[0][2]["light"][:, 0]), np.linspace(230, 320, 5), atol=1e-4)
    assert np.all(assigns[0][2]["latent"] == 0.5)
    # later epochs: the window halves around the previous best pose
    for e in range(1, max_epochs):
        prev = bests[e - 1][3]
        want = create_param_center(prev[0], 60 / 2 ** e, prev[1], 30 / 2 ** e)
        assert np.array_equal(assigns[e][2]["pose"], want)


def test_reconstruction_loop_rejects_other_batch_sizes():
    from rendernet_b200.Reconstruct_RenderNet_Face import create_param_center, reconstruction_loop
    with pytest.raises(ValueError):
        reconstruction_loop(lambda s, t: (s, np.zeros(4), None), lambda s, t: np.zeros(4), None, batch_size=4)
    with pytest.raises(ValueError):
        create_param_center(batch_size=6)
