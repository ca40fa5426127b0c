"""CPU tests of the Shader pose / light fit (rendernet_b200/shader_fit.py): the float64 restatement of the demo's composite
(oracle/phong_np.py) against the reference's fixture, the light-angle Jacobian, argument checks before anything reaches a device,
and the hypothesis search driven by a fake step function."""
import math
import os

import numpy as np
import pytest
import torch

from oracle import phong_np as pn


def test_phong_np_oracle_matches_reference_golden(golden_dir):
    """oracle/phong_np.py against the reference's np_phong_composite (tests/golden/phong.npz).  The fixture was computed from an
    fp32 normal map in fp32: where the mask is saturated the two agree to 7e-8; on the mask's transition (|s| < 15 for
    sigmoid(s)) the fixture's fp32 |n| rounding, times 255, moves it by up to 2.7e-6."""
    g = np.load(os.path.join(golden_dir, "phong.npz"))
    nm, L = torch.from_numpy(g["normal_map"]).double(), torch.from_numpy(g["light"]).double()
    for key, white in (("composite", False), ("composite_white", True)):
        got = pn.np_phong_composite(nm, L, torch.ones(2, 3, dtype=torch.float64), 0.1, 0.9, white, True).numpy()
        err = np.abs(got - g[key]).max(-1)
        edge = np.abs(pn.np_mask_arg(nm, white).numpy()[..., 0]) < 15
        assert err[~edge].max() < 2e-7, key
        assert (err[edge].max() if edge.any() else 0.0) < 5e-6, key


def test_mask_value_override_keeps_the_float64_derivative():
    n = torch.rand(1, 4, 4, 3, dtype=torch.float64) * 0.6
    n.requires_grad_(True)
    L, col = torch.tensor([[0.3, 0.4, 1.2]], dtype=torch.float64), torch.ones(1, 3, dtype=torch.float64)
    a = pn.np_phong_composite(n, L, col, 0.1, 0.9)
    ga, = torch.autograd.grad(a.sum(), n)
    m = torch.sigmoid(pn.np_mask_arg(n.detach())).float().double()          # rounded to fp32
    b = pn.np_phong_composite(n, L, col, 0.1, 0.9, mask_value=m)
    gb, = torch.autograd.grad(b.sum(), n)
    assert torch.equal(ga, gb) and (a - b).abs().max() < 1e-7


def test_light_jacobian_matches_finite_difference():
    from rendernet_b200.shader_fit import light_dir, light_dir_jacobian
    from rendernet_b200.Phong_shading import generate_light_pos
    rng = np.random.default_rng(0)
    light = np.stack([rng.uniform(0, 2 * math.pi, 7), rng.uniform(-1.5, 1.5, 7)], 1)
    J = light_dir_jacobian(light)
    h = 1e-6
    for k in range(2):
        e = np.zeros(2)
        e[k] = h

        def f(x):
            L = np.asarray(x, np.float64)
            return np.stack([-np.sin(L[:, 1]) * np.cos(L[:, 0]), np.cos(L[:, 1]), -np.sin(L[:, 1]) * np.sin(L[:, 0])], 1)
        fd = (f(light + e) - f(light - e)) / (2 * h)
        assert np.abs(fd - J[:, :, k]).max() < 1e-8
    # the map is the demo's generate_light_pos (degrees in, elevation first), rounded to fp32
    for az, el in ((250.0, 60.0), (10.0, 120.0)):
        want = generate_light_pos(el, az).astype(np.float32)
        assert np.abs(light_dir([[math.radians(az), math.radians(el)]]) - want).max() <= 1e-7
    assert np.array_equal(light_dir(light), pn.generate_light_pos(torch.from_numpy(light)).numpy().astype(np.float32))


def test_wrappers_refuse_malformed_input():
    from rendernet_b200 import ops
    img = torch.rand(2, 8, 8, 3)
    with pytest.raises(ValueError):
        ops.phong_composite_loss_grad(torch.rand(2, 8, 8, 1), torch.rand(2, 8, 8, 1), torch.ones(1, 3))
    with pytest.raises(ValueError):
        ops.phong_composite_loss_grad(img, torch.rand(2, 8, 4, 3), torch.ones(1, 3))
    with pytest.raises(ValueError):
        ops.phong_composite_loss_grad(img, img, torch.ones(3, 3))              # light rows not in {1, B}
    with pytest.raises(ValueError):
        ops.phong_composite_loss_grad(img, img, torch.ones(1, 3), light_col=np.ones((2, 4)))
    with pytest.raises(RuntimeError):                                          # well formed, but no CPU path
        ops.phong_composite_loss_grad(img, img, torch.ones(1, 3))
    with pytest.raises(ValueError):
        ops.image_loss_grad_items(img, img, "l1")
    with pytest.raises(ValueError):
        ops.image_loss_grad_items(torch.rand(2, 8, 8, 2), torch.rand(2, 8, 8, 2))
    with pytest.raises(ValueError):
        ops.image_loss_grad_items(img, torch.rand(2, 8, 8, 1))
    with pytest.raises(RuntimeError):
        ops.image_loss_grad_items(img, img, "bce")


def test_c_entries_check_their_arguments():
    from rendernet_b200._lib import lib
    fake = 256                                                                 # never dereferenced: the checks come first
    assert lib.rn_phong_composite_loss_grad(None, fake, fake, fake, 0.1, 0.9, 0, 1, fake, fake, None, 1, 4, 4, None) == -1
    assert lib.rn_phong_composite_loss_grad(fake, fake, fake, fake, 0.1, 0.9, 0, 1, fake, None, None, 1, 4, 4, None) == -1
    assert lib.rn_phong_composite_loss_grad(fake, fake, fake, fake, 0.1, 0.9, 0, 1, fake, fake, None, 0, 4, 4, None) == -1
    assert lib.rn_image_loss_grad_items(fake, fake, None, fake, 16, 2, 1, 0, None) == -1     # C = 2
    assert lib.rn_image_loss_grad_items(fake, fake, None, fake, 16, 3, 1, 2, None) == -1     # kind 2
    assert lib.rn_image_loss_grad_items(fake, fake, None, None, 16, 3, 1, 0, None) == -1
    assert lib.rn_image_loss_grad_items(fake, fake, None, fake, 16, 1, 0, 0, None) == -1


def _grey_weights():
    return {"encoder/e_conv11/weights": np.zeros((4, 4, 1, 16), np.float32)}


def test_fit_refuses_bad_arguments_before_the_device():
    from rendernet_b200.shader_fit import ShaderPoseFit, check_objective
    vox = np.zeros((64, 64, 64), np.float32)
    with pytest.raises(ValueError):
        ShaderPoseFit(None, vox, batch=4)
    with pytest.raises(ValueError):
        ShaderPoseFit(None, vox, objective="l1")
    with pytest.raises(ValueError):
        ShaderPoseFit(_grey_weights(), vox, objective="phong")                # greyscale network: no normal map to shade
    with pytest.raises(ValueError):
        ShaderPoseFit(None, vox, objective="phong", is_greyscale=True)
    with pytest.raises(ValueError):
        ShaderPoseFit(_grey_weights(), vox, objective="bce", is_greyscale=False)
    with pytest.raises(ValueError):
        ShaderPoseFit(None, np.zeros((3, 64, 64, 64)), objective="mse")
    check_objective("bce", True)
    check_objective("mse", True)


class _FakeFit:
    """A quadratic bowl around a hidden pose and light, steps of plain descent: enough to drive the search logic."""

    def __init__(self, pose, light):
        self.pose, self.light, self.calls = np.asarray(pose, np.float64), np.asarray(light, np.float64), []

    def loss(self, state, target):
        d = ((np.asarray(state["pose"], np.float64)[:, :2] - self.pose[:2]) ** 2).sum(1)
        if "light" in state:
            d = d + 0.1 * ((np.asarray(state["light"], np.float64) - self.light) ** 2).sum(1)
        return d

    def step(self, state, target):
        self.calls.append({k: np.array(v) for k, v in state.items()})
        loss = self.loss(state, target)
        g = dict(pose=np.zeros((5, 3)))
        g["pose"][:, :2] = 2 * (np.asarray(state["pose"], np.float64)[:, :2] - self.pose[:2])
        new = dict(pose=(state["pose"] - np.float32(0.1) * g["pose"].astype(np.float32)).astype(np.float32))
        if "light" in state:
            g["light"] = 0.2 * (np.asarray(state["light"], np.float64) - self.light)
            new["light"] = (state["light"] - np.float32(0.1) * g["light"].astype(np.float32)).astype(np.float32)
        return new, loss, g


def test_search_halves_the_window_and_keeps_the_argmin():
    from rendernet_b200.Reconstruct_RenderNet_Face import create_param_center
    from rendernet_b200.shader_fit import in_window, pose_search
    init = np.array([math.radians(250.0), math.radians(30.0), 1.1])
    fake = _FakeFit([math.radians(262.0), math.radians(36.0), 1.1], [math.radians(280.0), math.radians(50.0)])
    lights = np.stack([np.linspace(230, 320, 5) * math.pi / 180, np.full(5, math.radians(60.0))], 1).astype(np.float32)
    seen = []
    out = pose_search(fake.step, fake.loss, None, init, light=lights, max_epochs=3, inner_step=2,
                      callback=lambda e, i, s, loss, sel: seen.append((e, i, None if sel is None else sel.copy(),
                                                                       {k: v.copy() for k, v in s.items()})))
    assert len(fake.calls) == 6 and len(seen) == 6
    w = out["windows"]
    assert [x["phi_range"] for x in w] == [60.0, 30.0, 15.0] and [x["theta_range"] for x in w] == [30.0, 15.0, 7.5]
    assert w[0]["phi_mid"] == pytest.approx(250.0) and w[0]["theta_mid"] == pytest.approx(60.0)
    # epoch 0 starts from create_param_center around the initial guess, with its scale, and the given lights
    want = create_param_center(250.0, 60, 60.0, 30)
    want[:, 2] = np.float32(1.1)
    assert np.allclose(fake.calls[0]["pose"], want) and np.array_equal(fake.calls[0]["light"], lights)
    for e in range(3):
        sel = seen[2 * e + 1][2]
        state = seen[2 * e + 1][3]
        j = int(np.argmin(sel))
        assert seen[2 * e][2] is None and sel is not None
        np.testing.assert_array_equal(sel, fake.loss(state, None))              # re-evaluated after the last inner step
        if e + 1 < 3:                                                          # the next epoch restarts around the argmin
            nxt = fake.calls[2 * (e + 1)]
            assert w[e + 1]["phi_mid"] == pytest.approx(math.degrees(state["pose"][j][0]), abs=1e-9)
            assert w[e + 1]["theta_mid"] == pytest.approx(90 - math.degrees(state["pose"][j][1]), abs=1e-9)
            assert np.allclose(nxt["pose"][2, :2], state["pose"][j][:2], atol=1e-6)         # the centre hypothesis
            assert (nxt["pose"][:, 2] == state["pose"][j][2]).all()
            assert (nxt["light"] == state["light"][j]).all()
    j = out["best_index"]
    assert j == int(np.argmin(seen[-1][2])) and out["best_loss"][-1] == seen[-1][2].min()
    assert np.array_equal(out["pose"], seen[-1][3]["pose"][j]) and np.array_equal(out["light"], seen[-1][3]["light"][j])
    assert out["best_loss"][2] < out["best_loss"][0]
    assert in_window(out["pose"], w[-1], slack_deg=2.0)


def test_search_without_light_and_its_checks():
    from rendernet_b200.shader_fit import in_window, pose_search
    fake = _FakeFit([math.radians(5.0), math.radians(0.0), 1.0], [0.0, 0.0])
    out = pose_search(fake.step, fake.loss, None, [math.radians(355.0), 0.0, 1.0], max_epochs=2, inner_step=1)
    assert out["light"] is None and "light" not in out["state"]
    # the azimuth window wraps at 360 degrees
    assert in_window([math.radians(3.0), 0.0, 1.0], dict(phi_mid=355.0, phi_range=30.0, theta_mid=90.0, theta_range=10.0))
    assert not in_window([math.radians(12.0), 0.0, 1.0], dict(phi_mid=355.0, phi_range=30.0, theta_mid=90.0, theta_range=10.0))
    with pytest.raises(ValueError):
        pose_search(fake.step, fake.loss, None, [0.0, 0.0, 1.0], batch_size=4)
    with pytest.raises(ValueError):
        pose_search(fake.step, fake.loss, None, [0.0, 0.0, 1.0], inner_step=0)
    with pytest.raises(ValueError):
        pose_search(fake.step, fake.loss, None, [0.0, 0.0, 1.0], light=np.zeros((4, 2)))
