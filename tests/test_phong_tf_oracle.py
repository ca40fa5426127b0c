"""CPU tests of oracle/phong_tf.py, the torch restatement of the reference's TensorFlow Phong composite that the GPU tests of
rn_phong_recon_loss_grad and reconstruction_gradients differentiate: its forward is held to tests/golden/phong_tf.npz, frozen by
running the reference's own tools/Phong_shading.py over the NumPy shim of TF-1, and its kinks follow TF-1's gradient rules."""
import os

import numpy as np
import torch

from oracle import phong_tf as pt


def _fx(golden_dir):
    return np.load(os.path.join(golden_dir, "phong_tf.npz"))


def test_restatement_matches_reference_forward(golden_dir):
    d = _fx(golden_dir)
    nm, light, col = (torch.from_numpy(d[k]).double() for k in ("normal_map", "light", "light_col"))
    for name, black, mask in (("white_mask", False, True), ("black_mask", True, True), ("no_mask", False, False)):
        got = pt.tf_phong_composite(nm, light, col, float(d["ambient"]), float(d["k_diffuse"]), black, mask).numpy()
        assert np.abs(got - d[name]).max() < 2e-6, name                  # fp32 reference vs float64: measured <= 5.5e-7
    got = pt.tf_phong_composite(nm, light, torch.ones(2, 3, dtype=torch.float64), 0.0, 1.0, with_mask=False).numpy()
    assert np.abs(got - d["exact_light_k1"]).max() < 2e-6
    assert d["exact_light_k1"][0, 5, :4].min() == 1.0                     # the clip boundary is hit exactly
    lp = pt.tf_generate_light_pos(torch.from_numpy(d["light_azimuth"]).double(), float(d["light_elevation"])).numpy()
    assert np.abs(lp - d["light_pos"]).max() < 1e-6


def test_gradient_conventions_at_the_kinks():
    """tf.maximum(d, 0) passes at d = 0; clip_by_value passes at its bounds; both as TF-1 registers them."""
    n = torch.tensor([[[[0.75, 0.5, 0.5], [0.5, 0.5, 0.75]]]], dtype=torch.float64, requires_grad=True)   # u.L = 0 and 1
    L = torch.tensor([[0.0, 0.0, 2.0]], dtype=torch.float64, requires_grad=True)
    shade = pt.tf_phong_composite(n, L, torch.ones(1, 3, dtype=torch.float64), 0.0, 1.0, with_mask=False)
    assert shade[0, 0, 0, 0].item() == 0.0 and shade[0, 0, 1, 0].item() == 1.0
    shade.sum().backward()
    assert n.grad[0, 0, 0].abs().sum() > 0          # d = 0 exactly: the maximum passes the gradient
    assert n.grad[0, 0, 1].abs().sum() == 0         # d = 1: u is parallel to L, du is orthogonal to u -> 0 by geometry
    assert L.grad.abs().sum() > 0
    x = torch.tensor([0.0, 1.0, 1.5], dtype=torch.float64, requires_grad=True)
    torch.clamp(x, 0.0, 1.0).sum().backward()
    assert x.grad.tolist() == [1.0, 1.0, 0.0]
