"""Host tests of oracle/phong_vjp.py, the closed-form float64 vector-Jacobian products of the two Phong composites that the GPU
tests of the Phong kernels compare against at their singular pixels (tests/test_gpu_phong_edges.py)."""
import numpy as np
import pytest
import torch

from oracle import phong_np as pn
from oracle import phong_tf as pt
from oracle.phong_vjp import mask32, np_vjp64, tf_vjp64


def _case(B, H, W, seed):
    rng = np.random.default_rng(seed)
    n = rng.random((B, H, W, 3)).astype(np.float32)
    ld = (1.7 * rng.standard_normal((B, 3))).astype(np.float32)
    col = rng.uniform(0.6, 1.2, (B, 3)).astype(np.float32)
    alb = rng.random((B, H, W, 3)).astype(np.float32)
    g = rng.standard_normal((B, H, W, 3)).astype(np.float32)
    return n, ld, col, alb, g


def _autograd(composite, n, ld, col, ambient, kd, white, mask, g, alb):
    """(shading, dL/dn, dL/dalbedo or None, dL/dl) of oracle/phong_tf.py or oracle/phong_np.py (at mask32's value) by autograd."""
    nt = torch.tensor(n.astype(np.float64), requires_grad=True)
    lt = torch.tensor(ld.astype(np.float64), requires_grad=True)
    at = None if alb is None else torch.tensor(alb.astype(np.float64), requires_grad=True)
    c64 = torch.from_numpy(col).double()
    if composite == "numpy":
        mv = torch.from_numpy(mask32(n, white)) if mask else None
        shade = pn.np_phong_composite(nt, lt, c64, ambient, kd, white, mask, mv)
    else:
        shade = pt.tf_phong_composite(nt, lt, c64, ambient, kd, not white, mask)
    compos = shade if at is None else shade * at
    (compos * torch.from_numpy(g).double()).sum().backward()
    return shade.detach().numpy(), nt.grad.numpy(), None if at is None else at.grad.numpy(), lt.grad.numpy()


def _closed(composite, n, ld, col, ambient, kd, white, mask, g, alb):
    if composite == "numpy":
        return np_vjp64(n, ld, col, ambient, kd, white, mask, g, alb)
    return tf_vjp64(n, ld, col, ambient, kd, not white, mask, g, alb)


@pytest.mark.parametrize("with_albedo", [False, True])
@pytest.mark.parametrize("mask", [False, True])
@pytest.mark.parametrize("white", [False, True])
@pytest.mark.parametrize("composite", ["tf", "numpy"])
def test_closed_form_is_autograd_on_regular_pixels(composite, white, mask, with_albedo):
    """On random pixels (none on a kink or a singular point) tf_vjp64 / np_vjp64 equal float64 autograd of the restatements:
    shading, dL/dn, dL/dalbedo and dL/dl within 1e-12 of their scale."""
    n, ld, col, alb, g = _case(3, 24, 20, 1 + composite.startswith("n") + 2 * white + 4 * mask + 8 * with_albedo)
    # a band of pixels on the mask's transition, where m (1 - m) is far from 0
    rng = np.random.default_rng(5)
    dirs = rng.random((3, 4, 20, 3)) + 0.05
    dirs /= np.linalg.norm(dirs, axis=-1, keepdims=True)
    if composite == "numpy":
        band = 1.0 - dirs * rng.uniform(0.27, 0.36, (3, 4, 20, 1)) if white else dirs * rng.uniform(0.55, 0.63, (3, 4, 20, 1))
    else:
        band = 0.818 + rng.uniform(-0.05, 0.05, (3, 4, 20, 3)) if white else dirs * rng.uniform(0.27, 0.36, (3, 4, 20, 1))
    n[:, :4] = np.clip(band, 0.0, 1.0)
    alb = alb if with_albedo else None
    for ambient, kd in ((0.0, 1.0), (0.1, 0.9)):
        want = _autograd(composite, n, ld, col, ambient, kd, white, mask, g, alb)
        got = _closed(composite, n, ld, col, ambient, kd, white, mask, g, alb)
        for name, a, b in zip(("shade", "d_normal", "d_albedo", "d_light"), got, want):
            if b is None:
                assert a is None, name
                continue
            e = float(np.abs(a - b).max() / np.abs(b).max())
            assert e <= 1e-12, (name, ambient, kd, e)


@pytest.mark.parametrize("composite", ["tf", "numpy"])
def test_closed_form_is_finite_where_autograd_is_not(composite):
    """At n = (0.5, 0.5, 0.5) and where the mask's |a| is 0 (n = 0 for TF and the NumPy black background, n = 1 for the NumPy
    white one) autograd of the restatements is NaN, which is why the closed form exists: there it is finite, n = 0.5 is shaded
    as unlit and adds nothing to dL/dl, and the mask term is 0 where |a| = 0."""
    n, ld, col, alb, g = _case(2, 8, 8, 31)
    n[:, 0, 0] = 0.5
    n[:, 0, 1] = 0.0
    n[:, 0, 2] = 1.0
    for white in (False, True):
        for mask in (False, True):
            ag = _autograd(composite, n, ld, col, 0.1, 0.9, white, mask, g, alb)
            shade, dn, da, dl = _closed(composite, n, ld, col, 0.1, 0.9, white, mask, g, alb)
            assert all(np.isfinite(x).all() for x in (shade, dn, da, dl)), (white, mask)
            assert np.isnan(ag[1][:, 0, 0]).all() and np.isnan(ag[3]).all(), (white, mask)
            if mask:
                zero_a = 2 if composite == "numpy" and white else 1       # the pixel where the mask's |a| is 0
                assert np.isnan(ag[1][:, 0, zero_a]).all(), (white, mask)
            # n = 0.5: unlit (the diffuse term is 0), and dL/dl is that of the image without the pixel
            unlit = _closed(composite, n, ld, col, 0.1, 0.0, white, mask, g, alb)[0]          # k_d = 0
            assert np.array_equal(shade[:, 0, 0], unlit[:, 0, 0])
            g0 = g.copy()
            g0[:, 0, 0] = 0.0
            assert np.array_equal(dl, _closed(composite, n, ld, col, 0.1, 0.9, white, mask, g0, alb)[3])
