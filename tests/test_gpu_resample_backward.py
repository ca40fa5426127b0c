"""GPU tests of the resampler backward (rn_resample_backward_f32) at production size, 64^3 -> 128^3, against autograd through a
float64 resampler that samples in the device's cells (oracle/resample_cells.py).

dL/dMinv, and the pose gradient dL/d(azimuth, elevation, scale) built from it, are one-sided derivatives: of the trilinear patch
the fp32 sample coordinate falls in.  A reference with float64 coordinates differentiates other patches wherever a coordinate
lies within an ulp of an integer, which at the axis-aligned poses of every turntable moves dL/dpose by 1.6x its largest
component (see test_bars_discriminate); with the device's cells the only differences left are the kernel's fp32 arithmetic and reduction order.

Bars, per batch item: dvox max error / max |reference|; dMinv max entry error / the item's largest entry; dpose (through
pose_matrix_jacobian_vjp) max component error / the largest component.  Measured on one H100 80GB HBM3 (400 W power limit) over
the 19 batch items below, three runs: dvox <= 4.0e-7, dMinv <= 1.6e-6, dpose <= 9.0e-6; the bars are about 3x that.  The
kernel sums dMinv in fp32 (per lane, warp tree, block, then one atomic per block: 2048 per item), so the error changes from run to
run with the order of the atomics (suite pose: dpose 1.8e-6, 5.1e-7, 1.5e-6), and dpose cancels part of dMinv -- the grid
coordinates are centred on the rotation centre -- so it carries 2-10x dMinv's relative error.  In the whole network this part is
small: tests/test_gpu_backward.py measures the resampler's share of the dL/dpose error at 3e-6 to 9e-6 and the network's at 9e-5.
"""
import os

import numpy as np
import pytest
import torch

from oracle import rendernet_oracle as orc
from oracle import resample_cells as rc

pytestmark = pytest.mark.gpu
dev = "cuda"

BAR_DVOX, BAR_DMINV, BAR_DPOSE = 1.2e-6, 5e-6, 2.7e-5

POSES = {"suite": (250.0, 60.0, 3.3), "az0": (0.0, 60.0, 3.3), "az90": (90.0, 60.0, 3.3), "az180": (180.0, 60.0, 3.3),
         "az270": (270.0, 60.0, 3.3), "top": (180.0, 90.0, 3.3), "clipped": (300.0, 20.0, 1.8), "generic": (45.0, 30.0, 2.5)}


def _poses(*names):
    return np.concatenate([orc.compute_pose_param(*POSES[n]) for n in names]).astype(np.float32)


def _minv(poses):
    R, S = orc.rotation_around_grid_centroid(poses)
    return orc.inverse_total_matrix(R, S, 64, 128)


def _chair(B=1):
    """The chair fixture with continuous occupancies (what inverse rendering feeds), B copies with different speckle."""
    bv = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "binvox.npz"))
    vox = np.unpackbits(bv["chair_bits"]).reshape(1, 64, 64, 64, 1).astype(np.float32)
    rng = np.random.default_rng(2)
    return (vox * 0.75 + 0.125 * (rng.random((B, 64, 64, 64, 1)) < 0.02)).astype(np.float32)


def _field(kind, shape, seed):
    """dL/dgrid: white noise, 95 % zeros (the kernel's gv == 0 skip), or values spread over 2^-20 .. 2^20."""
    rng = np.random.default_rng(seed)
    g = rng.standard_normal(shape)
    if kind == "sparse":
        g *= rng.random(shape) < 0.05
    elif kind == "binades":
        g *= np.exp2(rng.integers(-20, 21, shape))
    return g.astype(np.float32)


def _reference(vox, minv, G, transform=True, device_cells=True):
    """(dvox, dminv) float64 by autograd through oracle/resample_cells.py."""
    vt = torch.tensor(vox.astype(np.float64), requires_grad=True)
    mt = torch.tensor(minv.astype(np.float64), requires_grad=True)
    out = rc.resample(vt, mt, G.shape[1], transform, device_cells)
    (out * torch.from_numpy(G.astype(np.float64))).sum().backward()
    return vt.grad.numpy(), mt.grad.numpy()


def _kernel(vox, minv, G, transform=True, want_dvox=True, want_dminv=True):
    from rendernet_b200 import ops
    dvox, dminv = ops.resample_backward(torch.from_numpy(vox).to(dev), torch.from_numpy(minv).to(dev), torch.from_numpy(G).to(dev),
                                        transform, want_dvox, want_dminv)
    return (dvox.cpu().numpy() if dvox is not None else None), (dminv.cpu().numpy() if dminv is not None else None)


def _rel(got, want):
    return float(np.abs(np.asarray(got, np.float64) - want).max() / max(np.abs(want).max(), 1e-300))


def _errors(poses, got, ref):
    """[(dvox, dMinv, dpose) relative errors] per batch item."""
    from rendernet_b200.backward import pose_matrix_jacobian_vjp
    dp_got = pose_matrix_jacobian_vjp(poses, got[1])
    dp_ref = pose_matrix_jacobian_vjp(poses, ref[1])
    return [(_rel(got[0][b], ref[0][b]) if got[0] is not None else 0.0, _rel(got[1][b], ref[1][b]), _rel(dp_got[b], dp_ref[b]))
            for b in range(len(poses))]


def _check(label, poses, got, ref):
    errs = _errors(poses, got, ref)
    for b, (e_v, e_m, e_p) in enumerate(errs):
        print(f"{label} item {b}: dvox {e_v:.2e}, dMinv {e_m:.2e}, dpose {e_p:.2e}")
    for e_v, e_m, e_p in errs:
        assert e_v < BAR_DVOX and e_m < BAR_DMINV and e_p < BAR_DPOSE, (label, errs)
    return errs


# ----------------------------------------------------------------------------------------- poses and gradient fields
@pytest.mark.parametrize("pose", list(POSES))
def test_resample_backward_pose(pose):
    """B = 1, white-noise dL/dgrid, at the suite's pose, the four turntable frames, a top view, a radius small enough that the
    grid border clips the rotated cube, and a generic pose."""
    poses = _poses(pose)
    minv, vox = _minv(poses), _chair()
    G = _field("white", (1, 128, 128, 128, 1), 10)
    if pose == "clipped":            # the rotated cube reaches past the grid border: some border planes sample it
        c = rc.sample_coords(minv, rc.output_grid(128)).reshape(3, 128, 128, 128)
        inside = ((c >= 0) & (c < 63)).all(0)
        assert inside[0].any() and inside[-1].any() and inside[:, :, 0].any() and inside[:, :, -1].any()
    _check(pose, poses, _kernel(vox, minv, G), _reference(vox, minv, G))


@pytest.mark.parametrize("kind", ["sparse", "binades"])
def test_resample_backward_gradient_fields(kind):
    """95 % zeros and values spanning 40 binades, at the turntable's az = 0 frame and at the suite's pose (B = 2)."""
    poses = _poses("az0", "suite")
    minv, vox = _minv(poses), _chair(2)
    G = _field(kind, (2, 128, 128, 128, 1), 11)
    _check(kind, poses, _kernel(vox, minv, G), _reference(vox, minv, G))


def test_resample_backward_batch_of_three():
    """B = 3, a different pose and gradient field per item: each block's dMinv partial must land on its own item."""
    poses = _poses("az0", "suite", "clipped")
    minv, vox = _minv(poses), _chair(3)
    G = np.concatenate([_field(k, (1, 128, 128, 128, 1), 12 + i) for i, k in enumerate(("white", "sparse", "binades"))])
    _check("B=3", poses, _kernel(vox, minv, G), _reference(vox, minv, G))


@pytest.mark.parametrize("pose", ["suite", "az0"])
def test_resample_backward_real_gradient_field(pose):
    """The dL/dgrid the Shader network's backward pass actually produces (ShaderInputGradients.last_dgrid, exact mode, full size)."""
    from rendernet_b200.backward import ShaderInputGradients
    poses = _poses(pose)
    vox = _chair()
    W = orc.init_shader_weights(seed=1, alpha_range=(0.05, 0.3), bias_jitter=0.02)
    ig = ShaderInputGradients(W, 1, precision="exact")
    ig.forward(vox, poses)
    ig.backward(np.random.default_rng(5).standard_normal((1, 512, 512, 3)).astype(np.float32))
    G = ig.last_dgrid.cpu().numpy()
    minv = ig.minv.cpu().numpy()
    assert np.array_equal(minv, _minv(poses))
    _check(f"real dL/dgrid at {pose}", poses, _kernel(vox, minv, G), _reference(vox, minv, G))


def test_resample_backward_four_channels_untransformed():
    """C = 4 (the Texture net's volume) and transform = 0 (the resampler without the axis transform)."""
    poses = _poses("az180", "generic")
    minv = _minv(poses)
    vox = np.random.default_rng(13).random((2, 64, 64, 64, 4)).astype(np.float32)
    G = _field("white", (2, 128, 128, 128, 4), 14)
    _check("C=4 transform=0", poses, _kernel(vox, minv, G, transform=False), _reference(vox, minv, G, transform=False))


def test_resample_backward_partial_outputs_equal_combined():
    """want_dvox / want_dminv alone give what the combined call gives, up to the order of the fp32 atomics (measured 1.2e-7 for
    dvox and 5.6e-7 to 7.0e-7 for dMinv)."""
    poses = _poses("suite", "az90")
    minv, vox = _minv(poses), _chair(2)
    G = _field("white", (2, 128, 128, 128, 1), 15)
    dvox, dminv = _kernel(vox, minv, G)
    dvox_only, none_m = _kernel(vox, minv, G, want_dminv=False)
    none_v, dminv_only = _kernel(vox, minv, G, want_dvox=False)
    assert none_m is None and none_v is None
    e_v, e_m = _rel(dvox_only, dvox), _rel(dminv_only, dminv)
    print(f"dvox-only vs combined {e_v:.2e}, dMinv-only vs combined {e_m:.2e}")
    assert e_v < BAR_DVOX / 2 and e_m < BAR_DMINV / 2


def test_resample_backward_rejects_unsupported_shapes():
    from rendernet_b200 import ops
    z = lambda *s: torch.zeros(s, device=dev)                                                         # noqa: E731
    with pytest.raises(RuntimeError, match="rc=-2"):                      # 6 * 6 rows: a block's 8 rows would span two items
        ops.resample_backward(z(2, 8, 8, 8, 1), z(2, 3, 4), z(2, 6, 6, 6, 1), True)
    for C in (2, 3):
        with pytest.raises(RuntimeError, match="rc=-3"):
            ops.resample_backward(z(1, 8, 8, 8, C), z(1, 3, 4), z(1, 8, 8, 8, C), True)
    with pytest.raises(RuntimeError, match="rc=-1"):
        ops.resample_backward(z(1, 8, 8, 8, 1), z(1, 3, 4), z(1, 8, 8, 8, 1), True, want_dvox=False, want_dminv=False)


# ----------------------------------------------------------------------------------------- the bars can tell
def test_bars_discriminate():
    """The bars catch what a reference with float64 coordinates (device_cells=False) gets wrong at the turntable's az = 0 frame
    and at the suite's pose, and one 128-point row of dL/dgrid left out of the reference.  Measured: float64 coordinates move
    199k points (az = 0) and 2.3k points (suite) to another cell or across the border, and put dpose off by 1.6 and 5.3e-2; the
    missing row puts dMinv off by 3.1e-2."""
    poses = _poses("az0", "suite")
    minv, vox = _minv(poses), _chair(2)
    G = _field("white", (2, 128, 128, 128, 1), 16)
    got = _kernel(vox, minv, G)
    g = rc.output_grid(128)
    c32 = rc.sample_coords(minv, g)
    c64 = np.matmul(minv.astype(np.float64), g)
    in32, in64 = ((c32 >= 0) & (c32 < 63)).all(1), ((c64 >= 0) & (c64 < 63)).all(1)
    moved = (in32 != in64) | (in32 & (np.floor(c32) != np.floor(c64)).any(1))
    errs = _errors(poses, got, _reference(vox, minv, G, device_cells=False))
    for b, (e_v, e_m, e_p) in enumerate(errs):
        print(f"float64-coordinate reference, {('az0', 'suite')[b]}: {int(moved[b].sum())} points in another cell or "
              f"inside/outside; dvox {e_v:.2e}, dMinv {e_m:.2e}, dpose {e_p:.2e}")
        assert e_p > BAR_DPOSE
    G_row = G.copy()
    G_row[1, 64, 64] = 0.0                                                # the row through the grid centre
    (e_v, e_m, e_p), = _errors(poses[1:], (got[0][1:], got[1][1:]), _reference(vox[1:], minv[1:], G_row[1:]))
    print(f"reference without one dL/dgrid row: dvox {e_v:.2e}, dMinv {e_m:.2e}, dpose {e_p:.2e}")
    assert e_m > BAR_DMINV
