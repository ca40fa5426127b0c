"""CPU tests of the shape fit (rendernet_b200/shape_fit.py) and what it writes and reads: argument checks before anything reaches
a device, the dataset's pose naming (data_util.extract_param_from_names), the binvox writer byte for byte against the reference's
own writer (tests/golden/binvox_write.npz, made by tests/golden/make_binvox_write_golden.py), and the carving rule on a hand-built
case with a fake resampler backward."""
import io
import math
import os

import numpy as np
import pytest
import torch

from rendernet_b200 import binvox_rw

SHAPES = ("bunny", "chair", "suzanne", "table", "teapot")


# ----------------------------------------------------------------------------------------- argument checks
def _vfg_args(**kw):
    a = dict(dvox=torch.zeros(3, 8, 8, 8), occ=torch.zeros(8, 8, 8), keep=None, lambda_smooth=0.1, lambda_bin=0.1)
    a.update(kw)
    return a


@pytest.mark.parametrize("bad", [
    dict(dvox=torch.zeros(3, 8, 8, 8, dtype=torch.float64)),              # dtype
    dict(occ=torch.zeros(8, 8, 8, dtype=torch.float16)),
    dict(occ=torch.zeros(8, 8, 7)),                                     # not a cube
    dict(dvox=torch.zeros(3, 8, 8, 4)),                                 # views of the wrong size
    dict(dvox=torch.zeros(0, 8, 8, 8)),                                 # no view
    dict(keep=torch.ones(8, 8, 8, dtype=torch.bool)),                   # keep not uint8
    dict(keep=torch.ones(8, 8, 4, dtype=torch.uint8)),
    dict(lambda_smooth=-1e-3), dict(lambda_bin=-1.0), dict(lambda_smooth=float("nan")), dict(lambda_bin=float("inf")),
    dict(dvox=np.zeros((3, 8, 8, 8), np.float32)),                      # not a tensor
    dict(),                                                             # well formed, but on the host
])
def test_voxel_fit_grad_rejects_malformed_input(bad):
    from rendernet_b200 import ops
    with pytest.raises(ValueError):
        ops.voxel_fit_grad(**_vfg_args(**bad))


def _poses(V):
    return np.stack([np.linspace(0.0, 2.0, V), np.full(V, 0.3), np.ones(V)], 1).astype(np.float32)


@pytest.mark.parametrize("kw,match", [
    (dict(poses=_poses(4), light=np.zeros((3, 2))), "light"),           # V mismatch: poses 4, lights 3
    (dict(poses=_poses(4)), "light"),                                   # phong needs the light
    (dict(poses=_poses(4), objective="mse", light=[0.1, 0.2]), "no light"),
    (dict(poses=_poses(4), objective="bce", light=np.zeros((4, 2))), "no light"),
    (dict(poses=_poses(4), is_greyscale=True, light=[0.1, 0.2]), "greyscale"),
    (dict(poses=_poses(4), light=[0.1, 0.2], lambda_smooth=-0.1), "lambda_smooth"),
    (dict(poses=_poses(4), light=[0.1, 0.2], lambda_bin=float("nan")), "lambda_bin"),
    (dict(poses=_poses(4), light=[0.1, 0.2], lr=0.0), "lr"),
    (dict(poses=_poses(4), light=[0.1, 0.2], betas=(1.0, 0.999)), "betas"),
    (dict(poses=np.zeros((4, 2)), light=[0.1, 0.2]), "poses"),
    (dict(poses=_poses(4), objective="l1"), "objective"),
])
def test_shape_fit_rejects_bad_arguments(kw, match):
    from rendernet_b200.shape_fit import ShaderShapeFit
    with pytest.raises(ValueError, match=match):
        ShaderShapeFit(None, **kw)


def _bare_fit(V, grey=False):
    """A ShaderShapeFit without its network (the view-count checks below run before anything reaches a device)."""
    from rendernet_b200.shape_fit import ShaderShapeFit
    fit = ShaderShapeFit.__new__(ShaderShapeFit)
    fit.V, fit.B, fit.is_greyscale, fit.device, fit._target, fit.poses = V, V, grey, "cpu", None, _poses(V)
    return fit


def test_view_count_mismatches_raise():
    from rendernet_b200.shape_fit import carve
    fit = _bare_fit(4)
    with pytest.raises(ValueError, match="target"):
        fit._targets(np.zeros((3, 512, 512, 3), np.float32))            # targets 3, poses 4
    with pytest.raises(ValueError, match="target"):
        _bare_fit(4, grey=True)._targets(np.zeros((4, 512, 512, 3), np.float32))
    with pytest.raises(ValueError, match="masks"):
        fit.run(np.zeros((4, 512, 512, 3), np.float32), masks=np.zeros((5, 512, 512), bool))
    with pytest.raises(ValueError, match="masks"):
        carve(_poses(3), np.zeros((2, 512, 512), bool), device="cpu")
    with pytest.raises(ValueError, match="masks"):
        carve(_poses(2), np.zeros((2, 256, 256), bool), device="cpu")


# ----------------------------------------------------------------------------------------- dataset names
def test_extract_param_from_names_on_the_reference_names():
    """The reference's own file names (`ply80024_p294_t105_r3.3`): azimuth 294 deg, elevation 90 - 105 = -15 deg, scale
    3.3 / 3.3, in radians; the radius is the three characters after "_r"."""
    from rendernet_b200.data_util import extract_param_from_names
    p = extract_param_from_names("ply80024_p294_t105_r3.3.png")
    assert p.shape == (1, 3)
    assert p[0, 0] == 294 * math.pi / 180.0 and p[0, 1] == -15 * math.pi / 180.0 and p[0, 2] == 1.0
    assert np.allclose(p[0, :2], np.radians([294.0, -15.0]), rtol=0, atol=1e-15)
    p = extract_param_from_names("chair_p30_t60_r6.6_view2.png")
    assert np.allclose(p[0], [math.radians(30.0), math.radians(30.0), 0.5], rtol=1e-15)
    assert extract_param_from_names("x_p0_t90_r3.3000")[0, 2] == 1.0      # "3.3000" -> "3.3"
    assert extract_param_from_names("x_p0_t90_r3.31")[0, 2] == 3.3 / 3.3   # the slice drops the last digit
    with pytest.raises(ValueError):
        extract_param_from_names("no_pose_here.png")


# ----------------------------------------------------------------------------------------- binvox writer
def _golden_cases(golden_dir):
    g = np.load(os.path.join(golden_dir, "binvox_write.npz"))
    bv = np.load(os.path.join(golden_dir, "binvox.npz"))
    grids = {nm: np.unpackbits(bv[nm + "_bits"]).reshape(64, 64, 64).astype(bool) for nm in SHAPES}
    for nm in ("soft", "runs"):
        grids[nm] = np.unpackbits(g[nm + "_bits"]).reshape(64, 64, 64).astype(bool)
    return g, grids


def test_binvox_writer_matches_the_reference_bytes(golden_dir, tmp_path):
    """save_binvox, Voxels.write (non-default header) and write in x-z-y order reproduce the reference writer's bytes for the
    five fixture shapes, a thresholded soft grid and a grid with runs of exactly 255 / 510 (the (value, 0) pairs)."""
    g, grids = _golden_cases(golden_dir)
    for nm, data in grids.items():
        binvox_rw.save_binvox(data, str(tmp_path / f"{nm}.binvox"))
        assert (tmp_path / f"{nm}.binvox").read_bytes() == g[nm + "_save"].tobytes(), nm
        buf = io.BytesIO()
        binvox_rw.Voxels(data, [64, 64, 64], [0.5, -1.25, 3.0], 2.5, "xyz").write(buf)
        assert buf.getvalue() == g[nm + "_write"].tobytes(), nm
        buf = io.BytesIO()
        binvox_rw.write(binvox_rw.Voxels(np.ascontiguousarray(data.transpose(0, 2, 1)), [64, 64, 64], [0.0, 0.0, 0.0], 1.0,
                                         "xzy"), buf)
        assert buf.getvalue() == g[nm + "_write_xzy"].tobytes(), nm


def test_binvox_round_trip_and_the_zero_length_run(golden_dir, tmp_path):
    """read_as_3d_array of what the writer wrote returns the input, header included.  The "runs" grid's payload holds the
    reference writer's (value, 0) pairs after runs of exactly 255 and 510, and no trailing pair after its last run of 255."""
    _, grids = _golden_cases(golden_dir)
    for nm, data in grids.items():
        path = tmp_path / f"{nm}.binvox"
        binvox_rw.save_binvox(data, str(path))
        with open(path, "rb") as f:
            v = binvox_rw.read_as_3d_array(f)
        assert np.array_equal(v.data, data) and v.dims == [64, 64, 64] and v.translate == [0.0, 0.0, 0.0] and v.scale == 1.0, nm
        with open(path, "rb") as f:
            pairs = binvox_rw.read_rle(f)[3]
        if nm == "runs":
            got = [tuple(int(x) for x in p) for p in pairs]
            assert got[:6] == [(0, 255), (0, 0), (1, 255), (1, 255), (1, 0), (0, 7)], got[:6]
            assert got[-1] == (1, 255) and sum(c == 0 for _, c in got) == 3
    binvox_rw.save_binvox(np.zeros((4, 4, 4), bool), str(tmp_path / "z.binvox"))   # 64 zeros: one run, no zero pair
    assert (tmp_path / "z.binvox").read_bytes().endswith(b"data\n\x00\x40")
    with pytest.raises(ValueError):
        binvox_rw.write(binvox_rw.Voxels(np.zeros((4, 4, 4), bool), [4, 4, 4], [0, 0, 0], 1.0, "zyx"), io.BytesIO())


# ----------------------------------------------------------------------------------------- carving
def test_mask_columns_downsample_and_dilate():
    from rendernet_b200.shape_fit import mask_columns
    m = np.zeros((2, 512, 512), bool)
    m[0, 4 * 10 + 3, 4 * 20] = True                                    # one pixel -> column (10, 20)
    m[1, 0, 511] = True                                                 # corner column (0, 127)
    c0 = mask_columns(m, margin=0)
    assert c0.shape == (2, 128, 128) and c0.sum() == 2 and c0[0, 10, 20] and c0[1, 0, 127]
    c1 = mask_columns(m, margin=1)
    assert c1[0].sum() == 9 and c1[0, 9:12, 19:22].all()
    assert c1[1].sum() == 4 and c1[1, 0:2, 126:128].all()
    assert mask_columns(m, margin=2)[0].sum() == 25


def test_carving_rule_on_a_hand_built_case():
    """8^3 grid, two views, a fake resampler backward in which voxel i sits on column (i // 128, i % 128) of the 128^2 grid in
    both views, observed there by the views its class says.  Classes (i % 5): 0 observed by both and inside both -> kept;
    1 inside view 0, outside view 1 -> carved; 2 observed by view 0 only, inside it -> kept; 3 observed by view 1 only, outside
    it -> carved; 4 unobserved by every view -> carved."""
    from rendernet_b200.shape_fit import carve, carve_rule
    S, V = 8, 2
    n = S ** 3
    cls = np.arange(n) % 5
    seen = np.array([[c in (0, 1, 2) for c in cls], [c in (0, 1, 3) for c in cls]])
    inside = np.array([[c in (0, 1, 2) for c in cls], [c == 0 for c in cls]])
    masks = np.zeros((V, 512, 512), bool)
    for v in range(V):
        for i in np.flatnonzero(inside[v]):
            p, q = divmod(int(i), 128)
            masks[v, 4 * p + 1, 4 * q + 2] = True                       # one pixel of the column's 4 x 4
    calls = []

    def fake_backward(minv, gout):
        assert tuple(minv.shape) == (V, 3, 4) and tuple(gout.shape) == (V, 128, 128, 128, 1)
        calls.append(gout)
        col = gout[..., 0].sum(-1).reshape(V, -1)[:, :n]                # depth sum of voxel i's column
        return (col * torch.from_numpy(seen)).reshape(V, S, S, S, 1)

    keep = carve(_poses(V), masks, margin=0, size=S, device="cpu", resample_backward=fake_backward)
    want = np.isin(cls, (0, 2)).reshape(S, S, S).astype(np.uint8)
    assert keep.dtype == np.uint8 and np.array_equal(keep, want)
    assert len(calls) == 2 and bool((calls[0] == 1).all())              # observed: the ones grid; inside: the broadcast mask
    assert bool((calls[1] == calls[1][:, :, :, :1]).all())              # constant along depth
    o = np.array([[1.0, 0.0, 2e-30], [0.5, 0.0, 0.0]])
    i = np.array([[1.0, 0.0, 0.0], [0.0, 0.0, 0.0]])
    assert carve_rule(o, i).tolist() == [0, 0, 0]                      # outside view 1; unobserved; outside view 0
    assert carve_rule(o, np.array([[1.0, 0, 1e-30], [3.0, 0, 0]])).tolist() == [1, 0, 1]
