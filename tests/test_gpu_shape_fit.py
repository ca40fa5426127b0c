"""GPU tests of the shape fit through the Shader network (rendernet_b200/shape_fit.py): rn_voxel_fit_grad against float64 NumPy, the
whole objective against the frozen-kink oracle, silhouette carving against a NumPy restatement on the device's sample
coordinates, the fixed point, chunking, the device paths of ShaderInputGradients, a short run and the command line.

References are float64: the network through the oracle Shader with the device's PReLU kinks frozen (oracle/frozen_kinks.py) and
the device-cell resampler (oracle/resample_cells.py).  Errors are max |error| / max |reference| unless stated otherwise."""
import json
import math
import os

import numpy as np
import pytest
import torch

from oracle import phong_np as pn
from oracle import rendernet_oracle as orc
from oracle import resample_cells as rc

pytestmark = pytest.mark.gpu
dev = "cuda"
D64 = torch.float64
SHAPES = ("bunny", "chair", "suzanne", "table", "teapot")
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def _d(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _rel(got, want):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert got.shape == want.shape, (got.shape, want.shape)
    return float(np.abs(got - want).max() / max(np.abs(want).max(), 1e-30))


def _shape(name):
    bv = np.load(os.path.join(GOLDEN, "binvox.npz"))
    return np.unpackbits(bv[name + "_bits"]).reshape(64, 64, 64).astype(np.float32)


def _soft_chair():
    vox = _shape("chair")
    return (vox * 0.75 + 0.125 * (np.random.default_rng(2).random(vox.shape) < 0.02)).astype(np.float32)


def _turntable(V, elevation=60.0):
    from rendernet_b200.RenderNet_demo import compute_pose_param
    return np.concatenate([compute_pose_param(360.0 * k / V, elevation, 3.3) for k in range(V)]).astype(np.float32)


def _lights(V):
    return np.stack([np.linspace(240, 310, V) * math.pi / 180, np.full(V, math.radians(60.0))], 1)


def _shape_masks(vox, poses):
    """Silhouettes of a shape from its own resampled grid: a 128^2 column is inside if any cell along depth is occupied (> 0),
    upsampled x4 to the image."""
    from rendernet_b200 import ops
    from rendernet_b200.engine import pose_to_matrix
    V = len(poses)
    v = _d(np.repeat(np.asarray(vox, np.float32).reshape(1, 64, 64, 64, 1), V, 0))
    grid = ops.resample(v, _d(pose_to_matrix(poses, 64, 128)), 128, True)
    cols = (grid[..., 0] > 0).any(-1).cpu().numpy()
    return np.repeat(np.repeat(cols, 4, 1), 4, 2)


# ----------------------------------------------------------------------------------------- the kernel
def _fit_grad_ref(dvox, occ, keep, ls, lb):
    o = occ.astype(np.float64)
    n = o.size
    gs = np.zeros_like(o)
    rs = 0.0
    for ax in range(3):
        d = np.diff(o, axis=ax)                                          # o[i+1] - o[i]
        rs += (d ** 2).sum()
        lo = [slice(None)] * 3
        hi = [slice(None)] * 3
        lo[ax], hi[ax] = slice(None, -1), slice(1, None)
        gs[tuple(lo)] -= 2 * d
        gs[tuple(hi)] += 2 * d
    rb = (o * (1 - o)).sum()
    g = dvox.astype(np.float64).sum(0) + (ls * gs + lb * (1 - 2 * o)) / n
    if keep is not None:
        g = g * keep
    return g, np.array([rs / n, rb / n])


@pytest.mark.parametrize("S", [64, 7])
def test_voxel_fit_grad_matches_float64(S):
    """rn_voxel_fit_grad for V = 1..24, with and without keep, lambda = 0 and nonzero, on grids holding exact 0s and 1s
    (border voxels included: every face of the grid is checked by the whole-grid comparison).  Bars: g 1e-6 of its scale,
    R_s and R_b 1e-6 relative.  Two launches are bit-identical."""
    from rendernet_b200 import ops
    rng = np.random.default_rng(S)
    worst = dict(g=0.0, rs=0.0, rb=0.0)
    for V in (1, 2, 3, 8, 13, 24):
        occ = rng.random((S, S, S)).astype(np.float32)
        occ[rng.random(occ.shape) < 0.2] = 0.0
        occ[rng.random(occ.shape) < 0.2] = 1.0
        dvox = (1e-5 * rng.standard_normal((V, S, S, S))).astype(np.float32)
        keep = (rng.random(occ.shape) < 0.7).astype(np.uint8)
        for k in (None, keep):
            for ls, lb in ((0.0, 0.0), (0.5, 0.3), (2.0, 0.0)):
                g, reg = ops.voxel_fit_grad(_d(dvox), _d(occ), None if k is None else _d(k), ls, lb)
                gw, rw = _fit_grad_ref(dvox, occ, k, ls, lb)
                worst["g"] = max(worst["g"], _rel(g.cpu().numpy(), gw))
                r = reg.cpu().numpy()
                worst["rs"] = max(worst["rs"], abs(r[0] - rw[0]) / rw[0])
                worst["rb"] = max(worst["rb"], abs(r[1] - rw[1]) / rw[1])
                if k is not None:
                    assert (g.cpu().numpy()[k == 0] == 0).all()
                g2, reg2 = ops.voxel_fit_grad(_d(dvox), _d(occ), None if k is None else _d(k), ls, lb)
                assert torch.equal(g, g2) and torch.equal(reg, reg2)
    print(f"S={S}: worst g {worst['g']:.2e}, R_s {worst['rs']:.2e}, R_b {worst['rb']:.2e}")
    assert worst["g"] <= 1e-6 and worst["rs"] <= 1e-6 and worst["rb"] <= 1e-6


# ----------------------------------------------------------------------------------------- the whole objective
@pytest.mark.parametrize("network", ["rgb", "grey"])
@pytest.mark.parametrize("precision", ["exact", "fast"])
def test_full_size_objective_matches_frozen_kink_oracle(precision, network):
    """ShaderShapeFit.gradients at V = 4 turntable views of the soft chair, random targets, lambda_smooth = 0.3, lambda_bin = 0.2
    and the chair's carve mask: "phong" and "mse" on the RGB network, "bce" on the greyscale one.  Reference: float64 autograd of
    sum_v loss_v + lambda_s R_s + lambda_b R_b, the data term pushed through the oracle Shader with the device's kinks frozen and
    the device-cell resampler, dL/dvox masked by the hull.  Bars: g exact 3e-4 / fast 6e-3 of scale (the chain tests' bars);
    loss, R_s, R_b 1e-6 relative."""
    from rendernet_b200 import tfcompat as tf
    from rendernet_b200.shape_fit import ShaderShapeFit, carve
    from oracle.frozen_kinks import prelu_kinks, tape_prelu_masks
    V, ls, lb = 4, 0.3, 0.2
    grey = network == "grey"
    W = orc.init_shader_weights(seed=1, is_greyscale=grey, alpha_range=(0.05, 0.3), bias_jitter=0.02)
    occ, poses, lights = _soft_chair(), _turntable(V), _lights(V)
    keep = carve(poses, _shape_masks(occ > 0.5, poses))
    rng = np.random.default_rng(8)
    C = 1 if grey else 3
    for obj in (("bce",) if grey else ("phong", "mse")):
        tgt = (rng.random((V, 512, 512, C)) < 0.3).astype(np.float32) if obj == "bce" else rng.random((V, 512, 512, C)).astype(np.float32)
        fit = ShaderShapeFit(W, poses, objective=obj, batch=V, precision=precision, is_greyscale=grey,
                             light=lights if obj == "phong" else None, lambda_smooth=ls, lambda_bin=lb)
        fit.keep = keep
        loss, reg, g = fit.gradients(occ, tgt)
        img = fit.ig.img.cpu().numpy()
        with tf.use_store(fit.ig.store):
            masks = tape_prelu_masks(fit.ig.tape)
        x = torch.tensor(img.astype(np.float64), requires_grad=True)
        t64 = torch.from_numpy(tgt).double()
        del fit
        torch.cuda.empty_cache()
        if obj == "phong":
            ref = pn.fit_loss(x, t64, pn.generate_light_pos(torch.from_numpy(lights)), torch.ones(V, 3, dtype=D64), 0.1, 0.9,
                              False, True, torch.from_numpy(_mask32(img)))
        elif obj == "mse":
            ref = ((x - t64) ** 2).mean(dim=(1, 2, 3))
        else:
            ref = -(t64 * torch.log(1e-6 + x) + (1 - t64) * torch.log(1e-6 + 1 - x)).sum(dim=(1, 2, 3))
        ref.sum().backward()
        minv = orc.inverse_total_matrix(*orc.rotation_around_grid_centroid(poses), 64, 128)
        vt = torch.tensor(np.repeat(occ.reshape(1, 64, 64, 64, 1), V, 0).astype(np.float64), requires_grad=True)
        grid = rc.resample(vt, torch.from_numpy(minv.astype(np.float64)), 128)
        with prelu_kinks(W, masks=masks):
            imgo = orc.rendernet_shader(grid.float(), W)
        dv, = torch.autograd.grad(imgo, vt, torch.from_numpy(x.grad.numpy().astype(np.float32)))
        o = torch.tensor(occ.astype(np.float64), requires_grad=True)
        rs = sum(((o.narrow(a, 1, 63) - o.narrow(a, 0, 63)) ** 2).sum() for a in range(3)) / o.numel()
        rb = (o * (1 - o)).mean()
        (ls * rs + lb * rb).backward()
        want = (dv.sum(0)[..., 0].numpy() + o.grad.numpy()) * keep
        e = dict(loss=float((np.abs(loss - ref.detach().numpy()) / ref.detach().numpy()).max()), g=_rel(g.cpu().numpy(), want),
                 rs=abs(reg[0] - rs.item()) / rs.item(), rb=abs(reg[1] - rb.item()) / rb.item())
        print(f"[{precision}] {obj} V=4 vs frozen-kink oracle: " + ", ".join(f"{k} {v:.2e}" for k, v in e.items()) +
              f"; hull {int(keep.sum())} voxels")
        assert (g.cpu().numpy()[keep == 0] == 0).all()
        assert e["loss"] < 1e-6 and e["rs"] < 1e-6 and e["rb"] < 1e-6, e
        assert e["g"] < (3e-4 if precision == "exact" else 6e-3), e


def _mask32(n):
    """The fp32 black-background mask phong_pixel evaluates, emulated with one rounding per operation (as the pose fit's test)."""
    f32 = lambda x: np.asarray(x, np.float64).astype(np.float32).astype(np.float64)   # noqa: E731
    a = n.astype(np.float64)
    s = f32(a[..., 0] * a[..., 0])
    s = f32(a[..., 1] * a[..., 1] + s)
    s = f32(a[..., 2] * a[..., 2] + s)
    arg = f32(255.0 * f32(np.sqrt(s)) - 150.0)
    with np.errstate(over="ignore"):
        return f32(1.0 / f32(1.0 + f32(np.exp(-arg))))[..., None]


# ----------------------------------------------------------------------------------------- carving
def _hull_numpy(poses, cols, S=64, N=128):
    """The carving rule restated on the host: each sample point's trilinear support from the fp32 coordinates the device computes
    (rc.sample_coords): corner (dx, dy, dz) of the point's cell counts iff its weight is nonzero, i.e. dx = 0 or the coordinate's
    fraction is nonzero (and likewise in y, z).  observed_v = voxels in some point's support; inside_v = those of points in a
    silhouette column."""
    from rendernet_b200.engine import pose_to_matrix
    minv = pose_to_matrix(poses, S, N)                                  # the matrices the device samples with
    g = rc.output_grid(N, True)
    col_of_point = np.repeat(np.arange(N * N), N)                       # flat order [p, q, r]: column p * N + q
    V = len(poses)
    observed = np.zeros((V, S ** 3), bool)
    inside = np.zeros((V, S ** 3), bool)
    for v in range(V):
        c = rc.sample_coords(minv[v:v + 1], g)[0]                        # [3, P] fp32
        ok = ((c >= 0) & (c < S - 1)).all(0)
        c = c[:, ok]
        pin = cols[v].reshape(-1)[col_of_point[ok]]
        base = np.floor(c)
        frac = c - base
        i0 = base.astype(np.int64)
        for dz in (0, 1):
            for dy in (0, 1):
                for dx in (0, 1):
                    nz = ((dx == 0) | (frac[0] != 0)) & ((dy == 0) | (frac[1] != 0)) & ((dz == 0) | (frac[2] != 0))
                    k = ((i0[2] + dz) * S + (i0[1] + dy)) * S + (i0[0] + dx)
                    observed[v, k[nz]] = True
                    inside[v, k[nz & pin]] = True
    return (observed.any(0) & (~observed | inside).all(0)).reshape(S, S, S).astype(np.uint8)


def test_carving_keeps_the_shape_and_matches_numpy():
    """Masks from each fixture shape's own resampled grid at 8 turntable views: the hull contains every occupied voxel (exactly,
    by construction) and equals the NumPy restatement on the device's fp32 sample coordinates."""
    from rendernet_b200.shape_fit import carve, mask_columns
    poses = _turntable(8)
    for name in SHAPES:
        vox = _shape(name)
        masks = _shape_masks(vox, poses)
        keep = carve(poses, masks)
        missing = int(((vox > 0) & (keep == 0)).sum())
        want = _hull_numpy(poses, mask_columns(masks, 1))
        diff = int((keep != want).sum())
        print(f"{name}: {int(vox.sum())} occupied, hull {int(keep.sum())}, missing {missing}, differs from NumPy at {diff}")
        assert missing == 0 and diff == 0


# ----------------------------------------------------------------------------------------- fixed point, chunking, device paths
def test_fixed_point_stays_fixed():
    """Targets = the fit's own "phong" renders of a grid in [0, 1], lambda = 0: the loss is exactly 0, g exactly 0, and a step
    leaves the occupancy bit-identical (an all-zero image gradient takes the loss scale 1 without a retry or a NaN)."""
    from rendernet_b200.shape_fit import ShaderShapeFit
    V = 4
    fit = ShaderShapeFit(None, _turntable(V), light=_lights(V), batch=V, lambda_smooth=0.0, lambda_bin=0.0)
    occ = _soft_chair()
    target = fit.render(occ)["shaded"]
    loss, reg, g = fit.gradients(occ, target)
    assert (loss == 0).all(), loss
    assert bool((g == 0).all()), float(g.abs().max())
    assert fit.ig.last_loss_scale == 1.0
    state = fit.init_state(occ)
    before = state["occ"].clone()
    loss2, _ = fit.step(state, target)
    assert (loss2 == 0).all() and torch.equal(state["occ"], before)


def test_chunking_equals_one_batch():
    """V = 6 in one batch of 6 equals three batches of 2: the loss within 1e-12 relative, g within 1e-5 of scale (the noise of
    the resampler's fp32 atomics)."""
    from rendernet_b200.shape_fit import ShaderShapeFit
    V = 6
    W = orc.init_shader_weights(seed=1, alpha_range=(0.05, 0.3), bias_jitter=0.02)
    occ, poses = _soft_chair(), _turntable(V)
    tgt = np.random.default_rng(9).random((V, 512, 512, 3)).astype(np.float32)
    out = {}
    for batch in (6, 2, 4):
        fit = ShaderShapeFit(W, poses, light=_lights(V), batch=batch, lambda_smooth=0.3, lambda_bin=0.2)
        loss, reg, g = fit.gradients(occ, tgt)
        out[batch] = (loss, reg, g.cpu().numpy())
        del fit
        torch.cuda.empty_cache()
    for batch in (2, 4):                                                 # 4: a padded last chunk
        el = float(np.abs(out[batch][0] - out[6][0]).max() / np.abs(out[6][0]).max())
        eg = _rel(out[batch][2], out[6][2])
        print(f"batch {batch} vs 6: loss {el:.2e}, g {eg:.2e}")
        assert el <= 1e-12 and eg <= 1e-5 and np.array_equal(out[batch][1], out[6][1])


def test_device_inputs_and_outputs_of_the_shader_gradients():
    """ShaderInputGradients.forward on a CUDA tensor renders the NumPy input's image bit for bit; backward(dvox_on_device=True)
    returns a CUDA tensor that agrees with the NumPy return within the resampler's atomics noise (1e-5 of scale)."""
    from rendernet_b200.backward import ShaderInputGradients
    ig = ShaderInputGradients(None, 2)
    vox = np.repeat(_soft_chair().reshape(1, 64, 64, 64, 1), 2, 0)
    poses = _turntable(2)
    a = ig.forward(vox, poses).clone()
    b = ig.forward(_d(vox), poses)
    assert torch.equal(a, b)
    dimg = np.random.default_rng(3).standard_normal(tuple(b.shape)).astype(np.float32) * 1e-3
    dn, pn_ = ig.backward(dimg, want_dpose=True)
    dd, pd_ = ig.backward(dimg, want_dpose=True, dvox_on_device=True)
    assert isinstance(dn, np.ndarray) and isinstance(dd, torch.Tensor) and dd.is_cuda
    e = _rel(dd.cpu().numpy(), dn)
    print(f"dvox device vs host {e:.2e}")
    assert e <= 1e-5


def test_binvox_zero_length_run_decodes_on_the_device(tmp_path):
    """A file holding the reference writer's (value, 0) pairs decodes on the device (rn_binvox_decode) to the written grid."""
    from rendernet_b200 import binvox_rw
    g = np.load(os.path.join(GOLDEN, "binvox_write.npz"))
    grid = np.unpackbits(g["runs_bits"]).reshape(64, 64, 64).astype(bool)
    binvox_rw.save_binvox(grid, str(tmp_path / "runs.binvox"))
    with open(tmp_path / "runs.binvox", "rb") as f:
        assert (binvox_rw.read_rle(f)[3][:, 1] == 0).sum() == 3          # after runs of 255, 510 and 255
    with open(tmp_path / "runs.binvox", "rb") as f:
        dv = binvox_rw.read_to_device(f)
    assert np.array_equal(dv.cpu().numpy().reshape(64, 64, 64), grid.astype(np.float32))


# ----------------------------------------------------------------------------------------- run and command line
def test_short_run_decreases_the_loss():
    """20 steps from the carved hull with seeded weights on targets rendered from the chair at 8 views: the data loss ends below
    the first step's.  The IoU at 0.1 against the truth is printed, not asserted (untrained weights give it no meaning)."""
    from rendernet_b200.shape_fit import ShaderShapeFit
    V = 8
    poses = _turntable(V)
    fit = ShaderShapeFit(None, poses, light=_lights(V), batch=V)
    truth = _shape("chair")
    target = fit.render(truth)["shaded"]
    seen = []
    out = fit.run(target, masks=_shape_masks(truth, poses), steps=20, callback=lambda k, loss, reg, occ: seen.append(k))
    total = out["loss"].sum(1)
    final = fit.loss(out["occupancy"], target).sum()
    occ = out["occupancy"] > 0.1
    iou = float((occ & (truth > 0)).sum() / max((occ | (truth > 0)).sum(), 1))
    print(f"loss {total[0]:.6e} -> {total[-1]:.6e} (after the last step {final:.6e}); hull {int(out['keep'].sum())}, "
          f"IoU at 0.1 {iou:.3f}, R {out['reg'][-1]}")
    assert seen == list(range(20)) and out["loss"].shape == (20, V)
    assert total[-1] < total[0] and final < total[0]
    assert ((out["occupancy"] >= 0) & (out["occupancy"] <= 1)).all() and (out["occupancy"][out["keep"] == 0] == 0).all()


def test_command_line_reconstructs_from_named_pngs(tmp_path):
    """python -m rendernet_b200.shape_fit on PNG targets named by the dataset convention (poses from the names): shape.binvox reads
    back through read_as_3d_array and rn_binvox_decode, fit.json's last loss is below its first, and one PNG per view."""
    from PIL import Image
    from rendernet_b200 import binvox_rw
    from rendernet_b200.shape_fit import ShaderShapeFit, main
    V = 4
    az = [30 + 90 * k for k in range(V)]
    from rendernet_b200.RenderNet_demo import compute_pose_param
    poses = np.concatenate([compute_pose_param(a, 60, 3.3) for a in az]).astype(np.float32)
    light = [math.radians(275.0), math.radians(60.0)]
    fit = ShaderShapeFit(None, poses, light=light, batch=V)
    u8 = fit.render(_shape("chair"))["shaded_u8"]
    del fit
    torch.cuda.empty_cache()
    paths = []
    for k in range(V):
        p = tmp_path / f"chair_p{az[k]}_t60_r3.3.png"
        Image.fromarray(u8[k]).save(p)
        paths.append(str(p))
    res = main(paths + ["--weights", str(tmp_path / "none.pb"), "--steps", "4", "--batch", "2", "--out", str(tmp_path / "out")])
    with open(tmp_path / "out" / "fit.json") as f:
        saved = json.load(f)
    assert saved == json.loads(json.dumps(res))
    print({k: saved[k] for k in ("loss", "R_s", "R_b", "hull_size", "occupied_at_threshold")})
    assert np.allclose(saved["poses"], poses, rtol=0, atol=1e-6)
    assert len(saved["loss"]) == 4 and saved["loss"][-1] < saved["loss"][0]
    occ = np.load(tmp_path / "out" / "occupancy.npy")
    with open(tmp_path / "out" / "shape.binvox", "rb") as f:
        v = binvox_rw.read_as_3d_array(f)
    assert np.array_equal(v.data, occ > 0.1) and saved["occupied_at_threshold"] == int((occ > 0.1).sum())
    with open(tmp_path / "out" / "shape.binvox", "rb") as f:
        assert np.array_equal(binvox_rw.read_to_device(f).cpu().numpy().reshape(64, 64, 64), (occ > 0.1).astype(np.float32))
    for k in range(V):
        assert np.asarray(Image.open(tmp_path / "out" / f"render_{k}.png")).shape == (512, 512, 3)
