#!/usr/bin/env python
"""Cost of the Shader shape fit on one GPU (the card's name, power limit and max SM clock are read in the same run).

1. One ShaderShapeFit step at V = 8 and V = 24 views (seeded weights, the chair, turntable poses, objective "phong", batch 8,
   both precisions), split per chunk into the network forward (ShaderInputGradients.forward, tape recorded), the objective
   (rn_phong_composite_loss_grad), the backward walk to dL/dgrid, the resampler backward (rn_resample_backward_f32, timed alone on
   the walk's dL/dgrid; the walk's time is ShaderInputGradients.backward minus it), and the update (rn_voxel_fit_grad over all V
   rows + rn_adam_step + the clamp).  Each part is bracketed by torch.cuda.synchronize() and timed with the host clock, summed
   over the chunks, after `--warmup` full steps; mean and spread over `--steps` steps.  The whole ShaderShapeFit.step is timed
   the same way, with its peak device memory (torch.cuda.max_memory_allocated).
2. `carve` at V = 8 (masks from the chair's own resampled grid), host clock around a synchronised call.
3. rn_voxel_fit_grad alone at V = 8, S = 64 (dvox, occ, keep read; g written), CUDA events around `--kernel-reps` launches,
   against its HBM floor: the bytes it must move, from the shapes, over the H100 SXM data sheet's 3.35 TB/s."""
import argparse
import math
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from rendernet_b200 import ops  # noqa: E402
from rendernet_b200.RenderNet_demo import compute_pose_param  # noqa: E402
from rendernet_b200.engine import pose_to_matrix  # noqa: E402
from rendernet_b200.shader_fit import light_dir  # noqa: E402
from rendernet_b200.shape_fit import ShaderShapeFit, carve  # noqa: E402

HBM = 3.35e12                # H100 SXM data sheet, HBM3 bytes/s


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                      # noqa: BLE001
        return f"{torch.cuda.get_device_name(0)} (nvidia-smi unavailable: {e})"


def chair():
    bv = np.load(os.path.join(ROOT, "tests", "golden", "binvox.npz"))
    return np.unpackbits(bv["chair_bits"]).reshape(64, 64, 64).astype(np.float32)


def turntable(V):
    return np.concatenate([compute_pose_param(360.0 * k / V, 60.0, 3.3) for k in range(V)]).astype(np.float32)


def lights(V):
    return np.stack([np.linspace(240, 310, V) * math.pi / 180, np.full(V, math.radians(60.0))], 1)


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, 1e3 * (time.perf_counter() - t0)


def chair_masks(poses):
    V = len(poses)
    v = torch.from_numpy(np.repeat(chair().reshape(1, 64, 64, 64, 1), V, 0)).cuda()
    grid = ops.resample(v, torch.from_numpy(pose_to_matrix(poses, 64, 128)).cuda(), 128, True)
    cols = (grid[..., 0] > 0).any(-1).cpu().numpy()
    return np.repeat(np.repeat(cols, 4, 1), 4, 2)


def fit_step(args, V, precision):
    poses = turntable(V)
    fit = ShaderShapeFit(None, poses, light=lights(V), batch=8, precision=precision)
    fit.keep = carve(poses, chair_masks(poses))
    target = torch.rand((V, 512, 512, 3), device="cuda", generator=torch.Generator("cuda").manual_seed(0))
    state = fit.init_state(0.5 * fit.keep.astype(np.float32))
    for _ in range(args.warmup):
        fit.step(state, target)
    parts = {k: [] for k in ("forward", "objective", "backward to dL/dgrid", "resampler backward", "fit_grad + adam", "step")}
    keep = torch.from_numpy(fit.keep.reshape(-1)).cuda()
    torch.cuda.reset_peak_memory_stats()
    for _ in range(args.steps):
        occ = state["occ"]
        vox = occ.reshape(1, 64, 64, 64, 1).expand(fit.B, 64, 64, 64, 1)
        dv = torch.empty((V, 64, 64, 64), device="cuda")
        acc = dict.fromkeys(parts, 0.0)
        for v0, n, rows in fit._chunks():
            img, t = timed(lambda: fit.ig.forward(vox, poses[rows]))
            acc["forward"] += t
            tg = target[torch.from_numpy(rows).cuda()]
            ld = torch.from_numpy(light_dir(fit.light[rows])).cuda()
            (_, dimg, _), t = timed(lambda: ops.phong_composite_loss_grad(img, tg, ld, (1.0, 1.0, 1.0), 0.1, 0.9))
            acc["objective"] += t
            (d, _), tb = timed(lambda: fit.ig.backward(dimg, want_dvox=True, want_dpose=False, dvox_on_device=True))
            _, tr = timed(lambda: ops.resample_backward(fit.ig.vox, fit.ig.minv, fit.ig.last_dgrid, True, True, False))
            acc["backward to dL/dgrid"] += tb - tr
            acc["resampler backward"] += tr
            dv[v0:v0 + n] = d[:n, ..., 0]
        m, vv = torch.zeros_like(occ), torch.zeros_like(occ)
        occ2 = occ.clone()

        def update():
            g, _ = ops.voxel_fit_grad(dv, occ2, keep, fit.lambda_smooth, fit.lambda_bin)
            ops.adam_step(occ2, g, m, vv, fit.lr, 0.9, 0.999, 1e-8)
            occ2.clamp_(0.0, 1.0)
        _, t = timed(update)
        acc["fit_grad + adam"] += t
        _, t = timed(lambda: fit.step(state, target))
        acc["step"] += t
        for k in parts:
            parts[k].append(acc[k])
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    print(f"[{precision}] shape-fit step V={V} batch 8 ('phong'): " + ", ".join(
        f"{k} {np.mean(v):.2f} ms ({min(v):.2f}-{max(v):.2f})" for k, v in parts.items()) + f"; peak memory {peak:.2f} GiB",
        flush=True)
    del fit, state
    torch.cuda.empty_cache()


def carve_time(args):
    poses = turntable(8)
    masks = chair_masks(poses)
    carve(poses, masks)
    ts = [timed(lambda: carve(poses, masks))[1] for _ in range(args.steps)]
    print(f"carve V=8: {np.mean(ts):.2f} ms ({min(ts):.2f}-{max(ts):.2f})", flush=True)


def kernel(args):
    V, S = 8, 64
    n = S ** 3
    g = torch.Generator(device="cuda").manual_seed(1)
    dvox = torch.randn((V, n), device="cuda", generator=g)
    occ = torch.rand(n, device="cuda", generator=g)
    keep = (torch.rand(n, device="cuda", generator=g) < 0.5).to(torch.uint8)
    out = torch.empty(n, device="cuda")
    reg = torch.empty(2, device="cuda", dtype=torch.float64)
    from rendernet_b200._lib import lib
    work = torch.empty(int(lib.rn_voxel_fit_grad_workspace(S)), device="cuda", dtype=torch.float64)

    def launch():
        lib.rn_voxel_fit_grad(dvox.data_ptr(), occ.data_ptr(), keep.data_ptr(), out.data_ptr(), reg.data_ptr(), work.data_ptr(),
                              V, S, 0.1, 0.01, torch.cuda.current_stream().cuda_stream)
    for _ in range(10):
        launch()
    e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
    e0.record()
    for _ in range(args.kernel_reps):
        launch()
    e1.record()
    e1.synchronize()
    us = 1e3 * e0.elapsed_time(e1) / args.kernel_reps
    nbytes = V * n * 4 + n * 4 + n + n * 4               # dvox, occ, keep read; g written
    floor = 1e6 * nbytes / HBM
    print(f"rn_voxel_fit_grad V=8 S=64: {us:.1f} us for {nbytes / 1e6:.1f} MB, HBM floor {floor:.1f} us "
          f"({us / floor:.1f}x the floor, {nbytes / us / 1e6:.2f} TB/s)", flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--kernel-reps", type=int, default=500)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("shape_fit_step_time.py measures on a GPU; none found")
    print("card:", card(), flush=True)
    kernel(args)
    carve_time(args)
    for V in (8, 24):
        for precision in ("exact", "fast"):
            fit_step(args, V, precision)


if __name__ == "__main__":
    main()
