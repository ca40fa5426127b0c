#!/usr/bin/env python
"""Cost of reproducibility on one GPU: each fixed-order twin against its atomic kernel, and one step of each fit with
torch.use_deterministic_algorithms off and on (the card's name and power limit are read in the same run).

1. Kernels, at B = 5 and 24: rn_resample_backward (C = 1, 64^3 -> 128^3, dvox + dMinv), rn_resample5_backward (whole grid,
   dvox + dtex + dMinv), rn_phong_recon_loss_grad, rn_phong_composite_loss_grad, rn_phong_shade_backward (TF composite, with
   albedo and d_light) and rn_image_loss_grad_items (MSE) at 512 x 512, each through its rendernet_b200.ops wrapper (so the
   twin's workspace allocation and zeroed outputs of the atomic path are in the time).  The two are alternated, `--reps`
   calls each between CUDA events, `--rounds` times; the median per call is printed.
2. Fits: ShaderPoseFit.step (B = 5), ShaderShapeFit.step (V = 8) and FaceReconstruction.step (B = 5), exact mode, the flag off
   and on alternated, each step bracketed by torch.cuda.synchronize() on the host clock after `--warmup` steps each way.

Without a GPU the script stops: no timing is made up."""
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
from oracle import rendernet_oracle as orc  # noqa: E402
from rendernet_b200 import ops  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                      # noqa: BLE001
        return f"{torch.cuda.get_device_name(0)} (nvidia-smi unavailable: {e})"


def chair(B):
    bv = np.load(os.path.join(ROOT, "tests", "golden", "binvox.npz"))
    v = np.unpackbits(bv["chair_bits"]).reshape(1, 64, 64, 64, 1).astype(np.float32)
    return np.ascontiguousarray(np.repeat(v, B, 0))


def kernel_cases(B):
    g = torch.Generator(device="cuda").manual_seed(B)
    r = lambda *s: torch.rand(s, device="cuda", generator=g)                                # noqa: E731
    poses = np.stack([np.linspace(3.5, 5.5, B), np.full(B, 0.9), np.full(B, 3.3)], 1).astype(np.float32)
    R, S = orc.rotation_around_grid_centroid(poses)
    minv = torch.from_numpy(orc.inverse_total_matrix(R, S, 64, 128)).cuda()
    vox, tex = torch.from_numpy(chair(B)).cuda(), r(B, 64, 64, 64, 4)
    G1, G5 = torch.randn(B, 128, 128, 128, 1, device="cuda", generator=g), torch.randn(B, 128, 128, 128, 5, device="cuda", generator=g)
    a, n, t, gc = (r(B, 512, 512, 3) for _ in range(4))
    ld, lc = torch.randn(B, 3, device="cuda", generator=g), torch.ones(B, 3, device="cuda")
    return {"resample_backward C=1": lambda: ops.resample_backward(vox, minv, G1, True),
            "resample5_backward": lambda: ops.resample5_backward(vox, tex, minv, G5),
            "phong_recon_loss_grad": lambda: ops.phong_recon_loss_grad(a, n, t, ld, lc),
            "phong_composite_loss_grad": lambda: ops.phong_composite_loss_grad(n, t, ld),
            "phong_shade_backward": lambda: ops.phong_shade_backward(n, gc, ld, albedo=a),
            "image_loss_grad_items": lambda: ops.image_loss_grad_items(a, t)}


def event_ms(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / reps


def kernels(args):
    for B in (5, 24):
        for name, fn in kernel_cases(B).items():
            t = {False: [], True: []}
            for flag in (False, True):                             # warm-up: module load, allocator
                torch.use_deterministic_algorithms(flag)
                fn()
            for _ in range(args.rounds):
                for flag in (False, True):
                    torch.use_deterministic_algorithms(flag)
                    t[flag].append(event_ms(fn, args.reps))
            torch.use_deterministic_algorithms(False)
            a, f = float(np.median(t[False])), float(np.median(t[True]))
            print(f"B={B:2d} {name:26s} atomic {a:8.3f} ms  fixed-order {f:8.3f} ms  ratio {f / a:5.2f}", flush=True)
        torch.cuda.empty_cache()


def host_ms(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0)


def fits(args):
    from oracle.shape_decoder import init_shape_decoder_weights
    from rendernet_b200.Reconstruct_RenderNet_Face import FaceReconstruction, create_param_center, pretrained_dict_from_texture_weights
    from rendernet_b200.RenderNet_demo import compute_pose_param
    from rendernet_b200.shader_fit import ShaderPoseFit
    from rendernet_b200.shape_fit import ShaderShapeFit
    rng = np.random.default_rng(3)
    pose_fit = ShaderPoseFit(None, chair(1)[0, ..., 0], objective="phong")
    pstate = dict(pose=create_param_center(250, 60, 60, 30),
                  light=np.stack([np.linspace(230, 320, 5) * math.pi / 180, np.full(5, math.radians(60.0))], 1).astype(np.float32))
    ptarget = torch.rand((5, 512, 512, 3), device="cuda")
    V = 8
    poses = np.concatenate([compute_pose_param(360.0 * k / V, 60.0, 3.3) for k in range(V)]).astype(np.float32)
    lights = np.stack([np.linspace(240, 310, V) * math.pi / 180, np.full(V, math.radians(60.0))], 1)
    shape_fit = ShaderShapeFit(None, poses, light=lights, batch=V)
    sstate = shape_fit.init_state(np.full((64, 64, 64), 0.5, np.float32))
    starget = torch.rand((V, 512, 512, 3), device="cuda")
    W = orc.init_texture_weights(seed=1, alpha_range=(-0.3, 0.3), bias_jitter=0.02)
    for k in list(W):
        if k.endswith("/alpha") and "/res" in k:
            W[k] = np.zeros_like(W[k])
    rec = FaceReconstruction(pretrained_dict_from_texture_weights(W), init_shape_decoder_weights(2), batch=5)
    fstate = dict(latent=(0.5 + 0.3 * rng.standard_normal((5, 200))).astype(np.float32), pose=create_param_center(270, 60, 90, 30),
                  texture=rng.standard_normal((5, 199)).astype(np.float32),
                  light=(np.linspace(230, 320, 5).reshape(5, 1) * math.pi / 180).astype(np.float32))
    ftarget = rng.random((5, 512, 512, 3)).astype(np.float32)
    cases = {"ShaderPoseFit.step B=5": lambda: pose_fit.step(pstate, ptarget),
             "ShaderShapeFit.step V=8": lambda: shape_fit.step(sstate, starget),
             "FaceReconstruction.step B=5": lambda: rec.step(fstate, ftarget)}
    for name, fn in cases.items():
        t = {False: [], True: []}
        for _ in range(args.warmup):
            for flag in (False, True):
                torch.use_deterministic_algorithms(flag)
                fn()
        for _ in range(args.steps):
            for flag in (False, True):
                torch.use_deterministic_algorithms(flag)
                t[flag].append(host_ms(fn))
        torch.use_deterministic_algorithms(False)
        a, f = float(np.median(t[False])), float(np.median(t[True]))
        print(f"{name:28s} flag off {a:8.2f} ms  on {f:8.2f} ms  ratio {f / a:5.3f}  (spread off {min(t[False]):.2f}-"
              f"{max(t[False]):.2f}, on {min(t[True]):.2f}-{max(t[True]):.2f})", flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--steps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("deterministic_time.py measures on a CUDA device; none is available")
    os.environ.pop("CUBLAS_WORKSPACE_CONFIG", None)
    print(f"card: {card()}", flush=True)
    kernels(args)
    fits(args)


if __name__ == "__main__":
    main()
