"""Cost of the shading-parameter gradients (DESIGN §8b): the three *_params backward entries against the entries they extend, at
B = 5 and 24 on 512^2 (CUDA events, alternated rounds, the median round reported), with the bytes each kernel must move and the
HBM floor at the H100 SXM data sheet's 3.35 TB/s; then one ShaderPoseFit and one FaceReconstruction step with fit_shading off
and on (seeded weights, alternated).  Prints the card's name and power limit first.

    python scripts/phong_params_time.py [--rounds 7] [--iters 50] [--fit_reps 5]
"""
import argparse
import math
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    return q or torch.cuda.get_device_name()


def time_pair(fa, fb, rounds, iters):
    """Median per-call ms of fa and fb over `rounds` alternated rounds of `iters` calls each."""
    for f in (fa, fb):
        f()
    torch.cuda.synchronize()
    res = {0: [], 1: []}
    for r in range(rounds):
        for k, f in ((0, fa), (1, fb)) if r % 2 == 0 else ((1, fb), (0, fa)):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                f()
            e1.record()
            e1.synchronize()
            res[k].append(e0.elapsed_time(e1) / iters)
    return float(np.median(res[0])), float(np.median(res[1]))


def kernels(rounds, iters):
    from rendernet_b200 import ops
    H = W = 512
    for B in (5, 24):
        rng = np.random.default_rng(B)
        d = lambda *s: torch.from_numpy(rng.random(s).astype(np.float32)).cuda()     # noqa: E731
        n, alb, tgt, g = d(B, H, W, 3), d(B, H, W, 3), d(B, H, W, 3), d(B, H, W, 3)
        ld, lc = d(B, 3) + 0.1, d(B, 3) + 0.5
        amb, ambv = 0.1, torch.full((B,), 0.1, device="cuda")
        px = B * H * W
        cases = [
            ("shade_backward tf+albedo", 60,
             lambda: ops.phong_shade_backward(n, g, ld, lc, amb, 0.9, albedo=alb),
             lambda: ops.phong_shade_backward(n, g, ld, lc, ambv, 0.9, albedo=alb, want_shading_grad=True)),
            ("composite_loss_grad", 36,
             lambda: ops.phong_composite_loss_grad(n, tgt, ld, lc, amb, 0.9),
             lambda: ops.phong_composite_loss_grad(n, tgt, ld, lc, ambv, 0.9, want_shading_grad=True)),
            ("recon_loss_grad", 60,
             lambda: ops.phong_recon_loss_grad(alb, n, tgt, ld, lc, amb, 0.9),
             lambda: ops.phong_recon_loss_grad(alb, n, tgt, ld, lc, ambv, 0.9, want_shading_grad=True)),
        ]
        for name, bpp, fa, fb in cases:
            ta, tb = time_pair(fa, fb, rounds, iters)
            floor = bpp * px / HBM * 1e3
            print(f"B={B:2d} {name:26s} existing {ta:.4f} ms, params {tb:.4f} ms ({tb / ta:.3f}x); {bpp * px / 1e6:.1f} MB, "
                  f"HBM floor {floor:.4f} ms ({floor / ta:.0%} / {floor / tb:.0%} of it)", flush=True)


def fits(reps):
    from oracle import rendernet_oracle as orc
    from oracle.shape_decoder import init_shape_decoder_weights
    from rendernet_b200.Reconstruct_RenderNet_Face import FaceReconstruction, pretrained_dict_from_texture_weights
    from rendernet_b200.RenderNet_demo import compute_pose_param
    from rendernet_b200.shader_fit import ShaderPoseFit
    bv = np.load(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "binvox.npz"))
    vox = np.unpackbits(bv["chair_bits"]).reshape(1, 64, 64, 64, 1).astype(np.float32)
    pose = np.tile(compute_pose_param(262.0, 54.0, 3.3)[0].astype(np.float32), (5, 1))
    light = np.tile(np.float32([math.radians(280.0), math.radians(60.0)]), (5, 1))
    off, on = (ShaderPoseFit(None, vox, objective="phong", fit_shading=f) for f in (False, True))
    target = off.render(dict(pose=pose, light=light))["shaded"]
    s_off, s_on = dict(pose=pose, light=light), dict(pose=pose, light=light, **on.initial_shading())
    W = orc.init_texture_weights(seed=61, alpha_range=(-0.3, 0.3), bias_jitter=0.02)
    Wp, Wd = pretrained_dict_from_texture_weights(W), init_shape_decoder_weights(62)
    r_off, r_on = (FaceReconstruction(Wp, Wd, fit_shading=f) for f in (False, True))
    rng = np.random.default_rng(3)
    st = dict(latent=np.full((5, 200), 0.5, np.float32), texture=rng.standard_normal((5, 199)).astype(np.float32),
              pose=np.tile(np.float32([math.radians(270.0), 0.0, 1.0]), (5, 1)), light=np.full((5, 1), 5.0, np.float32))
    ftarget = r_off.render(st)["compos"]
    for name, pair in (("ShaderPoseFit step (exact)", ((off, s_off, target), (on, s_on, target))),
                       ("FaceReconstruction step (exact)", ((r_off, st, ftarget), (r_on, dict(st, **r_on.initial_shading()),
                                                                                     ftarget)))):
        t = {0: [], 1: []}
        for k in (0, 1):
            fit, s, tg = pair[k]
            fit.step(s, tg)
        for r in range(reps):
            for k in ((0, 1) if r % 2 == 0 else (1, 0)):
                fit, s, tg = pair[k]
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fit.step(s, tg)
                torch.cuda.synchronize()
                t[k].append(time.perf_counter() - t0)
        a, b = np.median(t[0]) * 1e3, np.median(t[1]) * 1e3
        print(f"{name}: fit_shading off {a:.1f} ms, on {b:.1f} ms ({b / a:.3f}x); ranges "
              f"{min(t[0]) * 1e3:.1f}-{max(t[0]) * 1e3:.1f} / {min(t[1]) * 1e3:.1f}-{max(t[1]) * 1e3:.1f} ms", flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--fit_reps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("phong_params_time.py measures on the GPU; there is none")
    print("card:", card(), flush=True)
    kernels(args.rounds, args.iters)
    fits(args.fit_reps)


if __name__ == "__main__":
    main()
