#!/usr/bin/env python
"""Training on random patches (rendernet_b200.training, patch_size=P): time and peak memory of one optimiser step of both
trainers on one GPU at B = 1, 8, 24 and P = 32, 64, 128 (128 = whole frames), exact and fast precision, CUDA events around
fwd+loss+bwd (loss_and_gradients) and Adam (apply_gradients) separately; then the windowed fused resample + e_conv1 kernels
alone at B = 24 against the whole-grid launch.
  python scripts/patch_train_step_time.py [--steps 3] [--reps 20] [--batches 1,8,24]"""
import argparse
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from rendernet_b200 import ops  # noqa: E402
from rendernet_b200.engine import pose_to_matrix  # noqa: E402
from rendernet_b200.training import ShaderTrainer, TextureTrainer  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=3)
ap.add_argument("--reps", type=int, default=20)
ap.add_argument("--batches", default="1,8,24")
args = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("patch_train_step_time: needs a CUDA device")
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip().splitlines()
print(f"[patch_train_step_time] device: {torch.cuda.get_device_name()} | nvidia-smi name, power limit, max SM clock: "
      f"{card[0] if card else 'n/a'}", flush=True)
PATCHES = (32, 64, 128)


def scene(B, rng):
    """A filled 32^3 box in sparse noise, one generic pose: the patches at the drawn origins cover both object and empty space."""
    vox = (rng.random((B, 64, 64, 64, 1)) < 0.1).astype(np.float32)
    vox[:, 16:48, 16:48, 16:48] = 1.0
    z = rng.standard_normal((B, 199)).astype(np.float32)
    poses = np.tile(np.array([[4.36, 1.05, 3.3]], np.float32), (B, 1))
    return vox, z, poses, rng.random((B, 512, 512, 3)).astype(np.float32), rng.random((B, 512, 512, 3)).astype(np.float32)


# ------------------------------------------------------------------------------------------------ whole steps
rows = []
for network in ("shader", "texture"):
    for B in (int(b) for b in args.batches.split(",")):
        vox, z, poses, t_img, t_nrm = scene(B, np.random.default_rng(0))
        inputs = (vox, poses, t_img) if network == "shader" else (vox, z, poses, t_img, t_nrm)
        for precision in ("exact", "fast"):
            tr = (ShaderTrainer(None, B, precision=precision, seed=1) if network == "shader"
                  else TextureTrainer(None, B, precision=precision, seed=1))
            for P in PATCHES:
                tr.step(*inputs, patch_size=P)                                   # warm-up: allocator, packs of this shape
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
                t_f = t_a = 0.0
                for _ in range(args.steps):
                    e[0].record()
                    loss, grads = tr.loss_and_gradients(*inputs, patch_size=P)   # forward + loss + backward (synchronises)
                    e[1].record()
                    tr.apply_gradients(grads)
                    e[2].record()
                    torch.cuda.synchronize()
                    t_f += e[0].elapsed_time(e[1])
                    t_a += e[1].elapsed_time(e[2])
                    del grads
                t_f, t_a = t_f / args.steps, t_a / args.steps
                peak = torch.cuda.max_memory_allocated() / 2 ** 30
                rows.append((network, B, P, precision, t_f, t_a, peak))
                print(f"[patch_train_step_time] {network} {precision} B={B} P={P}: {t_f + t_a:.1f} ms/step = fwd+loss+bwd "
                      f"{t_f:.1f} ms + Adam {t_a:.1f} ms; peak memory {peak:.2f} GiB; last crop {tr.last_crop}", flush=True)
            del tr
            torch.cuda.empty_cache()

print("\n| network | B | P | exact: fwd+loss+bwd / Adam / peak | fast: fwd+loss+bwd / Adam / peak | exact step vs P = 128 |")
print("|---|---|---|---|---|---|")
full = {(n, B, pr): f + a for n, B, P, pr, f, a, _ in rows if P == 128}
for network, B, P in sorted({(r[0], r[1], r[2]) for r in rows}, key=lambda k: (k[0] != "shader", k[1], k[2])):
    cell = {pr: (f, a, m) for n, b, p, pr, f, a, m in rows if (n, b, p) == (network, B, P)}
    ex, fa = cell["exact"], cell["fast"]
    print(f"| {network} | {B} | {P} | {ex[0]:.1f} ms / {ex[1]:.1f} ms / {ex[2]:.2f} GiB | {fa[0]:.1f} ms / {fa[1]:.1f} ms / "
          f"{fa[2]:.2f} GiB | {(ex[0] + ex[1]) / full[network, B, 'exact']:.3f} |")


# ------------------------------------------------------------------------------------------------ fused kernels alone, B = 24
def timed(fn):
    for _ in range(3):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(args.reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / args.reps                                # us per call


B = 24
rng = np.random.default_rng(1)
d = lambda t: torch.from_numpy(t).cuda()                                    # noqa: E731
vox, _, poses, _, _ = scene(B, rng)
vox = d(vox)
tex = d(rng.random((B, 64, 64, 64, 4)).astype(np.float32))
minv = d(pose_to_matrix(poses, 64, 128))
w1, w5 = d(rng.standard_normal((5, 5, 5, 1, 8)).astype(np.float32) * 0.1), d(rng.standard_normal((5, 5, 5, 5, 8)).astype(np.float32) * 0.1)
b8, a8 = d(np.zeros(8, np.float32)), d(np.full(8, 0.2, np.float32))
print()
for fmt, name in ((2, "exact"), (0, "fast")):
    whole1 = timed(lambda: ops.resample_conv1(vox, minv, 128, w1, b8, a8, fmt=fmt))
    whole5 = timed(lambda: ops.resample5_conv1(vox, tex, minv, 128, w5, b8, a8, fmt=fmt))
    print(f"[patch_train_step_time] fused e_conv1 B={B} {name}, whole grid: resample_conv1 {whole1:.0f} us, "
          f"resample5_conv1 {whole5:.0f} us", flush=True)
    for P in (32, 64, 128):
        for origin in ((0, 0), ((128 - P) // 2, (128 - P) // 2)):
            win = origin + (P, P)
            u1 = timed(lambda: ops.resample_conv1(vox, minv, 128, w1, b8, a8, fmt=fmt, window=win))
            u5 = timed(lambda: ops.resample5_conv1(vox, tex, minv, 128, w5, b8, a8, fmt=fmt, window=win))
            share = (P / 128) ** 2
            print(f"[patch_train_step_time]   window {win}: resample_conv1 {u1:.0f} us ({u1 / whole1:.3f} of the whole grid; "
                  f"area share {share:.4f}), resample5_conv1 {u5:.0f} us ({u5 / whole5:.3f})", flush=True)
