#!/usr/bin/env python
"""Time of one training step of the Texture+Normal network (rendernet_b200.training.TextureTrainer: forward with tape, two MSE
losses, backward with all 186 weight gradients, Adam, re-pack) on one GPU, CUDA events around whole steps, both precisions, at
B = 1 (config_RenderNet_texture.json: keep_prob 1.0) and B = 8 (keep_prob 0.75); then the new weight-gradient kernels alone at
B = 24: the FC parameter gradient against its HBM floor, the three decoder filter gradients and e_conv1's filter gradient with
the re-materialisation of its 128^3 x 5 grid.
  python scripts/texture_train_step_time.py [--steps 5] [--reps 20]"""
import argparse
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from rendernet_b200 import ops  # noqa: E402
from rendernet_b200.engine import pose_to_matrix  # noqa: E402
from rendernet_b200.training import TextureTrainer  # noqa: E402

HBM_BYTES_PER_S = 3.35e12           # H100 SXM data sheet

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=5)
ap.add_argument("--reps", type=int, default=20)
args = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("texture_train_step_time: needs a CUDA device")
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip().splitlines()
print(f"[texture_train_step_time] device: {torch.cuda.get_device_name()} | nvidia-smi name, power limit, max SM clock: "
      f"{card[0] if card else 'n/a'}", flush=True)


def scene(B, rng):
    vox = (rng.random((B, 64, 64, 64, 1)) < 0.1).astype(np.float32)
    vox[:, 16:48, 16:48, 16:48] = 1.0
    z = rng.standard_normal((B, 199)).astype(np.float32)
    poses = np.tile(np.array([[4.36, 1.05, 3.3]], np.float32), (B, 1))
    return vox, z, poses, rng.random((B, 512, 512, 3)).astype(np.float32), rng.random((B, 512, 512, 3)).astype(np.float32)


# ------------------------------------------------------------------------------------------------ whole steps
for B, keep in ((1, 1.0), (8, 0.75)):
    inputs = scene(B, np.random.default_rng(0))
    for precision in ("exact", "fast"):
        torch.cuda.reset_peak_memory_stats()
        tr = TextureTrainer(None, B, precision=precision, keep_prob=keep, seed=1)
        losses = [tr.step(*inputs) for _ in range(2)]                          # warm-up: allocator, first packs
        e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        t_f = t_a = 0.0
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.steps):
            e[0].record()
            loss, grads = tr.loss_and_gradients(*inputs)                        # forward + losses + backward (synchronises)
            e[1].record()
            tr.apply_gradients(grads)
            e[2].record()
            torch.cuda.synchronize()
            t_f += e[0].elapsed_time(e[1])
            t_a += e[1].elapsed_time(e[2])
            losses.append(loss)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.steps
        print(f"[texture_train_step_time] {precision} B={B} keep_prob={keep}: {ms:.1f} ms/step ({B * 1000 / ms:.2f} frames/s) = "
              f"forward+loss+backward {t_f / args.steps:.1f} ms + Adam {t_a / args.steps:.1f} ms; "
              f"{len(grads)} variables, {sum(v.numel() for v in tr.store.vars.values()) / 1e6:.1f} M; loss {losses[0]:.5f} -> "
              f"{losses[-1]:.5f}; peak memory {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB", flush=True)
        del tr, grads
        torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ kernels alone, B = 24
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
K, N = 199, 32 * 32 * 32 * 4
x, gy, z = d(rng.standard_normal((B, K)).astype(np.float32)), d(rng.standard_normal((B, N)).astype(np.float32)), \
    d(rng.standard_normal((B, N)).astype(np.float32))
alpha = d(rng.uniform(-0.3, 0.3, N).astype(np.float32))
us = timed(lambda: ops.fully_connected_param_grad(x, gy, z, alpha))
nbytes = (K * N + 3 * N) * 4 + (2 * B * N + B * K + N) * 4
print(f"[texture_train_step_time] rn_fully_connected_param_grad B={B} K={K} N={N}: {us:.1f} us; {nbytes / 1e6:.1f} MB moved, "
      f"HBM floor {nbytes / HBM_BYTES_PER_S * 1e6:.1f} us at {HBM_BYTES_PER_S / 1e12:.2f} TB/s -> "
      f"{nbytes / HBM_BYTES_PER_S * 1e6 / us * 100:.0f} % of the floor's speed", flush=True)
del x, gy, z, alpha

for name, S, C, tr_, s, cb in (("e_tex_conv0", 32, 4, True, 1, 4), ("e_tex_conv1", 32, 4, True, 2, 8),
                               ("e_tex_conv2", 64, 8, False, 1, 4)):
    xin = d(rng.standard_normal((B, S, S, S, C)).astype(np.float32))
    So = S * s if tr_ else S
    g = d(rng.standard_normal((B, So, So, So, cb)).astype(np.float32))
    zz = d(rng.standard_normal((B, So, So, So, cb)).astype(np.float32))
    al = d(rng.uniform(-0.3, 0.3, cb).astype(np.float32))
    if tr_:
        pad = (ops.same_pad_before(S * s, 4, s),) * 3
        wg = lambda: ops.conv_weight_grad_direct(xin, g, (4, 4, 4), (s, s, s), pad, Ca=C, Cb=cb)          # noqa: E731
    else:
        pad = (ops.same_pad_before(S, 4, 1),) * 3
        wg = lambda: ops.conv_weight_grad_direct(g, xin, (4, 4, 4), (1, 1, 1), pad, Ca=cb, Cb=C)          # noqa: E731
    us_p = timed(lambda: ops.prelu_grad_f32(g, zz, al))
    us_w = timed(wg)
    print(f"[texture_train_step_time] {name} B={B}: rn_prelu_grad_f32 ({So}^3 x {cb}) {us_p:.1f} us, filter gradient "
          f"({'transposed ' if tr_ else ''}s{s}, Ca x Cb = {C if tr_ else cb} x {cb if tr_ else C}) {us_w:.1f} us", flush=True)
    del xin, g, zz, al
    torch.cuda.empty_cache()

vox = d((rng.random((B, 64, 64, 64, 1)) < 0.2).astype(np.float32))
tex = d(rng.random((B, 64, 64, 64, 4)).astype(np.float32))
minv = d(pose_to_matrix(np.tile(np.array([[4.36, 1.05, 3.3]], np.float32), (B, 1)), 64, 128))
g16 = ops.cast_to_16(d(rng.standard_normal((B, 64, 64, 64, 8)).astype(np.float32)), fmt=2)
pad = (ops.same_pad_before(128, 5, 2),) * 3


def grid():
    return ops.concat_channels(ops.resample(vox, minv, 128, True), ops.resample(tex, minv, 128, True))


q = grid()
us_g = timed(grid)
us_c = timed(lambda: ops.conv_weight_grad_direct(g16, q, (5, 5, 5), (2, 2, 2), pad, Ca=8, Cb=5))
print(f"[texture_train_step_time] e_conv1 filter gradient B={B} (exact g): grid re-materialisation {us_g:.0f} us + (8,5) "
      f"correlation {us_c:.0f} us = {us_g + us_c:.0f} us", flush=True)
