#!/usr/bin/env python
"""Timing of one face-reconstruction step (Reconstruct_RenderNet_Face.FaceReconstruction.step, the reference's :402-412) at B = 5,
both precisions, CUDA events around work that ends in a device synchronise, mean of `--reps` runs after two warm-up runs.

Reports the shape decoder's forward (ShapeDecoderGradients.forward), its backward (dL/dvoxels on the device -> dL/dlatent on the
host), the rest of the step (Texture+Normal forward / backward, objective, host update) and the total; then each decoder layer
alone (rn_conv3d_f32 forward + epilogue, and its data gradient) with the achieved GFLOP/s from the layer's MAC count and the share
of the H100 SXM's 67 TFLOP/s fp32 data-sheet rate.  Weights are seeded (random); the cost does not depend on their values.
The card's name and power limit are read in the same run."""
import argparse
import math
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from rendernet_b200 import ops  # noqa: E402
from rendernet_b200.Reconstruct_RenderNet_Face import FaceReconstruction, create_param_center, pretrained_dict_from_texture_weights  # noqa: E402
from oracle import rendernet_oracle as orc  # noqa: E402  (seeded weights only)
from oracle.shape_decoder import CONV_LAYERS, init_shape_decoder_weights  # noqa: E402

FP32_PEAK = 67e12            # H100 SXM data sheet, dense fp32 (FLOP/s)


def timed(fn, reps):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                      # noqa: BLE001
        q = f"{torch.cuda.get_device_name(0)} (nvidia-smi unavailable: {e})"
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("reconstruction_step_time.py measures on a CUDA device; none is available")
    print(f"card: {card()}", flush=True)
    B = 5
    W = orc.init_texture_weights(seed=1, alpha_range=(-0.3, 0.3), bias_jitter=0.02)
    for k in list(W):
        if k.endswith("/alpha") and "/res" in k:
            W[k] = np.zeros_like(W[k])
    Wp, Wd = pretrained_dict_from_texture_weights(W), init_shape_decoder_weights(2)
    rng = np.random.default_rng(3)
    state = dict(latent=(0.5 + 0.3 * rng.standard_normal((B, 200))).astype(np.float32), pose=create_param_center(270, 60, 90, 30),
                 texture=rng.standard_normal((B, 199)).astype(np.float32),
                 light=(np.linspace(230, 320, 5).reshape(B, 1) * math.pi / 180).astype(np.float32))
    target = rng.random((B, 512, 512, 3)).astype(np.float32)
    dvox = torch.randn(B, 64, 64, 64, 1, device="cuda")
    for precision in ("exact", "fast"):
        rec = FaceReconstruction(Wp, Wd, batch=B, precision=precision)
        t_step = timed(lambda: rec.step(state, target), args.reps)
        t_fwd = timed(lambda: rec.sdg.forward(state["latent"]), args.reps)
        rec.sdg.forward(state["latent"])
        t_bwd = timed(lambda: rec.sdg.backward(dvox), args.reps)
        print(f"[{precision}] B={B} step {t_step:.2f} ms: shape decoder forward {t_fwd:.3f} ms, backward {t_bwd:.3f} ms "
              f"({100 * (t_fwd + t_bwd) / t_step:.1f} % of the step), rest {t_step - t_fwd - t_bwd:.2f} ms", flush=True)
        del rec
        torch.cuda.empty_cache()

    # each decoder layer alone: forward (with its epilogue) and data gradient
    side = {256: 4, 128: 8, 64: 16, 32: 32, 16: 64}
    tot = [0.0, 0.0]
    for name, shape, s in CONV_LAYERS:
        co, ci = shape[3], shape[4]
        n_in = side[ci]
        n_out = n_in * s
        x = torch.randn(B, n_in, n_in, n_in, ci, device="cuda")
        g = torch.randn(B, n_out, n_out, n_out, co, device="cuda")
        w = torch.from_numpy(Wd[name + "_weights"]).cuda()
        b = torch.from_numpy(Wd[name + "_biases"]).cuda()
        act = "sigmoid" if name == "g_conv5" else "elu"
        mac = B * n_out ** 3 * co * ci * 64 / (s ** 3)          # stride 2: each output sums 8 of the 64 taps
        t_f = timed(lambda: ops.conv3d_f32(x, w, b, s, True, act), args.reps * 4)
        t_b = timed(lambda: ops.conv3d_f32(g, w, None, s, False), args.reps * 4)
        tot[0] += t_f
        tot[1] += t_b
        for what, t in (("forward", t_f), ("data gradient", t_b)):
            rate = 2 * mac / (t * 1e-3)
            print(f"  {name} {what}: {t:.3f} ms, {mac / 1e6:.0f} MMAC, {rate / 1e9:.0f} GFLOP/s = {100 * rate / FP32_PEAK:.1f} % of "
                  f"the 67 TFLOP/s fp32 data-sheet rate", flush=True)
    print(f"  conv layers alone: forward {tot[0]:.3f} ms, data gradients {tot[1]:.3f} ms", flush=True)


if __name__ == "__main__":
    main()
