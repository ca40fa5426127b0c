#!/usr/bin/env python
"""Cost of fine-tuning the face-reconstruction shape decoder on one GPU (the card's name, power limit and max SM clock are read
in the same run).

At B = 5 (the reconstruction's batch) and B = 32, seeded weights and operands, CUDA events around each call, the variants
alternated in one process over `--rounds` rounds of `--reps` calls each (after one warm-up call of each):
  * each layer's weight-gradient launch alone: rn_conv3d_f32_weight_grad of g_conv1 .. g_conv5 (the GEMM / direct kernel and the
    fixed-order reduction), and rn_fully_connected_param_grad of g_gc1 without activation;
  * the latent-only decoder walk: ShapeDecoderGradients.backward(G, on_device=True);
  * the walk with weight gradients: backward(G, on_device=True, want_weight_grads=True).
Each line gives the median ms, and for the kernels the achieved GFLOP/s (2 x the layer's MACs over the median time) and its share
of the H100 SXM data sheet's 67 TFLOP/s fp32 peak (the peak of a card allowed 700 W)."""
import argparse
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.shape_decoder import CONV_LAYERS, init_shape_decoder_weights  # noqa: E402
from rendernet_b200 import ops  # noqa: E402
from rendernet_b200.backward import ShapeDecoderGradients  # noqa: E402

FP32_PEAK = 67e12            # H100 SXM data sheet, dense fp32 FLOP/s


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                      # noqa: BLE001
        return f"{torch.cuda.get_device_name(0)} (nvidia-smi unavailable: {e})"


def event_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def alternate(variants, rounds, reps):
    """{name: [ms per call]}: every variant once to warm up, then `rounds` rounds of `reps` calls of each, in turn."""
    for fn in variants.values():
        fn()
    torch.cuda.synchronize()
    out = {k: [] for k in variants}
    for _ in range(rounds):
        for k, fn in variants.items():
            out[k].append(event_ms(lambda: [fn() for _ in range(reps)]) / reps)
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--batches", type=int, nargs="+", default=[5, 32])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("shape_decoder_wgrad_time: needs a CUDA device")
    print(f"[shape_decoder_wgrad_time] card: {card()}")
    W = init_shape_decoder_weights(seed=5)
    for B in a.batches:
        g = torch.Generator(device="cuda").manual_seed(B)
        variants, flops = {}, {}
        for name, shape, s in CONV_LAYERS:
            side = {256: 4, 128: 8, 64: 16, 32: 32, 16: 64}[shape[4]]
            x = torch.randn((B, side, side, side, shape[4]), device="cuda", generator=g)
            gz = torch.randn((B, side * s, side * s, side * s, shape[3]), device="cuda", generator=g)
            variants[name] = (lambda x=x, gz=gz, s=s: ops.conv3d_f32_weight_grad(x, gz, s, True))
            flops[name] = 2.0 * 64 * shape[3] * shape[4] * B * side ** 3        # every tap meets every input voxel once
        xf = torch.randn((B, 200), device="cuda", generator=g)
        gf = torch.randn((B, 16384), device="cuda", generator=g)
        variants["g_gc1"] = lambda: ops.fully_connected_param_grad(xf, gf, None, None)
        flops["g_gc1"] = 2.0 * B * 200 * 16384
        sdg = ShapeDecoderGradients(W, B)
        sdg.forward(np.random.default_rng(B).standard_normal((B, 200)).astype(np.float32))
        G = torch.randn((B, 64, 64, 64, 1), device="cuda", generator=g)
        variants["walk: latent only"] = lambda: sdg.backward(G, on_device=True)
        variants["walk: + weight gradients"] = lambda: sdg.backward(G, on_device=True, want_weight_grads=True)
        res = alternate(variants, a.rounds, a.reps)
        med = {k: float(np.median(v)) for k, v in res.items()}
        for k, v in res.items():
            line = f"B={B:2d} {k:26s} {med[k]:8.3f} ms (min {min(v):.3f}, max {max(v):.3f})"
            if k in flops:
                r = flops[k] / (med[k] * 1e-3)
                line += f"  {r / 1e9:8.0f} GFLOP/s = {100 * r / FP32_PEAK:5.1f} % of the 67 TFLOP/s fp32 peak"
            print(line)
        conv = sum(med[n] for n, _, _ in CONV_LAYERS)
        print(f"B={B:2d} five conv weight gradients together: {conv:.3f} ms; the walk's weight-gradient part "
              f"{med['walk: + weight gradients'] - med['walk: latent only']:.3f} ms")
        del sdg
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
