#!/usr/bin/env python
"""Time one res1 convolution (3^3, 32 -> 32, B = 24, 64 x 64 x 32) through the banded and the depth-sliced kernels,
alternated in one process: both precisions, both epilogues (PReLU; none + residual), three rounds of >= 20 launches each,
CUDA events.  Prints ms/launch, algorithmic TFLOP/s and its share of the H100 SXM data sheet's 989 dense fp16 TFLOP/s, and
the L2 -> shared and shared -> tensor-core operand bytes each kernel moves, computed from the shapes.
  python scripts/res1_time.py [--launches 20] [--rounds 3]"""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from rendernet_b200 import ops  # noqa: E402

PEAK_TFLOPS = 989.0
B, H, W, D, C = 24, 64, 64, 32, 32


def bytes_moved(passes):
    """(L2 -> shared, shared -> tensor-core operand reads) per launch, from the tile schedules."""
    tiles_b = B * H * W // 128 * (D * C // 128)                 # banded: 128 pixels x 4 depths
    # banded group = one (kx, K block): a 16 x 10-pixel halo of 64 channels + three 128 x 64 weight tiles
    l2_b = tiles_b * passes * 3 * 3 * (16 * 10 * 128 + 3 * 128 * 128)
    # per warpgroup and tap, 4 k16 steps of: one full K block (2 x m64n64: A 2 KB + B 2 KB each) + two half blocks (1 each)
    ops_b = tiles_b * 2 * passes * 9 * 4 * (2 + 1 + 1) * (2048 + 2048)
    tiles_s = B * (H // 8) * (W // 8) * (D // 8)                # sliced: 8 x 8 pixels x 8 depths
    l2_s = tiles_s * passes * 3 * 5 * (8 * 10 * 128) + 132 * (2 if passes == 3 else 1) * 9 * 96 * 64
    # 24 (input depth, output depth) pairs per tile and tap, two m64n32k16 each (A 2 KB + B 1 KB)
    ops_s = tiles_s * passes * 9 * 24 * 2 * (2048 + 1024)
    return (l2_b, ops_b), (l2_s, ops_s)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "res1_time.py measures on the GPU"
    p = torch.cuda.get_device_properties(0)
    print(f"[res1] device {p.name}, {p.multi_processor_count} SMs")
    rng = np.random.default_rng(0)
    x = torch.from_numpy(rng.standard_normal((B, H, W, D, C)).astype(np.float32)).cuda()
    res = torch.from_numpy(rng.standard_normal((B, H, W, D, C)).astype(np.float32)).cuda()
    w = torch.from_numpy((rng.uniform(-1, 1, (3, 3, 3, C, C)) * 0.06).astype(np.float32))
    b = torch.from_numpy(rng.uniform(-0.1, 0.1, C).astype(np.float32))
    alpha = torch.from_numpy(rng.uniform(0.05, 0.3, C).astype(np.float32)).cuda()
    macs = B * H * W * D * C * C * 27
    for prec, fmt in (("exact", 2), ("fast", 0)):
        passes = 3 if fmt == 2 else 1
        xs, rs = ops.cast_to_16(x, fmt=fmt), ops.cast_to_16(res, fmt=fmt)
        kern = {"banded": (ops.BandedConv3d(w, b, fmt=fmt), ops.conv3d_banded),
                "sliced": (ops.SlicedConv3d(w, b, fmt=fmt), ops.conv3d_sliced)}
        (l2_b, op_b), (l2_s, op_s) = bytes_moved(passes)
        print(f"[res1] {prec}: per launch L2->smem banded {l2_b / 1e9:.2f} GB, sliced {l2_s / 1e9:.2f} GB; "
              f"smem operand reads banded {op_b / 1e9:.2f} GB, sliced {op_s / 1e9:.2f} GB")
        for epi in ("prelu", "none+res"):
            def call(name):
                L, fn = kern[name]
                if epi == "prelu":
                    return fn(xs, L, act="prelu", alpha=alpha, alpha_tag="a")
                return fn(xs, L, act=None, residual=rs)
            times = {k: [] for k in kern}
            for name in kern:                                  # warm-up (module load, per-depth vectors)
                for _ in range(3):
                    call(name)
            torch.cuda.synchronize()
            for _ in range(args.rounds):
                for name in kern:
                    e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
                    e0.record()
                    for _ in range(args.launches):
                        call(name)
                    e1.record()
                    e1.synchronize()
                    times[name].append(e0.elapsed_time(e1) / args.launches)
            for name, t in times.items():
                ms = float(np.median(t))
                tf = 2.0 * macs * passes / (ms * 1e-3) / 1e12
                print(f"[res1] {prec:5s} {epi:8s} {name}: {ms:.3f} ms/launch (rounds {', '.join(f'{v:.3f}' for v in t)}), "
                      f"{tf:.0f} TFLOP/s = {100 * tf / PEAK_TFLOPS:.0f}% of 989")
            print(f"[res1] {prec:5s} {epi:8s} speed-up sliced vs banded: "
                  f"{np.median(times['banded']) / np.median(times['sliced']):.2f}x", flush=True)


if __name__ == "__main__":
    main()
