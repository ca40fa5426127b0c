#!/usr/bin/env python
"""Time the exact-mode 3x3 C -> C trunk convolution at B = 24, 64 x 64 (res2: C = 1024, res3: C = 512) through the direct
igemm kernel and the Winograd F(2x2, 3x3) and F(4x4, 3x3) paths (rn_winograd.cu), alternated in one process: three rounds
of 20 launches each, CUDA events; then each Winograd stage of both tiles alone (input transform, the 16 or 36 per-position
GEMMs at the default and at two K blocks per pipeline stage, output transform).  Prints the card's name, power limit and
clocks, ms per launch, algorithmic TFLOP/s (2 * B*H*W * C * 9C per conv, the direct conv's MACs), issued TFLOP/s of the GEMM
stage (3 products per MAC), its time per 128 x 256 tile on one SM (tiles / SMs run one after another on each SM) and the
transforms' GB/s from the bytes they must move, as JSON on stdout and, with --out, to a file.
  python scripts/winograd_time.py [--launches 20] [--rounds 3] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from rendernet_b200 import ops  # noqa: E402
from rendernet_b200._lib import check, lib  # noqa: E402

B, H, W = 24, 64, 64


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"nvidia-smi unavailable: {e}"


def timed(fn, launches):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(launches):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / launches


def _stages(tile, L, x, y, C, launches, rounds):
    """Each stage of one Winograd tile alone, on a workspace of its own: ms per launch, the GEMM's issued TFLOP/s and time per
    128 x 256 tile on one SM (tiles / SMs run one after another on each SM), and the transforms' GB/s from the bytes they must
    move."""
    n = (tile + 2) ** 2                                 # positions of the tile
    U, s = ops.winograd_filter_exp(L, tile)
    sfx = "" if tile == 2 else "4"
    ws = torch.empty(getattr(lib, f"rn_winograd{sfx}_workspace_bytes")(B, H, W, C), device="cuda", dtype=torch.uint8)
    pos = B * (H // tile) * (W // tile) * C
    v = ws[:n * pos * 4]
    m = ws[n * pos * 4:].view(torch.float32)
    st = torch.cuda.current_stream().cuda_stream
    f_in, f_gemm = getattr(lib, f"rn_winograd{sfx}_in"), getattr(lib, f"rn_winograd{sfx}_gemm")
    out_args = (m.data_ptr(), L.bias.data_ptr(), L.alpha.data_ptr(), 1, None, 0, y.planes.data_ptr(), None, B, H, W, C)
    stages = {
        "in": lambda: check(f_in(x.data_ptr(), v.data_ptr(), B, H, W, C, st)),
        "gemm": lambda: check(f_gemm(v.data_ptr(), U.data_ptr(), m.data_ptr(), B, H, W, C, None, st)),
        "gemm_kps2": lambda: check(f_gemm(v.data_ptr(), U.data_ptr(), m.data_ptr(), B, H, W, C, ops._tune(dict(kps=2)), st)),
        "out": (lambda: check(lib.rn_winograd_out(*out_args, st))) if tile == 2 else
               (lambda: check(lib.rn_winograd4_out(*out_args, s, st))),
    }
    st_ms = {k: min(timed(fn, launches) for _ in range(rounds)) for k, fn in stages.items()}
    gemm_ms = min(st_ms["gemm"], st_ms["gemm_kps2"])
    tiles = n * pos // 128 // 256                       # 128-row x 256-column tiles of the one GEMM launch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    act_bytes = B * H * W * C * 4                       # one hi/lo activation (two fp16 planes)
    gbs = {"in": (act_bytes + n * pos * 4) / st_ms["in"] / 1e6,      # read x pair, write V pair
           "out": (n * pos * 4 + act_bytes) / st_ms["out"] / 1e6}    # read M fp32, write y pair (no residual here)
    return {"stage_ms": st_ms, "gemm_tflops_issued": 3 * 2.0 * n * pos * C / gemm_ms / 1e9, "gemm_tiles": tiles,
            "gemm_us_per_tile": gemm_ms * 1e3 / (tiles / sms), "transform_gbs": gbs}


def one_width(C, launches, rounds):
    g = torch.Generator().manual_seed(C)
    x = ops.cast_to_16(((torch.rand(B, H, W, C, generator=g) * 2 - 1) * 3).to("cuda"), fmt=2)
    w = (torch.rand(3, 3, C, C, generator=g) * 2 - 1) * (6.0 / (18 * C)) ** 0.5
    al = torch.rand(C, generator=g) * 0.3
    L = ops.pack_conv("conv2d", w, torch.zeros(C), al, device="cuda", fmt=2)
    y = ops.conv2d(x, L, act="prelu")
    tunes = {"direct": dict(winograd=-1), "winograd": dict(winograd=1, wino_tile=2), "winograd4": dict(winograd=1, wino_tile=4)}
    arms = {k: (lambda t=t: ops.conv2d(x, L, act="prelu", out16=y, tune=t)) for k, t in tunes.items()}
    times = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            times[k].append(timed(fn, launches))
    flop = 2.0 * B * H * W * C * 9 * C
    res = {"C": C}
    res.update({f"{k}_ms": v for k, v in times.items()})
    res.update({f"{k}_tflops_alg": flop / min(v) / 1e9 for k, v in times.items()})
    res["f2x2"] = _stages(2, L, x, y, C, launches, rounds)
    res["f4x4"] = _stages(4, L, x, y, C, launches, rounds)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", type=str, default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    out = {"card": card(), "widths": [one_width(C, a.launches, a.rounds) for C in (1024, 512)], "card_after": card()}
    print(json.dumps(out, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
