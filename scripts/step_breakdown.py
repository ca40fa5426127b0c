#!/usr/bin/env python
"""Where the flagship step's GPU time goes: one eager (non-graph) B = 24 render step per precision under torch.profiler
(CUDA activities), in a process of its own, after warm-up steps.  Writes per-kernel-name totals (ms, launches, share of
the step's kernel time) to OUT/step_breakdown_<precision>.csv and prints the top entries.
  python scripts/step_breakdown.py --out /tmp/step_breakdown"""
import argparse
import collections
import os
import sys

import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from rendernet_b200.engine import RenderEngine  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--batch", type=int, default=24)
    ap.add_argument("--top", type=int, default=12)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "step_breakdown.py profiles on the GPU"
    os.makedirs(args.out, exist_ok=True)
    B = args.batch
    rng = np.random.default_rng(0)
    vox = (rng.random((B, 64, 64, 64, 1)) < 0.10).astype(np.float32)
    pose = np.stack([rng.uniform(0, 2 * np.pi, B), (90 - rng.uniform(10, 170, B)) * np.pi / 180,
                     3.3 / rng.uniform(2.5, 4.5, B)], 1).astype(np.float32)
    for prec in ("exact", "fast"):
        eng = RenderEngine(None, B, use_graph=False, seed=0, precision=prec)
        eng.upload(vox, pose)
        for _ in range(3):
            eng.step_device()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            eng.step_device()
            torch.cuda.synchronize()
        tot = collections.defaultdict(float)
        cnt = collections.Counter()
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA:
                tot[ev.name] += ev.device_time_total / 1e3    # us -> ms
                cnt[ev.name] += 1
        step = sum(tot.values())
        rows = sorted(tot.items(), key=lambda kv: -kv[1])
        path = os.path.join(args.out, f"step_breakdown_{prec}.csv")
        with open(path, "w") as f:
            f.write("kernel,launches,ms,share\n")
            for name, ms in rows:
                f.write(f"\"{name}\",{cnt[name]},{ms:.4f},{ms / step:.4f}\n")
        print(f"[breakdown] {prec}: {step:.2f} ms of kernel time in {sum(cnt.values())} launches -> {path}")
        for name, ms in rows[:args.top]:
            print(f"[breakdown] {prec}   {ms:8.3f} ms {100 * ms / step:5.1f}%  x{cnt[name]:<3d} {name[:110]}")
        del eng
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
