#!/usr/bin/env python
"""One eager (non-graph) forward step bracketed by cudaProfilerStart/Stop, for ncu:
  ncu --profile-from-start off --metrics gpu__time_duration.sum --clock-control none --csv \
      --log-file out/launches.csv python scripts/profile_step.py --batch 24
  ncu --profile-from-start off --set full --clock-control none --import-source on -k regex:igemm_kernel \
      -s 30 -c 2 -o out/prof python scripts/profile_step.py --batch 24"""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from rendernet_b200.engine import RenderEngine  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=24)
ap.add_argument("--steps", type=int, default=1)
ap.add_argument("--precision", default="exact", choices=["exact", "fast"])
args = ap.parse_args()
B = args.batch
eng = RenderEngine(None, B, use_graph=False, seed=0, precision=args.precision)
rng0, rng1 = np.random.default_rng(0), np.random.default_rng(1)
vox = (rng0.random((B, 64, 64, 64, 1)) < 0.10).astype(np.float32)
poses = np.stack([rng1.uniform(0, 2 * np.pi, B), (90 - rng1.uniform(10, 170, B)) * np.pi / 180,
                  3.3 / rng1.uniform(2.5, 4.5, B)], axis=1).astype(np.float32)
eng.upload(vox, poses)
eng.step_device()
torch.cuda.synchronize()
torch.cuda.profiler.start()
for _ in range(args.steps):
    eng.step_device()
torch.cuda.synchronize()
torch.cuda.profiler.stop()
print("done")
