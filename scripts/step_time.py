#!/usr/bin/env python
"""Whole-step time (CUDA-graph replay, B = 24) of ONE build/configuration, long enough (>= 2 s) for the power
governor to settle.  Run it alternately for the builds/configurations to compare on one box:
  RENDERNET_B200_LIB=ab/librn_v2.so python scripts/step_time.py --tag v2
  RN_TUNE=msub=1 python scripts/step_time.py --tag msub1 --precision fast
(RN_TUNE is read once by the library at first use: the launch-heuristic defaults of one process, see include/rendernet_b200.h)"""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from rendernet_b200 import layer_util  # noqa: E402
from rendernet_b200.engine import RenderEngine  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--tag", default="default")
ap.add_argument("--chunks", type=int, default=5)
ap.add_argument("--precision", default="exact", choices=["exact", "fast"])
args = ap.parse_args()
if os.environ.get("RN_UNFUSED"):
    layer_util.USE_FUSED_RESAMPLE_CONV1 = False
B = 24
rng = np.random.default_rng(0)
vox = (rng.random((B, 64, 64, 64, 1)) < 0.10).astype(np.float32)
pose = np.stack([rng.uniform(0, 2 * np.pi, B), (90 - rng.uniform(10, 170, B)) * np.pi / 180,
                 3.3 / rng.uniform(2.5, 4.5, B)], 1).astype(np.float32)
eng = RenderEngine(None, B, seed=0, precision=args.precision)
eng.upload(vox, pose, non_blocking=False)
for _ in range(20):
    eng.step_device()
torch.cuda.synchronize()
ms = []
for _ in range(args.chunks):
    e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
    e0.record()
    for _ in range(10):
        eng.step_device()
    e1.record()
    torch.cuda.synchronize()
    ms.append(e0.elapsed_time(e1) / 10)
med = sorted(ms)[len(ms) // 2]
print(f"[step_time] {args.tag} [{args.precision}] RN_TUNE={os.environ.get('RN_TUNE', '')}: median {med:.2f} ms/step ({B / med * 1e3:.1f} renders/s); chunks " +
      " ".join(f"{m:.2f}" for m in ms) + f"; launches {eng.launches_per_step}; checksum {float(eng.out.double().sum()):.6f}",
      flush=True)
