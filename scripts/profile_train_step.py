#!/usr/bin/env python
"""One training step (rendernet_b200.training.ShaderTrainer, B = 1) bracketed by cudaProfilerStart/Stop, for ncu:
  ncu --profile-from-start off --metrics gpu__time_duration.sum --clock-control none --csv \
      --log-file out/launches_train.csv python scripts/profile_train_step.py --precision exact
  ncu --profile-from-start off --set full --clock-control none --import-source on -k regex:wgrad -c 2 \
      -o out/prof_wgrad python scripts/profile_train_step.py"""
import argparse
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from rendernet_b200.training import ShaderTrainer  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--precision", default="exact", choices=["exact", "fast"])
ap.add_argument("--keep-prob", type=float, default=0.75)
args = ap.parse_args()
rng = np.random.default_rng(0)
vox = (rng.random((1, 64, 64, 64, 1)) < 0.1).astype(np.float32)
vox[:, 16:48, 16:48, 16:48] = 1.0
poses = np.array([[4.36, 1.05, 3.3]], np.float32)
target = rng.random((1, 512, 512, 3)).astype(np.float32)
tr = ShaderTrainer(None, 1, precision=args.precision, keep_prob=args.keep_prob, seed=1)
tr.step(vox, poses, target)
tr.step(vox, poses, target)
torch.cuda.synchronize()
torch.cuda.profiler.start()
tr.step(vox, poses, target)
torch.cuda.synchronize()
torch.cuda.profiler.stop()
print("done")
