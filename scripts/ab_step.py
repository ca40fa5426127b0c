#!/usr/bin/env python
"""Same-box A/B of whole-step time (CUDA-graph replay, B = 24): runs scripts/step_time.py alternately for a list of
configurations (each in its own process: RN_TUNE / RENDERNET_B200_LIB are read once per process), three rounds interleaved.
Box-to-box variance of the pool is several percent, so optimisations are judged only by runs interleaved on one box.
  python scripts/ab_step.py "base|exact|" "msub1|exact|RN_TUNE=msub=1" "old|fast|RENDERNET_B200_LIB=ab/old.so"
Each argument is tag|precision|ENV=VALUE[,ENV=VALUE...]."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
specs = sys.argv[1:] or ["exact|exact|", "fast|fast|"]
for rnd in range(3):
    for spec in specs:
        tag, prec, envs = (spec.split("|") + ["", ""])[:3]
        env = dict(os.environ)
        for kv in filter(None, envs.split(";")):
            k, v = kv.split("=", 1)
            env[k] = v
        p = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "step_time.py"), "--tag", f"r{rnd}:{tag}", "--precision", prec,
                            "--chunks", "3"], env=env, capture_output=True, text=True)
        line = [ln for ln in p.stdout.splitlines() if ln.startswith("[step_time]")]
        print(line[0] if line else f"[ab] {tag}: FAILED rc={p.returncode} {p.stderr[-300:]}", flush=True)
