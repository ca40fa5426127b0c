#!/usr/bin/env python
"""Timing of the wgmma weight-gradient kernel on the full-size trunk layer (3x3 1024->1024 @64x64, B=24): same algorithmic FLOPs
as the forward conv (1.855 TFLOP).  CUDA events on the launch stream, 10 back-to-back launches after 3 warm-ups."""
import os, sys
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from rendernet_b200 import ops  # noqa: E402

for fmt, name in ((0, "fast"), (2, "exact")):
    for (k, cin, cout) in ((3, 1024, 1024), (1, 1024, 1024), (3, 512, 512)):
        x = ops.cast_to_16(torch.randn(24, 64, 64, cin, device="cuda"), fmt=fmt)
        g = ops.cast_to_16(torch.randn(24, 64, 64, cout, device="cuda"), fmt=fmt)
        for _ in range(3):
            dw = ops.conv2d_weight_grad(x, g, k, k)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
        e0.record()
        for _ in range(10):
            dw = ops.conv2d_weight_grad(x, g, k, k)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 10
        fl = 2.0 * 24 * 64 * 64 * cin * cout * k * k
        print(f"[wgrad {name}] k{k} {cin}->{cout} @64^2 B=24: {ms:.3f} ms  {fl / ms / 1e9:.0f} TFLOP/s algorithmic"
              f" ({fl * (3 if fmt == 2 else 1) / ms / 1e9:.0f} issued)", flush=True)
        del x, g, dw
