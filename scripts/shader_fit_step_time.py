#!/usr/bin/env python
"""Cost of one Shader pose / light fit step on one GPU (the card's name, power limit and max SM clock are read in the same run).

1. ShaderPoseFit's gradient step at B = 5 (the search's five hypotheses, seeded weights, the chair at the search's first poses,
   objective "phong"), both precisions, split into the network forward (ShaderInputGradients.forward, tape recorded), the
   objective (rn_phong_composite_loss_grad) and the backward walk to dL/dpose (ShaderInputGradients.backward, which ends in a
   device synchronise and the host-side pose Jacobian).  Each part is bracketed by torch.cuda.synchronize() and timed with the
   host clock, after `--warmup` full steps; mean and spread over `--steps` steps.  The whole ShaderPoseFit.step is timed the
   same way.
2. rn_phong_composite_loss_grad alone at B = 24 (img + target in, d_img out), CUDA events around `--kernel-reps` launches, against
   its HBM floor: the bytes it must move, from the shapes, over the H100 SXM data sheet's 3.35 TB/s."""
import argparse
import math
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from rendernet_b200 import ops  # noqa: E402
from rendernet_b200.Reconstruct_RenderNet_Face import create_param_center  # noqa: E402
from rendernet_b200.shader_fit import ShaderPoseFit, light_dir  # noqa: E402

HBM = 3.35e12                # H100 SXM data sheet, HBM3 bytes/s


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                      # noqa: BLE001
        return f"{torch.cuda.get_device_name(0)} (nvidia-smi unavailable: {e})"


def chair():
    bv = np.load(os.path.join(ROOT, "tests", "golden", "binvox.npz"))
    return np.unpackbits(bv["chair_bits"]).reshape(64, 64, 64).astype(np.float32)


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, 1e3 * (time.perf_counter() - t0)


def fit_step(args, precision):
    fit = ShaderPoseFit(None, chair(), objective="phong", precision=precision)
    state = dict(pose=create_param_center(250, 60, 60, 30),
                 light=np.stack([np.linspace(230, 320, 5) * math.pi / 180, np.full(5, math.radians(60.0))], 1).astype(np.float32))
    target = torch.rand((5, 512, 512, 3), device="cuda", generator=torch.Generator("cuda").manual_seed(0))
    ld = torch.from_numpy(light_dir(state["light"])).cuda()
    for _ in range(args.warmup):
        fit.step(state, target)
    parts = {"forward": [], "objective": [], "backward": [], "step": []}
    for _ in range(args.steps):
        img, t = timed(lambda: fit.ig.forward(fit.voxels, state["pose"]))
        parts["forward"].append(t)
        (_, dimg, _), t = timed(lambda: ops.phong_composite_loss_grad(img, target, ld, (1.0, 1.0, 1.0), 0.1, 0.9))
        parts["objective"].append(t)
        _, t = timed(lambda: fit.ig.backward(dimg, want_dvox=False, want_dpose=True))
        parts["backward"].append(t)
        _, t = timed(lambda: fit.step(state, target))
        parts["step"].append(t)
    print(f"[{precision}] fit step B=5 ('phong'): " + ", ".join(
        f"{k} {np.mean(v):.2f} ms ({min(v):.2f}-{max(v):.2f})" for k, v in parts.items()), flush=True)
    del fit
    torch.cuda.empty_cache()


def kernel(args):
    B, H, W = 24, 512, 512
    g = torch.Generator(device="cuda").manual_seed(1)
    img = torch.rand((B, H, W, 3), device="cuda", generator=g)
    tgt = torch.rand((B, H, W, 3), device="cuda", generator=g)
    ld = torch.randn((B, 3), device="cuda", generator=g)
    lc = torch.ones((B, 3), device="cuda")
    loss = torch.zeros(B, device="cuda", dtype=torch.float64)
    dimg = torch.empty_like(img)
    dl = torch.zeros((B, 3), device="cuda")
    from rendernet_b200._lib import lib

    def launch():
        lib.rn_phong_composite_loss_grad(img.data_ptr(), tgt.data_ptr(), ld.data_ptr(), lc.data_ptr(), 0.1, 0.9, 0, 1,
                                         loss.data_ptr(), dimg.data_ptr(), dl.data_ptr(), B, H, W,
                                         torch.cuda.current_stream().cuda_stream)
    for _ in range(10):
        launch()
    e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
    e0.record()
    for _ in range(args.kernel_reps):
        launch()
    e1.record()
    e1.synchronize()
    us = 1e3 * e0.elapsed_time(e1) / args.kernel_reps
    nbytes = 3 * img.numel() * 4                        # img and target read, d_img written
    floor = 1e6 * nbytes / HBM
    print(f"rn_phong_composite_loss_grad B=24 512^2: {us:.1f} us for {nbytes / 1e6:.0f} MB, HBM floor {floor:.1f} us "
          f"({floor / us * 100:.0f} % of it, {nbytes / us / 1e6:.2f} TB/s)", flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--kernel-reps", type=int, default=200)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("shader_fit_step_time.py measures on a GPU; none found")
    print("card:", card(), flush=True)
    kernel(args)
    for precision in ("exact", "fast"):
        fit_step(args, precision)


if __name__ == "__main__":
    main()
