#!/usr/bin/env python
"""Cost of shading the Texture+Normal render on one GPU (the card's name, power limit and max SM clock are read in the same run).

1. TextureRenderEngine at B = 24 on the bench's inputs (seeded weights), both precisions: the unshaded step, the step with
   phong (composite "tf") and with phong (composite "numpy"), each one CUDA-graph replay.  The three engines live side by side
   and are timed in alternation, CUDA events around `--block` replays, `--rounds` rounds after warm-up; the mean per replay is
   reported (rounds x block >= 20 replays each).
2. rn_phong_shade alone at B = 24 (normal + albedo in, compos fp32 + uint8 out, as in the engine; and the shading alone), CUDA
   events around `--kernel-reps` launches, against the HBM floor: the bytes the kernel must move, computed from the shapes, over
   the H100 SXM data sheet's 3.35 TB/s.
3. FaceReconstruction.render at B = 5 (shape decoder, Texture+Normal forward, shading, download), exact precision."""
import argparse
import math
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from rendernet_b200._lib import RN_PHONG_NUMPY, RN_PHONG_TF, lib  # noqa: E402
from rendernet_b200.engine import TextureRenderEngine  # noqa: E402
from rendernet_b200.Reconstruct_RenderNet_Face import (FaceReconstruction, create_param_center,  # noqa: E402
                                                        pretrained_dict_from_texture_weights)
from oracle import rendernet_oracle as orc  # noqa: E402  (seeded weights only)
from oracle.shape_decoder import init_shape_decoder_weights  # noqa: E402

HBM = 3.35e12                # H100 SXM data sheet, HBM3 bytes/s
PHONG = dict(light_dir=np.array([[0.4, 0.5, 0.77]], np.float32))


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                      # noqa: BLE001
        return f"{torch.cuda.get_device_name(0)} (nvidia-smi unavailable: {e})"


def events_ms(fn, n):
    e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / n


def engines(args, precision):
    vox, poses = bench.synthetic_batch(24)
    tex = bench.synthetic_texture(24)
    engs = {"unshaded": TextureRenderEngine(None, 24, precision=precision),
            "tf": TextureRenderEngine(None, 24, precision=precision, phong=dict(PHONG, composite="tf")),
            "numpy": TextureRenderEngine(None, 24, precision=precision, phong=dict(PHONG, composite="numpy"))}
    for e in engs.values():
        e.upload(vox, tex, poses)
        for _ in range(3):
            e.step_device()
    torch.cuda.synchronize()
    times = {k: [] for k in engs}
    for _ in range(args.rounds):
        for k, e in engs.items():
            times[k].append(events_ms(e.graph.replay, args.block))
    base = float(np.mean(times["unshaded"]))
    for k, t in times.items():
        m = float(np.mean(t))
        print(f"[{precision}] B=24 {k:8s}: {m:.3f} ms per replay ({24e3 / m:.0f} renders/s), spread {min(t):.3f}-{max(t):.3f} ms, "
              f"{engs[k].launches_per_step} launches; vs unshaded {100 * (m / base - 1):+.2f} %", flush=True)
    del engs
    torch.cuda.empty_cache()


def kernel(args):
    B, H, W = 24, 512, 512
    g = torch.Generator(device="cuda").manual_seed(0)
    normal = torch.rand((B, H, W, 3), device="cuda", generator=g)
    albedo = torch.rand((B, H, W, 3), device="cuda", generator=g)
    ld = torch.tensor(PHONG["light_dir"], device="cuda").expand(B, 3).contiguous()
    lc = torch.ones((B, 3), device="cuda")
    f32 = torch.empty_like(normal)
    u8 = torch.empty(normal.shape, device="cuda", dtype=torch.uint8)
    px = B * H * W * 3
    st = torch.cuda.current_stream().cuda_stream
    cases = [("tf, albedo -> compos f32 + u8", RN_PHONG_TF, albedo, None, f32, u8, px * (4 + 4 + 4 + 1)),
             ("numpy, albedo -> compos f32 + u8", RN_PHONG_NUMPY, albedo, None, f32, u8, px * (4 + 4 + 4 + 1)),
             ("tf, shading f32 only", RN_PHONG_TF, None, f32, None, None, px * (4 + 4))]
    for name, comp, alb, sh, co, c8, nbytes in cases:
        def call():
            rc = lib.rn_phong_shade(normal.data_ptr(), None if alb is None else alb.data_ptr(), ld.data_ptr(), lc.data_ptr(), 0.0,
                                    1.0, comp, 1, 1, None if sh is None else sh.data_ptr(), None if co is None else co.data_ptr(),
                                    None if c8 is None else c8.data_ptr(), B, H, W, st)
            assert rc == 0, rc
        for _ in range(5):
            call()
        torch.cuda.synchronize()
        t = min(events_ms(call, args.kernel_reps) for _ in range(3))
        floor = nbytes / HBM * 1e3
        print(f"rn_phong_shade B=24 {name}: {t * 1e3:.1f} us, {nbytes / 1e6:.0f} MB -> {nbytes / (t * 1e-3) / 1e12:.2f} TB/s; "
              f"HBM floor {floor * 1e3:.1f} us at 3.35 TB/s ({t / floor:.2f}x the floor)", flush=True)


def face(args):
    B = 5
    W = orc.init_texture_weights(seed=1, alpha_range=(-0.3, 0.3), bias_jitter=0.02)
    for k in list(W):
        if k.endswith("/alpha") and "/res" in k:
            W[k] = np.zeros_like(W[k])
    rec = FaceReconstruction(pretrained_dict_from_texture_weights(W), init_shape_decoder_weights(2), batch=B)
    rng = np.random.default_rng(3)
    state = dict(latent=(0.5 + 0.3 * rng.standard_normal((B, 200))).astype(np.float32), pose=create_param_center(270, 60, 90, 30),
                 texture=rng.standard_normal((B, 199)).astype(np.float32),
                 light=(np.linspace(230, 320, 5).reshape(B, 1) * math.pi / 180).astype(np.float32))
    for _ in range(2):
        rec.render(state)
    torch.cuda.synchronize()
    t = events_ms(lambda: rec.render(state), args.reps)
    print(f"FaceReconstruction.render B=5 exact: {t:.2f} ms (shape decoder, Texture+Normal forward, shading, NumPy download)",
          flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--block", type=int, default=3)
    ap.add_argument("--kernel-reps", type=int, default=200)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("face_render_time.py measures on a CUDA device; none is available")
    print(f"card: {card()}", flush=True)
    kernel(args)
    for precision in ("fast", "exact"):
        engines(args, precision)
    face(args)
    kernel(args)


if __name__ == "__main__":
    main()
