#!/usr/bin/env python
"""Timing of the Texture+Normal input gradients (backward.TextureInputGradients): forward (tape recorded) and backward at B = 5
(the reference's reconstruction batch) and B = 24, both precisions, CUDA events, mean of 3 runs after one warm-up.

The backward is broken down by timing its pieces alone on the same shapes: the e_conv1 data gradient (-> dL/d(concat), fp32
[B,128^3,5]), rn_resample5_backward_f32, the texture decoder (three rn_conv3d_small data gradients, their PReLU derivatives and
the re-runs that give the pre-activations) and the FC data gradient; the trunk / head data gradients are the rest.  The
reconstruction objective (rn_phong_recon_loss_grad: Phong-shaded albedo vs a target, loss and image gradients) is timed on its own.  The
backward's figure includes the copy of the three gradients to the host and the float64 pose Jacobian.

Two weight sets: PReLU slopes >= 0, where the stored outputs tell each unit's side of the kink, and mixed-sign slopes (as
pretrained weights have), where the backward re-runs each PReLU layer (decoder layers included) without its activation to get
the pre-activation."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from rendernet_b200 import ops, tfcompat as tf  # noqa: E402
from rendernet_b200.backward import TextureInputGradients, _key  # noqa: E402
from rendernet_b200.engine import pose_to_matrix  # noqa: E402


def timed(fn, reps=3):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def weights(lo, seed=0):
    """Seeded Texture weights (TF variable names), PReLU slopes drawn from [lo, 0.3]."""
    tig = TextureInputGradients(None, 1, seed=seed)
    rng = np.random.default_rng(seed)
    with tf.use_store(tig.store):
        tig.forward(np.zeros((1, 64, 64, 64, 1), np.float32), np.zeros((1, 199), np.float32), np.zeros((1, 3), np.float32) + 1)
    W = {n: v.cpu().numpy() for n, v in tig.store.vars.items()}
    for n in W:
        if n.endswith("/alpha"):
            W[n] = rng.uniform(lo, 0.3, W[n].shape).astype(np.float32)
    return W


def main():
    for lo in (0.0, -0.3):
        run(weights(lo), "slopes >= 0" if lo == 0.0 else "mixed-sign slopes")


def run(W, label):
    rng = np.random.default_rng(1)
    for B in (5, 24):
        vox = ((rng.random((B, 64, 64, 64, 1)) < 0.25) * 0.9).astype(np.float32)
        z = rng.standard_normal((B, 199)).astype(np.float32)
        poses = np.stack([rng.uniform(0, 6.28, B), rng.uniform(0.3, 1.2, B), np.full(B, 3.3)], 1).astype(np.float32)
        Ga = rng.standard_normal((B, 512, 512, 3)).astype(np.float32)
        Gn = rng.standard_normal((B, 512, 512, 3)).astype(np.float32)
        for precision in ("fast", "exact"):
            tig = TextureInputGradients(W, B, precision=precision)
            t_fwd = timed(lambda: tig.forward(vox, z, poses))
            Ga_d, Gn_d = torch.from_numpy(Ga).cuda(), torch.from_numpy(Gn).cuda()
            t_bwd = timed(lambda: tig.backward(Ga_d, Gn_d))
            fmt = tig.store.fmt
            dev = tig.store.device
            rec = next(r for r in tig.tape if r["op"] == "resample5_conv1")
            g16 = ops.cast_to_16(torch.randn(B, 64, 64, 64, 8, device=dev), fmt=fmt)
            w32 = tig._w32(rec["w"])
            t_conv1 = timed(lambda: ops.conv3d_backward_data_direct(g16, w32, (B, 128, 128, 128, 5), (2, 2, 2), want32=True,
                                                                    out_scale=1.0 / tig.last_loss_scale))
            dgrid = torch.randn(B, 128, 128, 128, 5, device=dev)
            minv = torch.from_numpy(pose_to_matrix(poses, 64, 128)).to(dev)
            t_res = timed(lambda: ops.resample5_backward(tig.vox, tig.tex3d, minv, dgrid))
            G3 = torch.randn(B, 64, 64, 64, 4, device=dev)

            def decoder():
                with tf.use_store(tig.store):
                    tig._reverse_walk({_key(tig.tex3d): G3}, False, True)
            t_dec = timed(decoder)
            fc = next(r for r in tig.tape if r["op"] == "fc")
            gfc = torch.randn(B, int(fc["y"].shape[1]), device=dev)
            wfc = tig._w32(fc["w"])
            t_fc = timed(lambda: ops.fully_connected_backward_data(gfc, wfc))
            ones = torch.ones(B, 3, device=dev)
            tgt = torch.rand(B, 512, 512, 3, device=dev)
            t_phong = timed(lambda: ops.phong_recon_loss_grad(tig.albedo, tig.normal, tgt, ones, ones))
            t_trunk = t_bwd - t_conv1 - t_res - t_dec
            print(f"[texture grad {precision}, {label}] B={B}: forward {t_fwd:.2f} ms, backward {t_bwd:.2f} ms ({t_bwd / t_fwd:.2f}x): "
                  f"trunk/heads {t_trunk:.2f}, e_conv1 dgrad {t_conv1:.2f}, resample5_backward {t_res:.2f}, "
                  f"decoder {t_dec - t_fc:.2f} + FC backward {t_fc:.3f} ms; Phong loss + gradient {t_phong:.3f} ms", flush=True)
            del tig
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
