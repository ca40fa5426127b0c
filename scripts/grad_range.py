#!/usr/bin/env python
"""Where the 16-bit gradients of the backward walk land in fp16's range (DESIGN §4).

For every record of the tape that the walk differentiates (ShaderInputGradients / TextureInputGradients._data_grad_of, i.e.
each 16-bit dL/d(pre-activation) after the PReLU or sigmoid step) it prints the largest |g| and, over the nonzero elements,
the fraction whose HI half is an fp16 subnormal (|hi| < 2^-14: fewer bits in both precisions) and the fraction below 2^-3
(the exact mode's LO half is subnormal there: fewer than 21 bits).  The gradients carry the loss scale, so "growth" is the
largest interior |g| over the largest |g| at the output heads: the headroom LOSS_SCALE_TARGET has to leave.

Cases: white noise G ~ N(0, 1) per pixel (the whole-network tests), the Shader MSE gradient at B = 1 and the same divided by
24 (exactly the per-pixel magnitude at B = 24), the training walk (B = 2, dropout 0.75, weight gradients), the reconstruction objective at a random start and near convergence (target
rendered from the state itself plus noise of 0.01, loss ~1e-4); each with the old fixed scale 4096 and the adaptive one.
Seeded random weights (the test suite's): trained weights may grow gradients differently."""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from rendernet_b200 import ops  # noqa: E402
from rendernet_b200.backward import LOSS_SCALE_TARGET, OVERFLOW_RETRIES, ShaderInputGradients, TextureInputGradients  # noqa: E402
from rendernet_b200.training import ShaderTrainer  # noqa: E402
from rendernet_b200.Reconstruct_RenderNet_Face import light_pos  # noqa: E402
from oracle import phong_tf as pt  # noqa: E402
from oracle import rendernet_oracle as orc  # noqa: E402

SUB, SMALL = 2.0 ** -14, 2.0 ** -3


def stats(g):
    """(amax, fraction of nonzero elements with a subnormal HI half, fraction of nonzero elements below 2^-3)."""
    if isinstance(g, ops.Split16):
        hi, v = g.planes[0].float(), g.float()
    else:
        hi = v = g.float()
    nz = v != 0
    n = max(int(nz.sum().item()), 1)
    a = v.abs()
    return (float(a.max().item()), int((nz & (hi.abs() < SUB)).sum().item()) / n, int((nz & (a < SMALL)).sum().item()) / n)


def walk_stats(ig, run):
    """Run `run()` (one backward) with _data_grad_of wrapped; -> [(layer name, amax, frac subnormal HI, frac < 2^-3, is a
    sigmoid output head)]."""
    rows = []
    orig = ig._data_grad_of

    def wrapped(rec, g, acc=None):
        rows.append((rec["w"]._rn_name.rsplit("/", 1)[0],) + stats(g) + (rec.get("act") == "sigmoid",))
        return orig(rec, g, acc)
    ig._data_grad_of = wrapped
    try:
        run()
    finally:
        del ig._data_grad_of
    return rows


def input_chain_stats(ig):
    """stats of the gradient e_conv1 receives (the fused input record is not a _data_grad_of call)."""
    seen = []
    orig = ig._input_chain

    def wrapped(rec, g, grads):
        seen.append(stats(g))
        return orig(rec, g, grads)
    ig._input_chain = wrapped
    return seen


def report(label, rows, first, scale):
    out_amax = max(r[1] for r in rows if r[4])
    worst = max((r for r in rows if not r[4]), key=lambda r: r[1])
    all_rows = rows + [("e_conv1",) + first[0] + (False,)] if first else rows
    sub = max(r[2] for r in all_rows)
    small = max(r[3] for r in all_rows)
    print(f"{label}: loss scale {scale:g}; output amax {out_amax:.3e}, largest interior amax {worst[1]:.3e} at {worst[0]} "
          f"(growth {worst[1] / out_amax:.2f}); worst layer: {100 * sub:.1f} % of nonzero elements with a subnormal HI, "
          f"{100 * small:.1f} % below 2^-3", flush=True)
    return worst[1] / out_amax


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", action="store_true", help="print every layer of the adaptive white-noise walks")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("grad_range.py runs the backward pass on a CUDA device; none is available")
    golden = os.path.join(ROOT, "tests", "golden")
    bv = np.load(os.path.join(golden, "binvox.npz"))
    chair = np.unpackbits(bv["chair_bits"]).reshape(1, 64, 64, 64, 1).astype(np.float32)
    vox = chair * 0.75 + 0.125 * (np.random.default_rng(2).random(chair.shape) < 0.02)
    poses = orc.compute_pose_param(250.0, 60.0, 3.3).astype(np.float32)
    Ws = orc.init_shader_weights(seed=1, alpha_range=(0.05, 0.3), bias_jitter=0.02)
    growth = []
    for precision in ("exact", "fast"):
        for mode in (4096.0, None):
            ig = ShaderInputGradients(Ws, 1, precision=precision, loss_scale=mode)
            img = ig.forward(vox, poses)
            G = torch.from_numpy(np.random.default_rng(5).standard_normal((1, 512, 512, 3)).astype(np.float32)).cuda()
            target = img.detach().clone()
            target += 0.3 * torch.from_numpy(np.random.default_rng(6).standard_normal((1, 512, 512, 3)).astype(np.float32)).cuda()
            _, dmse = ops.image_loss_grad(img.contiguous(), target.clamp(0, 1).contiguous(), "mse")
            for name, d in (("N(0,1)", G), ("MSE B=1", dmse), ("MSE B=1 / 24", dmse / 24.0)):
                first = input_chain_stats(ig)
                rows = walk_stats(ig, lambda: ig.backward(d, want_dpose=False))
                del ig._input_chain
                tag = "fixed 4096" if mode else "adaptive"
                growth.append(report(f"[shader {precision}, {tag}] {name}", rows, first, ig.last_loss_scale))
                if args.layers and mode is None and name == "N(0,1)":
                    for r in rows:
                        print(f"    {r[0]}: amax {r[1]:.3e}, subnormal HI {100 * r[2]:.2f} %, < 2^-3 {100 * r[3]:.2f} %")
            del ig
            torch.cuda.empty_cache()

    # the training walk: dropout (1 / keep on the kept elements), PReLU on the recorded pre-activations, weight gradients
    for mode in (4096.0, None):
        tr = ShaderTrainer(Ws, 2, precision="exact", keep_prob=0.75, seed=3, loss_scale=mode)
        tr.overflow_retries = OVERFLOW_RETRIES
        v2, p2 = np.repeat(vox, 2, 0), np.concatenate([poses, orc.compute_pose_param(70.0, 60.0, 3.3).astype(np.float32)])
        img = tr.forward(v2, p2)
        tgt = (img + 0.3 * torch.randn(img.shape, device="cuda", generator=torch.Generator("cuda").manual_seed(1))).clamp(0, 1)
        _, dimg = ops.image_loss_grad(img.contiguous(), tgt.contiguous(), "mse")
        first = input_chain_stats(tr)
        rows = walk_stats(tr, lambda: tr.backward(dimg, want_dvox=False, want_dpose=False, want_weight_grads=True))
        del tr._input_chain
        growth.append(report(f"[trainer exact B=2 keep 0.75, {'fixed 4096' if mode else 'adaptive'}] MSE", rows, first,
                             tr.last_loss_scale))
        if args.layers and mode is None:
            for r in rows:
                print(f"    {r[0]}: amax {r[1]:.3e}, subnormal HI {100 * r[2]:.2f} %, < 2^-3 {100 * r[3]:.2f} %")
        del tr
        torch.cuda.empty_cache()

    B = 2
    W = orc.init_texture_weights(seed=21, alpha_range=(-0.3, 0.3), bias_jitter=0.02)
    rng = np.random.default_rng(22)
    tvox = ((rng.random((B, 64, 64, 64, 1)) < 0.25) * rng.uniform(0.5, 1.0, (B, 64, 64, 64, 1))).astype(np.float32)
    z = rng.standard_normal((B, 199)).astype(np.float32)
    tposes = np.concatenate([orc.compute_pose_param(45.0, 30.0, 2.5), orc.compute_pose_param(300.0, 20.0, 1.8)]).astype(np.float32)
    az, el = np.array([[0.4], [2.1]], np.float32), 0.7
    ldir = torch.from_numpy(light_pos(az, el)).cuda()
    ones = torch.ones(B, 3, device="cuda")
    for precision in ("exact", "fast"):
        for mode in (4096.0, None):
            tig = TextureInputGradients(W, B, precision=precision, loss_scale=mode)
            albedo, normal = tig.forward(tvox, z, tposes)
            shade = pt.tf_phong_composite(normal.double().cpu(), torch.from_numpy(light_pos(az, el)).double(),
                                          torch.ones(B, 3, dtype=torch.float64), 0.0, 1.0)
            near = (albedo.double().cpu() * shade).float().cuda()
            near += 0.01 * torch.from_numpy(np.random.default_rng(7).standard_normal((B, 512, 512, 3)).astype(np.float32)).cuda()
            rand = torch.from_numpy(np.random.default_rng(8).random((B, 512, 512, 3)).astype(np.float32)).cuda()
            for name, tgt in (("recon random start", rand), ("recon near convergence", near)):
                loss, da, dn, _ = ops.phong_recon_loss_grad(albedo, normal, tgt.contiguous(), ldir, ones, 0.0, 1.0,
                                                            black_background=False, with_mask=True)
                first = input_chain_stats(tig)
                rows = walk_stats(tig, lambda: tig.backward(da, dn))
                del tig._input_chain
                tag = "fixed 4096" if mode else "adaptive"
                growth.append(report(f"[texture {precision}, {tag}] {name} (loss {loss.mean().item():.1e})", rows, first,
                                     tig.last_loss_scale))
            del tig
            torch.cuda.empty_cache()
    print(f"largest interior growth over all cases {max(growth):.2f}; LOSS_SCALE_TARGET = 2^{np.log2(LOSS_SCALE_TARGET):.0f} "
          f"leaves {65504 / (LOSS_SCALE_TARGET * max(growth)):.1f}x headroom below 65504", flush=True)


if __name__ == "__main__":
    main()
