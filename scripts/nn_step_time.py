#!/usr/bin/env python
"""Cost of the autograd layers (rendernet_b200.nn) against the direct calls they wrap, on one GPU (the card's name, power limit
and max SM clock are read in the same run).

1. At B = 5 and 24, both precisions, seeded weights, the chair at random poses, CUDA events around each call, the variants
   alternated in one process over `--rounds` rounds of `--reps` calls each (after one warm-up call of each):
   * input gradients: ShaderRenderer forward + backward of (img * G).sum() to the voxels and the pose, against
     ShaderInputGradients.forward + backward(G, dvox_on_device=True);
   * parameter gradients: ShaderRenderer(trainable=True) forward + F.mse_loss(...).backward(), against
     ShaderTrainer(keep_prob=1).loss_and_gradients.
   The same kernels run in both, so the expected difference is within the run-to-run spread.
2. rn_phong_shade_backward alone at B = 24, 512 x 512 (TF composite with an albedo: normal, albedo and g_compos read, d_normal
   and d_albedo written, d_light reduced; and the NumPy composite without an albedo), CUDA events around `--kernel-reps`
   launches, against its HBM floor (the bytes it must move over the H100 SXM data sheet's 3.35 TB/s) and against the fused
   objective rn_phong_recon_loss_grad, which moves the same five arrays."""
import argparse
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from rendernet_b200.backward import ShaderInputGradients  # noqa: E402
from rendernet_b200.nn import ShaderRenderer  # noqa: E402
from rendernet_b200.training import ShaderTrainer  # noqa: E402

HBM = 3.35e12                # H100 SXM data sheet, HBM3 bytes/s


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                      # noqa: BLE001
        return f"{torch.cuda.get_device_name(0)} (nvidia-smi unavailable: {e})"


def chair(B):
    bv = np.load(os.path.join(ROOT, "tests", "golden", "binvox.npz"))
    v = np.unpackbits(bv["chair_bits"]).reshape(1, 64, 64, 64, 1).astype(np.float32)
    return np.ascontiguousarray(np.repeat(v, B, 0))


def event_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def alternate(variants, rounds, reps):
    """{name: [ms per call]}: every variant once to warm up, then `rounds` rounds of `reps` calls of each, in turn."""
    for fn in variants.values():
        fn()
    out = {k: [] for k in variants}
    for _ in range(rounds):
        for k, fn in variants.items():
            out[k] += [event_ms(fn) for _ in range(reps)]
    return out


def release(o):
    o.tape = o.img = o.vox = None


def step_times(args, precision, B):
    rng = np.random.default_rng(B)
    vox_np = chair(B)
    vp = np.stack([rng.uniform(3.5, 5.5, B), rng.uniform(0.2, 0.9, B), rng.uniform(3.0, 3.6, B)], 1).astype(np.float32)
    vox = torch.from_numpy(vox_np).cuda()
    G = torch.randn((B, 512, 512, 3), device="cuda", generator=torch.Generator("cuda").manual_seed(B))
    tgt = torch.rand((B, 512, 512, 3), device="cuda", generator=torch.Generator("cuda").manual_seed(B + 1))
    ig = ShaderInputGradients(None, B, precision=precision)
    m = ShaderRenderer(None, precision=precision)

    def direct():
        ig.forward(vox, vp)
        ig.backward(G, dvox_on_device=True)
        release(ig)

    def module():
        v = vox.clone().requires_grad_()
        p = torch.from_numpy(vp).requires_grad_()
        (m(v, p) * G).sum().backward()

    res = alternate({"direct": direct, "module": module}, args.rounds, args.reps)
    del ig, m
    torch.cuda.empty_cache()
    tr = ShaderTrainer(None, B, precision=precision, keep_prob=1.0)
    mt = ShaderRenderer(None, precision=precision, trainable=True)

    def trainer():
        tr.loss_and_gradients(vox_np, vp, tgt)
        release(tr)
        tr.weight_grads = None

    def trainable():
        mt.zero_grad(set_to_none=True)
        F.mse_loss(mt(vox, vp), tgt).backward()

    res.update(alternate({"trainer": trainer, "trainable": trainable}, args.rounds, args.reps))
    del tr, mt
    torch.cuda.empty_cache()
    med = {k: float(np.median(v)) for k, v in res.items()}
    spread = {k: float(np.max(v) - np.min(v)) for k, v in res.items()}
    print(f"[{precision}] B={B}: input gradients: module {med['module']:.1f} ms vs direct {med['direct']:.1f} ms "
          f"({100 * (med['module'] / med['direct'] - 1):+.1f} %; spread {spread['module']:.1f} / {spread['direct']:.1f} ms); "
          f"parameter gradients: module {med['trainable']:.1f} ms vs ShaderTrainer {med['trainer']:.1f} ms "
          f"({100 * (med['trainable'] / med['trainer'] - 1):+.1f} %; spread {spread['trainable']:.1f} / {spread['trainer']:.1f} ms)",
          flush=True)


def kernel_times(args):
    B, H, W = 24, 512, 512
    gen = torch.Generator("cuda").manual_seed(0)
    normal, albedo, g, tgt = (torch.rand((B, H, W, 3), device="cuda", generator=gen) for _ in range(4))
    ld = torch.randn((B, 3), device="cuda", generator=gen)
    lc = torch.ones((B, 3), device="cuda")
    dn, da = torch.empty_like(normal), torch.empty_like(normal)
    dl = torch.zeros((B, 3), device="cuda")
    loss = torch.zeros(B, device="cuda", dtype=torch.float64)
    from rendernet_b200._lib import RN_PHONG_NUMPY, RN_PHONG_TF, lib
    st = torch.cuda.current_stream().cuda_stream

    def bwd(comp, alb):
        return lambda: lib.rn_phong_shade_backward(normal.data_ptr(), None if alb is None else alb.data_ptr(), ld.data_ptr(),
                                                   lc.data_ptr(), 0.0, 1.0, comp, 1, 1, g.data_ptr(), dn.data_ptr(),
                                                   da.data_ptr(), dl.data_ptr(), B, H, W, st)

    fused = lambda: lib.rn_phong_recon_loss_grad(albedo.data_ptr(), normal.data_ptr(), tgt.data_ptr(), ld.data_ptr(),  # noqa: E731
                                                 lc.data_ptr(), 0.0, 1.0, 0, 1, loss.data_ptr(), da.data_ptr(), dn.data_ptr(),
                                                 dl.data_ptr(), B, H, W, st)
    arr = B * H * W * 3 * 4
    cases = (("rn_phong_shade_backward tf + albedo", bwd(RN_PHONG_TF, albedo), 5 * arr),
             ("rn_phong_shade_backward numpy, no albedo", bwd(RN_PHONG_NUMPY, None), 3 * arr),
             ("rn_phong_recon_loss_grad (fused)", fused, 5 * arr))
    for name, fn, nbytes in cases:
        for _ in range(5):
            fn()
        t = event_ms(lambda: [fn() for _ in range(args.kernel_reps)]) / args.kernel_reps * 1e3
        floor = nbytes / HBM * 1e6
        print(f"{name} B=24 512^2: {t:.1f} us for {nbytes / 1e6:.0f} MB, HBM floor {floor:.1f} us ({t / floor:.2f}x), "
              f"{nbytes / (t * 1e-6) / 1e12:.2f} TB/s", flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--kernel-reps", type=int, default=200)
    ap.add_argument("--batches", type=int, nargs="+", default=[5, 24])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("nn_step_time.py measures on a GPU: none found")
    print("card:", card(), flush=True)
    kernel_times(args)
    for precision in ("exact", "fast"):
        for B in args.batches:
            step_times(args, precision, B)


if __name__ == "__main__":
    main()
