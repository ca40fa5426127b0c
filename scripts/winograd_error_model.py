#!/usr/bin/env python
"""CPU emulation of the exact-mode Winograd trunk convolution against float64, for F(2x2, 3x3) and F(4x4, 3x3) (rn_winograd.cu).

It models what sets the error of the device path:
  * the hi/lo splits of x, V and U (hi = fp16(v), lo = fp16(v - hi), as cast_to_16(fmt=2) and the transform kernels split);
  * V = B^T d B in fp32 (F(4x4): times 1/2), U = G g G^T in float64 from the fp32 filter, rounded once (F(4x4): times 2^s);
  * the three pass-major products of the GEMM (x_lo.w_hi, x_hi.w_lo, then x_hi.w_hi) into the tensor core's fp32 accumulator,
    truncated toward zero after every k16 step;
  * the output transform in fp32.
It does not model the order of the fp32 additions inside the transform kernels (a few ulps of V and of y).
Prints, per variant, the largest error and the rms error as shares of the output scale, and max |V| / max |x|.
  python scripts/winograd_error_model.py [--cout 64] [--hw 16] [--scale 3] [--seed 0]"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

F2 = (np.array([[1, 0, -1, 0], [0, 1, 1, 0], [0, -1, 1, 0], [0, 1, 0, -1]], dtype=np.float64),
      np.array([[1, 0, 0], [0.5, 0.5, 0.5], [0.5, -0.5, 0.5], [0, 0, 1]], dtype=np.float64),
      np.array([[1, 1, 1, 0], [0, 1, -1, -1]], dtype=np.float64))


def split16(v):
    """fp32 -> (hi, lo) fp16 planes as float64: hi = fp16(v), lo = fp16(v - hi)."""
    v = np.asarray(v, dtype=np.float32)
    hi = v.astype(np.float16)
    lo = (v - hi.astype(np.float32)).astype(np.float16)
    return hi.astype(np.float64), lo.astype(np.float64)


def trunc32(v):
    """float64 -> the fp32 value next to it toward zero (the tensor core's accumulator rounding)."""
    r = v.astype(np.float32)
    over = np.abs(r.astype(np.float64)) > np.abs(v)
    r[over] = np.nextafter(r[over], np.float32(0))
    return r


def tc_gemm(v_hi, v_lo, u_hi, u_lo):
    """[P, R, K] x [P, N, K] -> [P, R, N] fp32: three passes over K in k16 steps, truncating after each step."""
    acc = np.zeros((v_hi.shape[0], v_hi.shape[1], u_hi.shape[1]), dtype=np.float32)
    for a, b in ((v_lo, u_hi), (v_hi, u_lo), (v_hi, u_hi)):
        for k in range(0, a.shape[2], 16):
            part = np.einsum("prk,pnk->prn", a[:, :, k:k + 16], b[:, :, k:k + 16])   # exact: 16 products of 22 bits
            acc = trunc32(acc.astype(np.float64) + part)
    return acc


def emulate(x, w, mats, m, v_half=False, u_exp_rule=None):
    """x [H, W, C] float64 (the hi + lo activation), w [3, 3, C, N] fp32 -> (y fp32 [H, W, N], max |V|)."""
    BT, G, AT = mats
    H, W, C = x.shape
    n = m + 2
    xp = np.pad(x, ((1, n - m - 1), (1, n - m - 1), (0, 0)))
    d = np.stack([np.stack([xp[m * ty:m * ty + n, m * tx:m * tx + n] for tx in range(W // m)]) for ty in range(H // m)])
    bt32 = BT.astype(np.float32)
    V = np.einsum("ai,yxijc,bj->abyxc", bt32, d.astype(np.float32), bt32)      # fp32 transform
    if v_half:
        V = V * np.float32(0.5)
    U = np.einsum("ak,klio,bl->aboi", G, w.astype(np.float64), G)            # float64, [n, n, N, C]
    s = u_exp_rule(float(np.abs(U).max())) if u_exp_rule else 0
    U = (U * 2.0 ** s).astype(np.float32)
    v_hi, v_lo = split16(V.reshape(n * n, -1, C))
    u_hi, u_lo = split16(U.reshape(n * n, -1, C))
    M = tc_gemm(v_hi, v_lo, u_hi, u_lo).reshape(n, n, H // m, W // m, -1)
    at32 = AT.astype(np.float32)
    y = np.einsum("ia,abyxo,jb->yixjo", at32, M, at32).reshape(H, W, -1)
    scale = 2.0 ** ((1 if v_half else 0) - s)
    return (y * np.float32(scale)).astype(np.float32), float(np.abs(V).max())


def direct(x, w):
    H, W, _ = x.shape
    xp = np.pad(x, ((1, 1), (1, 1), (0, 0)))
    ref = np.zeros((H, W, w.shape[3]))
    for ky in range(3):
        for kx in range(3):
            ref += np.einsum("hwi,io->hwo", xp[ky:ky + H, kx:kx + W], w[ky, kx].astype(np.float64))
    return ref


def inputs(hw=16, C=1024, cout=64, scale=3.0, seed=0, uniform=False):
    """The inputs of test_exact_trunk_conv_k9216_accumulation_error: x ~ scale N(0,1) (or U(-scale, scale)), split hi/lo;
    xavier-uniform weights."""
    rng = np.random.default_rng(seed)
    x = (rng.uniform(-1, 1, (hw, hw, C)) if uniform else rng.standard_normal((hw, hw, C))) * scale
    hi, lo = split16(x.astype(np.float32))
    lim = (6.0 / (9 * C + 9 * cout)) ** 0.5
    w = rng.uniform(-lim, lim, (3, 3, C, cout)).astype(np.float32)
    return hi + lo, w


def variants():
    from rendernet_b200 import ops
    return {
        "F(2x2)": dict(mats=F2, m=2),
        "F(4x4) points 0, +-1, +-2": dict(mats=ops.wino4_matrices((0.0, 1.0, -1.0, 2.0, -2.0)), m=4),
        "F(4x4) points 0, +-1, +-1/2": dict(mats=ops.wino4_matrices(), m=4),
        "F(4x4) points 0, +-1, +-1/2, V/2, U 2^s (shipped)": dict(mats=ops.wino4_matrices(), m=4, v_half=True,
                                                                   u_exp_rule=ops.wino4_exponent),
    }


def measure(x, w, **variant):
    y, vmax = emulate(x, w, **variant)
    ref = direct(x, w)
    s = float(np.abs(ref).max())
    err = y.astype(np.float64) - ref
    return {"max_err": float(np.abs(err).max()) / s, "rel_rms": float(np.sqrt((err ** 2).mean() / (ref ** 2).mean())),
            "v_over_x": vmax / float(np.abs(x).max()), "finite": bool(np.isfinite(y).all())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cout", type=int, default=64)
    ap.add_argument("--hw", type=int, default=16)
    ap.add_argument("--scale", type=float, default=3.0)
    ap.add_argument("--uniform", action="store_true", help="x ~ U(-scale, scale) instead of scale N(0, 1)")
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    x, w = inputs(a.hw, 1024, a.cout, a.scale, a.seed, a.uniform)
    print(json.dumps({k: measure(x, w, **v) for k, v in variants().items()}, indent=1))


if __name__ == "__main__":
    main()
