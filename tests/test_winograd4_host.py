"""Host side of the exact-mode Winograd F(4x4, 3x3) trunk convolution (rn_winograd.cu): the transform matrices derived again
from their interpolation points in float64, the whole transform chain against a direct float64 convolution, the filter
transform against NumPy float64 with its power-of-two scale, the workspace size, the output-tile routing and the 36-position
GEMM's launch plan.  No GPU needed."""
import ctypes as C
from fractions import Fraction

import numpy as np
import pytest
import torch

from rendernet_b200 import ops
from rendernet_b200._lib import PLAN_FIELDS, lib, rn_conv_desc, rn_tuning


def _toom_cook(points):
    """B^T, G, A^T of F(4, 3) for the finite points plus infinity, in exact rationals (independent of ops.wino4_matrices)."""
    p = [Fraction(q).limit_denominator(16) for q in points]
    n = len(p) + 1
    BT = [[Fraction(0)] * n for _ in range(n)]
    G = [[Fraction(0)] * 3 for _ in range(n)]
    AT = [[Fraction(0)] * n for _ in range(4)]
    for j in range(n):
        poly = [Fraction(1)]                                             # coefficients, lowest power first
        for l, q in enumerate(p):
            if l != j:
                poly = [(poly[i - 1] if i > 0 else 0) - q * (poly[i] if i < len(poly) else 0) for i in range(len(poly) + 1)]
        BT[j][:len(poly)] = poly
        if j < n - 1:
            den = Fraction(1)
            for l, q in enumerate(p):
                if l != j:
                    den *= p[j] - q
            G[j] = [p[j] ** k / den for k in range(3)]
            for i in range(4):
                AT[i][j] = p[j] ** i
    G[n - 1][2] = Fraction(1)
    AT[3][n - 1] = Fraction(1)
    f = lambda m: np.array([[float(v) for v in row] for row in m])
    return f(BT), f(G), f(AT)


def test_matrices_are_the_interpolation_points_toom_cook():
    BT, G, AT = ops.wino4_matrices()
    rBT, rG, rAT = _toom_cook(ops.WINO4_POINTS)
    assert ops.WINO4_POINTS == (0.0, 1.0, -1.0, 0.5, -0.5)
    assert np.array_equal(BT, rBT) and np.array_equal(AT, rAT)
    assert np.abs(G - rG).max() <= 1e-15
    # the rows the kernels spell out (rn_winograd.cu)
    assert np.array_equal(BT[0], [0.25, 0, -1.25, 0, 1, 0]) and np.array_equal(BT[5], [0, 0.25, 0, -1.25, 0, 1])
    assert np.array_equal(AT[3], [0, 1, -1, 0.125, -0.125, 1])
    assert np.abs(BT).sum(axis=1).max() == 3.0                          # |1/2 B^T d B| <= 4.5 |x|


def test_transform_chain_is_the_3x3_same_convolution():
    """V = 1/2 B^T d B per 6x6 patch (zero padded), U = 2^s G g G^T, y = 2^(1-s) A^T (sum_ci U V) A per 4x4 block, in float64,
    equals TF's SAME cross-correlation on a non-square image whose sides are multiples of 4."""
    BT, G, AT = ops.wino4_matrices()
    rng = np.random.default_rng(1)
    H, W, cin, cout, s = 8, 20, 3, 2, 7
    x = rng.standard_normal((H, W, cin))
    w = rng.standard_normal((3, 3, cin, cout))
    U = 2.0 ** s * np.einsum("ak,klio,bl->abio", G, w, G)
    xp = np.pad(x, ((1, 1), (1, 1), (0, 0)))
    y = np.zeros((H, W, cout))
    for ty in range(H // 4):
        for tx in range(W // 4):
            d = xp[4 * ty:4 * ty + 6, 4 * tx:4 * tx + 6]                   # rows 4ty-1 .. 4ty+4 of x
            V = 0.5 * np.einsum("ai,ijc,bj->abc", BT, d, BT)
            M = np.einsum("abio,abi->abo", U, V)
            y[4 * ty:4 * ty + 4, 4 * tx:4 * tx + 4] = 2.0 ** (1 - s) * np.einsum("ia,abo,jb->ijo", AT, M, AT)
    ref = np.zeros((H, W, cout))
    for ky in range(3):
        for kx in range(3):
            ref += np.einsum("hwi,io->hwo", xp[ky:ky + H, kx:kx + W], w[ky, kx])
    assert np.abs(y - ref).max() <= 1e-12 * np.abs(ref).max()


@pytest.mark.parametrize("scale", [0.01, 1.0, 3e-5])
def test_filter_transform_matches_numpy_float64(scale):
    """U = 2^s G g G^T in float64, then ONE rounding to fp32; s puts max |U| in (2^11, 2^12]."""
    rng = np.random.default_rng(int(scale * 1e5))
    cin, cout = 48, 32
    w = (rng.standard_normal((3, 3, cin, cout)) * scale).astype(np.float32)
    U, s = ops.winograd4_filter_f32(torch.from_numpy(w))
    U = U.numpy()
    assert U.shape == (36, cout, cin) and U.dtype == np.float32
    G = _toom_cook(ops.WINO4_POINTS)[1]
    u64 = np.einsum("ak,klio,bl->aboi", G, w.astype(np.float64), G).reshape(36, cout, cin)
    assert 2.0 ** 11 < np.abs(u64).max() * 2.0 ** s <= 2.0 ** 12
    # one rounding: within half an fp32 ulp of the float64 value.  Not bit-equal to NumPy's: sums of fp32 filter values land
    # on fp32 rounding ties, and the last float64 bits of torch's and NumPy's einsum decide those either way.
    err = np.abs(U.astype(np.float64) - u64 * 2.0 ** s)
    assert (err <= 0.5 * np.spacing(np.abs(U)).astype(np.float64) * (1 + 1e-6)).all()


def test_exponent_rule():
    assert ops.wino4_exponent(4096.0) == 0 and ops.wino4_exponent(4095.0) == 0
    assert ops.wino4_exponent(2048.0) == 1 and ops.wino4_exponent(2049.0) == 0
    assert ops.wino4_exponent(0.03) == 17
    assert ops.wino4_exponent(0.0) == 0
    for v in np.geomspace(1e-6, 1e6, 97):
        s = ops.wino4_exponent(float(v))
        assert 2.0 ** 11 < v * 2.0 ** s <= 2.0 ** 12


def test_workspace_bytes():
    B, H, W, C = 24, 64, 64, 1024
    pos = B * (H // 4) * (W // 4) * C
    assert lib.rn_winograd4_workspace_bytes(B, H, W, C) == 36 * pos * 2 * 2 + 36 * pos * 4   # V hi/lo fp16 + M fp32
    assert lib.rn_winograd4_workspace_bytes(1, 20, 36, 64) == 36 * 5 * 9 * 64 * 8
    # 9/16 of F(2x2)'s workspace
    assert lib.rn_winograd4_workspace_bytes(B, H, W, C) * 16 == lib.rn_winograd_workspace_bytes(B, H, W, C) * 9
    for bad in ((24, 62, 64, 1024), (24, 64, 18, 1024), (24, 64, 64, 1000), (0, 64, 64, 1024), (1, 0, 4, 64)):
        assert lib.rn_winograd4_workspace_bytes(*bad) == -1


def _tune(**kw):
    t = rn_tuning()
    for k, v in kw.items():
        setattr(t, k, v)
    return C.byref(t)


@pytest.mark.parametrize("args,want", [((2, 3, 3, 64, 64, 1024, 1024, 1024), 4),     # res2 trunk
                                       ((2, 3, 3, 18, 34, 1024, 1024, 1024), 2),     # even, not multiples of 4
                                       ((2, 3, 3, 20, 36, 1024, 1024, 1024), 4),
                                       ((2, 3, 3, 64, 64, 512, 512, 512), 0),        # res3: below the threshold
                                       ((0, 3, 3, 64, 64, 1024, 1024, 1024), 0),     # fast mode stays direct
                                       ((2, 3, 3, 63, 64, 1024, 1024, 1024), 0)])    # odd H
def test_tile_routing(args, want):
    assert lib.rn_conv2d_winograd_tile(*args, None) == want
    assert lib.rn_conv2d_winograd_tile(*args, _tune(winograd=-1)) == 0
    assert lib.rn_conv2d_winograd_tile(*args, _tune(wino_tile=2)) == (2 if want else 0)
    assert lib.rn_conv2d_winograd_tile(*args, _tune(wino_tile=4)) == want
    assert bool(lib.rn_conv2d_winograd_eligible(*args, None)) == bool(want)     # eligibility keeps its meaning


def test_forced_res3_takes_f4():
    assert lib.rn_conv2d_winograd_tile(2, 3, 3, 64, 64, 512, 512, 512, _tune(winograd=1)) == 4


def test_tuning_struct_appends_wino_tile():
    names = [f[0] for f in rn_tuning._fields_]
    assert names[-2:] == ["winograd", "wino_tile"]


def _gemm_plan(B=36 * 24, b_tap_div=24, hw=16):
    taps = (C.c_int8 * 3)()
    d = rn_conv_desc()
    d.ndim, d.B, d.H, d.W, d.D, d.Cin, d.Cout, d.cout_pad, d.ntaps = 2, B, hw, hw, 1, 1024, 1024, 1024, 1
    d.taps = C.cast(taps, C.c_void_p)
    d.x = d.w_packed = d.bias = d.out32 = 0x10000
    d.bias = None
    d.o_b, d.o_y, d.o_x = hw * hw * 1024, hw * 1024, 1024
    d.fmt, d.x_plane, d.w_plane, d.b_tap_div = 2, B * hw * hw * 1024, 36 * 1024 * 1024, b_tap_div
    d.force_bn = 256
    out = (C.c_int * 16)()
    rc = lib.rn_conv_plan(C.byref(d), out, 16)
    return rc, dict(zip(PLAN_FIELDS, out))


def test_36_position_gemm_plan():
    """The 36 GEMMs of a B = 24 trunk layer: one launch over 36*24 images of 16x16, 16 x 8 boxes (a 128-row tile never
    straddles two position images, so every tile reads one position's filter and B = 24, 8 and 1 give the same bits), N-fastest
    256-column tiles: 6 912 tiles, 56 % of F(2x2)'s 12 288."""
    rc, p = _gemm_plan()
    assert rc == 0
    assert (p["bn"], p["tile_w"], p["tile_h"], p["msub"]) == (256, 16, 8, 1)
    assert p["tiles"] == 36 * 24 * 2 * (1024 // 256) == 6912
    for b in (8, 1):
        rc, q = _gemm_plan(B=36 * b, b_tap_div=b)
        assert rc == 0 and (q["tile_w"], q["tile_h"]) == (16, 8) and q["tiles"] == 36 * b * 2 * 4
    assert _gemm_plan(B=36 * 24 + 1)[0] == -23
