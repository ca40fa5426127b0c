"""Host side of the exact-mode Winograd F(2x2, 3x3) trunk convolution (rn_winograd.cu): the filter transform against NumPy
float64, the whole transform chain against a direct float64 convolution (so the B^T / G / A^T matrices are the ones the
kernels use), the workspace size, the routing decision and the per-position GEMM's launch plan.  No GPU needed."""
import ctypes as C

import numpy as np
import pytest
import torch

from rendernet_b200 import ops
from rendernet_b200._lib import lib, rn_tuning

BT = np.array([[1, 0, -1, 0], [0, 1, 1, 0], [0, -1, 1, 0], [0, 1, 0, -1]], dtype=np.float64)
G = np.array([[1, 0, 0], [0.5, 0.5, 0.5], [0.5, -0.5, 0.5], [0, 0, 1]], dtype=np.float64)
AT = np.array([[1, 1, 1, 0], [0, 1, -1, -1]], dtype=np.float64)


def test_filter_transform_matches_numpy_float64():
    rng = np.random.default_rng(0)
    cin, cout = 48, 32
    w = rng.standard_normal((3, 3, cin, cout)).astype(np.float32)
    U = ops.winograd_filter_f32(torch.from_numpy(w)).numpy()
    assert U.shape == (16, cout, cin) and U.dtype == np.float32
    ref = np.einsum("ak,klio,bl->aboi", G, w.astype(np.float64), G).reshape(16, cout, cin)
    assert np.array_equal(U, ref.astype(np.float32))          # float64, then ONE rounding to fp32


def test_transform_chain_is_the_3x3_same_convolution():
    """V = B^T d B per 4x4 patch (zero padded), U per position, y = A^T (sum_ci U V) A per 2x2 block, in float64, equals the
    SAME cross-correlation of TF's conv2d, on a non-square image."""
    rng = np.random.default_rng(1)
    H, W, cin, cout = 6, 10, 3, 2
    x = rng.standard_normal((H, W, cin))
    w = rng.standard_normal((3, 3, cin, cout)).astype(np.float32)
    U = np.einsum("ak,klio,bl->abio", G, w.astype(np.float64), G)
    xp = np.pad(x, ((1, 1), (1, 1), (0, 0)))
    y = np.zeros((H, W, cout))
    for ty in range(H // 2):
        for tx in range(W // 2):
            d = xp[2 * ty:2 * ty + 4, 2 * tx:2 * tx + 4]                  # rows 2ty-1 .. 2ty+2 of x
            V = np.einsum("ai,ijc,bj->abc", BT, d, BT)
            M = np.einsum("abio,abi->abo", U, V)
            y[2 * ty:2 * ty + 2, 2 * tx:2 * tx + 2] = np.einsum("ia,abo,jb->ijo", AT, M, AT)
    ref = np.zeros((H, W, cout))
    for ky in range(3):
        for kx in range(3):
            ref += np.einsum("hwi,io->hwo", xp[ky:ky + H, kx:kx + W], w[ky, kx].astype(np.float64))
    assert np.abs(y - ref).max() <= 1e-12 * np.abs(ref).max()


def test_workspace_bytes():
    B, H, W, C = 24, 64, 64, 1024
    pos = B * (H // 2) * (W // 2) * C
    assert lib.rn_winograd_workspace_bytes(B, H, W, C) == 16 * pos * 2 * 2 + 16 * pos * 4   # V hi/lo fp16 + M fp32
    assert lib.rn_winograd_workspace_bytes(1, 18, 34, 64) == 16 * 9 * 17 * 64 * 8
    for bad in ((24, 63, 64, 1024), (24, 64, 64, 1000), (0, 64, 64, 1024)):
        assert lib.rn_winograd_workspace_bytes(*bad) == -1


def _tune(w):
    t = rn_tuning()
    t.winograd = w
    return C.byref(t)


@pytest.mark.parametrize("args,want", [((2, 3, 3, 64, 64, 1024, 1024, 1024), 1),     # res2 trunk
                                       ((2, 3, 3, 64, 64, 512, 512, 512), 0),        # res3: below the threshold
                                       ((0, 3, 3, 64, 64, 1024, 1024, 1024), 0),     # fast mode stays direct
                                       ((2, 1, 1, 64, 64, 1024, 1024, 1024), 0),     # projection
                                       ((2, 3, 3, 63, 64, 1024, 1024, 1024), 0),     # odd H
                                       ((2, 3, 3, 64, 64, 1024, 512, 512), 0)])      # Cin != Cout
def test_routing(args, want):
    assert lib.rn_conv2d_winograd_eligible(*args, None) == want
    assert lib.rn_conv2d_winograd_eligible(*args, _tune(-1)) == 0
    if want:
        assert lib.rn_conv2d_winograd_eligible(*args, _tune(1)) == 1


def test_forcing_takes_res3_but_no_unsupported_shape():
    assert lib.rn_conv2d_winograd_eligible(2, 3, 3, 64, 64, 512, 512, 512, _tune(1)) == 1
    assert lib.rn_conv2d_winograd_eligible(0, 3, 3, 64, 64, 512, 512, 512, _tune(1)) == 0
    assert lib.rn_conv2d_winograd_eligible(2, 3, 3, 64, 63, 512, 512, 512, _tune(1)) == 0


def _gemm_plan(ntaps=1, B=16 * 24, b_tap_div=24):
    from rendernet_b200._lib import PLAN_FIELDS, rn_conv_desc
    taps = (C.c_int8 * (3 * ntaps))()
    d = rn_conv_desc()
    d.ndim, d.B, d.H, d.W, d.D, d.Cin, d.Cout, d.cout_pad, d.ntaps = 2, B, 32, 32, 1, 1024, 1024, 1024, ntaps
    d.taps = C.cast(taps, C.c_void_p)
    d.x = d.w_packed = d.bias = d.out32 = 0x10000
    d.o_b, d.o_y, d.o_x = 32 * 32 * 1024, 32 * 1024, 1024
    d.fmt, d.x_plane, d.w_plane, d.b_tap_div = 2, B * 32 * 32 * 1024, 16 * 1024 * 1024, b_tap_div
    out = (C.c_int * 16)()
    rc = lib.rn_conv_plan(C.byref(d), out, 16)
    return rc, dict(zip(PLAN_FIELDS, out))


def test_per_position_gemm_plan():
    """The 16 GEMMs of a B = 24 trunk layer: one launch over 16*24 images of 32x32, tiles never straddle an image (so each
    reads one position's filter), N-fastest 256-column tiles."""
    rc, p = _gemm_plan()
    assert rc == 0
    assert (p["bn"], p["tile_w"], p["tile_h"]) == (256, 32, 4)
    assert p["tiles"] == 16 * 24 * (32 // 4) * (1024 // 256)
    assert _gemm_plan(ntaps=9)[0] == -23              # the per-image filter tap is for one-tap convs only
    assert _gemm_plan(B=16 * 24 + 1)[0] == -23         # every position holds the same number of images
