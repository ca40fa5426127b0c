"""Launch-plan heuristics of the implicit-GEMM convolution (rn_conv_plan: pure host arithmetic, runs without a GPU).
Pins the decisions the sizing code makes on the H100 (132 SMs, 227 KB of shared memory per block) for the BASELINE-size
layers (DESIGN.md §3.1) so that a change to it cannot silently drop the banded convs' halo sharing, turn the (slower)
weight multicast clusters on by default or drop the thin layers' second accumulator -- and checks the argument validation of rn_conv_igemm's front end."""
import ctypes as C

import pytest

from rendernet_b200._lib import PLAN_FIELDS, lib, rn_conv_desc

FAKE = 0x10000       # non-null, 16-byte aligned; rn_conv_plan never dereferences pointers


def plan(ndim=2, B=24, H=64, W=64, D=1, Cin=1024, Cout=1024, cout_pad=None, k=3, ny=0, residual=False, out32=False,
         force_bn=0, x_channels=0, w_banded=0, cluster=0, cta_group=0, msub=0, taps=None, expect=0, **extra):
    if taps is None:
        lo = -((k - 1) // 2)
        taps = [(kx + lo, ky + lo, 0) for ky in range(k) for kx in range(k)]     # tap = ky*k + kx, dy consecutive
    arr = (C.c_int8 * (3 * len(taps)))(*[v for t in taps for v in t])
    d = rn_conv_desc()
    d.ndim, d.B, d.H, d.W, d.D = ndim, B, H, W, D
    d.Cin, d.Cout, d.cout_pad, d.ntaps = Cin, Cout, cout_pad or Cout, len(taps)
    d.taps = C.cast(arr, C.c_void_p)
    d.x = d.w_packed = d.bias = d.alpha = FAKE
    d.act = 1
    d.residual = FAKE if residual else None
    d.out16 = None if out32 else FAKE
    d.out32 = FAKE if out32 else None
    cp = d.cout_pad
    d.o_base, d.o_b, d.o_y, d.o_x, d.o_z = 0, H * W * cp, W * cp, cp, 0
    d.force_bn, d.x_channels, d.w_banded = force_bn, x_channels, w_banded
    d.cluster, d.cta_group, d.ny, d.msub = cluster, cta_group, ny, msub
    for key, val in extra.items():
        setattr(d, key, val)
    out = (C.c_int * 16)()
    rc = lib.rn_conv_plan(C.byref(d), out, 16)
    assert rc == expect, f"rn_conv_plan rc={rc}, expected {expect}"
    return dict(zip(PLAN_FIELDS, out)) if rc == 0 else None


def test_plan_trunk_and_projection():
    p = plan(Cin=1024, Cout=1024, k=3, ny=3)                       # res2 conv: the dominant kernel
    # three full 256-row weight tiles per halo group would leave fewer than 3 stages: one activation load per tap
    assert (p["bn"], p["cluster"], p["cta_group"], p["msub"], p["ny"]) == (256, 1, 1, 1, 1)
    assert (p["tile_w"], p["tile_h"]) == (64, 2) and p["stages"] >= 3 and p["epilogue_mode"] == 0
    assert p["epilogue_groups"] == 2                               # both consumer warpgroups store their own rows
    assert p["smem_bytes"] <= 232448 and p["grid"] == 132 and p["tiles"] == 24 * 32 * 4
    q = plan(Cin=1024, Cout=1024, k=1)                             # projection unit: 16 k-blocks per tile
    assert (q["bn"], q["cluster"], q["ny"]) == (256, 1, 1) and q["stages"] >= 3
    r = plan(H=32, W=32, Cin=512, Cout=512, k=3, ny=3)             # res3
    assert (r["bn"], r["cluster"]) == (256, 1) and r["stages"] >= 3


def test_plan_banded_res1_and_thin_layers():
    # res1: depth-folded 3^3 conv, K per tap = 192 of the 1024 folded channels, N tile 128 (rn_conv3d_banded_same)
    kw = dict(Cin=192, Cout=1024, k=3, ny=3, force_bn=128, x_channels=1024, w_banded=1)
    p = plan(**kw)                                                 # a second accumulator would cost the third stage
    assert (p["bn"], p["cluster"], p["msub"], p["ny"]) == (128, 1, 1, 3) and p["stages"] >= 3
    assert (p["tile_w"], p["tile_h"]) == (16, 8) and p["tiles"] == 24 * 4 * 8 * 8      # 16x8-pixel CTA tiles
    p1 = plan(cluster=2, **kw)                                     # per-call multicast cluster
    assert (p1["cluster"], p1["msub"], p1["ny"]) == (2, 1, 3) and p1["stages"] >= 3
    assert plan(msub=1, **kw)["msub"] == 1
    # x-folded e_conv11-like thin layer: N tile 16, two M sub-tiles
    t = plan(H=512, W=128, Cin=64, Cout=16, k=1, taps=[(dx, dy, 0) for dy in (-2, -1, 0, 1) for dx in (-1, 0, 1)], ny=4)
    assert (t["bn"], t["cluster"], t["msub"], t["epilogue_groups"], t["ny"]) == (16, 1, 2, 2, 4)
    # tiny image: nothing to pair, halo sharing falls away when the pipeline would starve
    s = plan(B=1, H=4, W=8, Cin=64, Cout=64, k=3, ny=3)
    assert s["msub"] == 1 and s["stages"] >= 2


def test_plan_tuning_switches_and_validation():
    # per-call overrides travel in the descriptor (the library has no mutable global state)
    assert plan(Cin=1024, Cout=1024, k=3, ny=3, cluster=4)["cluster"] == 4
    assert plan(Cin=1024, Cout=1024, k=3, ny=3, cta_group=1)["cta_group"] == 1
    plan(Cin=1024, Cout=1024, k=3, cta_group=2, expect=-22)        # no paired (two-CTA) MMA on sm_90
    assert plan(Cin=1024, Cout=1024, k=3, ny=3, tma_store=-1)["epilogue_mode"] == 0
    assert plan(Cin=1024, Cout=1024, k=3, ny=3, out32=True)["epilogue_mode"] == 0      # fp32 output: direct stores
    plan(Cin=1000, expect=-4)                        # Cin % 16
    plan(Cout=1030, cout_pad=1024, expect=-4)        # Cout > cout_pad
    plan(ndim=4, expect=-2)
    plan(B=0, expect=-7)
    plan(force_bn=96, expect=-9)
    plan(k=3, ny=3, taps=[(0, 0, 0)] * 9, expect=-14)      # taps not ordered for halo sharing
    plan(msub=3, expect=-16)
    assert lib.rn_conv_plan(None, (C.c_int * 16)(), 16) == -1


def test_plan_exact_mode_split_operands():
    """RN_FMT_F16X2: every tap becomes 3 pseudo-taps (x_hi.w_hi, x_lo.w_hi, x_hi.w_lo); split kernels run on single CTAs
    (no multicast cluster); the LO-plane offsets are mandatory."""
    planes = dict(fmt=2, x_plane=24 * 64 * 64 * 1024, w_plane=9 * 1024 * 1024, o_plane=24 * 64 * 64 * 1024)
    p = plan(Cin=1024, Cout=1024, k=3, ny=3, **planes)
    assert (p["bn"], p["cluster"], p["cta_group"], p["epilogue_mode"]) == (256, 1, 1, 0)
    assert p["stages"] >= 3 and p["smem_bytes"] <= 232448
    q = plan(Cin=1024, Cout=1024, k=1, **planes)
    assert (q["bn"], q["cluster"]) == (256, 1)
    b = plan(Cin=192, Cout=1024, k=3, ny=3, force_bn=128, x_channels=1024, w_banded=1, **planes)
    assert (b["bn"], b["cluster"], b["msub"], b["ny"]) == (128, 1, 1, 3)
    odd = plan(B=1, H=24, W=8, Cin=64, Cout=256, k=3, fmt=2, x_plane=8 * 24 * 64, w_plane=9 * 256 * 64, o_plane=8 * 24 * 256)
    assert (odd["cluster"], odd["cta_group"]) == (1, 1)
    k4 = plan(Cin=64, Cout=64, k=4, taps=[(kx - 1, ky - 1, 0) for ky in range(4) for kx in range(4)], fmt=2,
              x_plane=24 * 64 * 64 * 64, w_plane=16 * 64 * 64, o_plane=24 * 64 * 64 * 64)       # 16 taps x 3 = 48 pseudo-taps
    assert k4["stages"] >= 2
    plan(Cin=64, Cout=64, k=3, fmt=2, expect=-18)                                   # LO-plane offsets missing
    plan(ndim=3, D=8, Cin=32, Cout=32, k=3, taps=[(a, b, c) for a in (-1, 0, 1) for b in (-1, 0, 1) for c in (-1, 0, 1)],
         fmt=2, x_plane=8, w_plane=8, o_plane=8, expect=-3)                         # 27 taps x 3 > 48
    plan(fmt=3, expect=-17)
