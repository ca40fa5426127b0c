"""Which implicit-GEMM kernel variants exist, and that every launch plan names one of them (rn_conv_plan: host arithmetic,
runs without a GPU).

igemm_kernel is compiled once per <N tile, cluster, M sub-tiles, split, half, raw> variant: the Makefile's VARIANTS list
builds the objects and RN_IGEMM_VARIANTS (rn_igemm.cuh) is the dispatch table.  The two lists must be the same set, and a
descriptor that rn_conv_plan accepts must lead to a built variant -- otherwise the plan says yes to something the device
cannot launch (-25 now, a cudaErrorInvalidDeviceFunction from the dispatch before)."""
import ctypes as C
import itertools
import os
import re

from rendernet_b200._lib import PLAN_FIELDS, lib, rn_conv_desc

CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "rendernet_b200", "csrc")
FAKE = 0x10000       # non-null, 16-byte aligned; rn_conv_plan never dereferences pointers
NO_KERNEL = -25


def makefile_variants():
    text = open(os.path.join(CSRC, "Makefile")).read()
    body = re.search(r"^VARIANTS :=((?:.*\\\n)*.*)$", text, re.M).group(1)
    names = body.replace("\\", " ").split()
    return {tuple(int(f) for f in (n.split("_") + ["0"])[:6]) for n in names}     # a missing sixth field (raw) is 0


def dispatch_variants():
    text = open(os.path.join(CSRC, "rn_igemm.cuh")).read()
    body = re.search(r"^#define RN_IGEMM_VARIANTS\(X\)((?:.*\\\n)*.*)$", text, re.M).group(1)
    return {tuple(int(v) for v in m) for m in re.findall(r"X\((\d+), (\d+), (\d+), (\d+), (\d+), (\d+)\)", body)}


BUILT = makefile_variants()


def test_makefile_and_dispatch_table_list_the_same_variants():
    table = dispatch_variants()
    assert len(BUILT) == 33 and len(table) == 33
    assert BUILT == table, f"only in the Makefile: {sorted(BUILT - table)}, only in RN_IGEMM_VARIANTS: {sorted(table - BUILT)}"
    src = open(os.path.join(CSRC, "rn_igemm.cu")).read()
    assert "RN_IGEMM_VARIANTS(RN_V)" in src and "igemm_variant_built(" in src     # launch_variant and plan_conv both use it


# band geometry of the depth-folded 3^3 conv3d as rn_conv3d_banded_same fills it: band_cin = 32 input and band_cout = 32
# output channels per depth, z stride 1 -> 3 K blocks of 64 per (ky, kx) tap
BAND = dict(band_cin=32, band_cout=32, band_sz=1, Cin=192)


def desc(ndim=2, fmt=0, cout_pad=64, force_bn=0, cluster=0, msub=0, banded=False, bias=True, large=True, ny=0, **extra):
    """A descriptor for rn_conv_plan.  bias=False: the raw fp32 path (out32 only, no activation or residual)."""
    if ndim == 2:
        taps = [(kx - 1, ky - 1, 0) for ky in range(3) for kx in range(3)]          # tap = ky*3 + kx, dy consecutive
        B, H, W, D = (2, 64, 64, 1) if large else (1, 8, 8, 1)
    else:
        taps = [(0, 0, dz) for dz in (-1, 0, 1)]
        B, H, W, D = (2, 16, 16, 8) if large else (1, 4, 4, 4)
    d = rn_conv_desc()
    d.ndim, d.B, d.H, d.W, d.D = ndim, B, H, W, D
    d.Cin, d.Cout, d.cout_pad, d.ntaps = 64, cout_pad, cout_pad, len(taps)
    arr = (C.c_int8 * (3 * len(taps)))(*[v for t in taps for v in t])
    d.taps = C.cast(arr, C.c_void_p)
    d.x = d.w_packed = FAKE
    d.bias = FAKE if bias else None
    d.alpha = FAKE
    d.act = 1 if bias else 0
    d.residual = FAKE if bias else None
    d.out16 = FAKE if bias else None
    d.out32 = FAKE
    d.o_base, d.o_b, d.o_y, d.o_x, d.o_z = 0, H * W * D * cout_pad, W * D * cout_pad, D * cout_pad, cout_pad
    d.fmt, d.force_bn, d.cluster, d.msub, d.ny = fmt, force_bn, cluster, msub, ny
    if fmt == 2:
        d.x_plane = d.w_plane = d.o_plane = 8
    if banded:
        d.w_banded, d.x_channels = 1, D * 32
        d.band_cin, d.band_cout, d.band_sz, d.Cin = BAND["band_cin"], BAND["band_cout"], BAND["band_sz"], BAND["Cin"]
    for key, val in extra.items():
        setattr(d, key, val)
    d._taps = arr                   # keep the tap array alive with the descriptor
    return d


def plan(d):
    out = (C.c_int * 16)()
    rc = lib.rn_conv_plan(C.byref(d), out, 16)
    return rc, dict(zip(PLAN_FIELDS, out))


def variant_of(d, p):
    return (p["bn"], p["cluster"], p["msub"], 1 if d.fmt == 2 else 0, 1 if (d.w_banded and d.band_cin > 0) else 0,
            0 if d.bias else 1)


COUT_PADS = (16, 32, 48, 64, 96, 128, 192, 256, 384, 512, 1024)


def test_every_accepted_plan_names_a_built_variant():
    """rn_conv_plan over ndim x fmt x cout_pad x force_bn x cluster x msub x banded x bias x image size x halo sharing: every
    plan it accepts names a built variant, and the grid reaches all of them (the raw one only with fmt 2 and cout_pad % 256
    == 0, the banded ones only with force_bn = 128 -- so a miss here means the grid is incomplete)."""
    reached, accepted, bad = set(), 0, []
    for ndim, fmt, cp in itertools.product((2, 3), (0, 1, 2), COUT_PADS):
        for fbn, cl, ms, banded, bias, large, ny in itertools.product(
                [0] + [b for b in (16, 32, 64, 128, 256) if cp % b == 0], (0, 1, 2, 4), (0, 1, 2), (False, True),
                (True, False), (False, True), (0, 3)):
            if ndim == 3 and (banded or ny):
                continue               # the banded conv and halo sharing are 2-D descriptors
            d = desc(ndim, fmt, cp, fbn, cl, ms, banded, bias, large, ny)
            rc, p = plan(d)
            if rc != 0:
                continue
            accepted += 1
            v = variant_of(d, p)
            reached.add(v)
            if v not in BUILT:
                bad.append((dict(ndim=ndim, fmt=fmt, cout_pad=cp, force_bn=fbn, cluster=cl, msub=ms, banded=banded,
                                 bias=bias, large=large, ny=ny), v))
    assert not bad, f"{len(bad)} accepted plans name an unbuilt variant, e.g. {bad[:4]}"
    assert accepted > 1000
    assert reached == BUILT, f"variants the grid never reaches: {sorted(BUILT - reached)}"


def test_plans_without_a_kernel_are_rejected():
    """bias = NULL (raw fp32 output) is built only as the exact-mode N = 256, unbanded variant."""
    assert plan(desc(fmt=2, cout_pad=256, bias=False))[0] == 0                      # the Winograd per-position GEMM
    assert plan(desc(ndim=3, fmt=2, cout_pad=512, bias=False))[0] == 0
    assert plan(desc(fmt=0, cout_pad=256, bias=False))[0] == NO_KERNEL              # fast mode
    assert plan(desc(fmt=1, cout_pad=256, bias=False))[0] == NO_KERNEL              # bf16
    assert plan(desc(fmt=2, cout_pad=128, bias=False))[0] == NO_KERNEL              # N tile 128
    assert plan(desc(fmt=2, cout_pad=384, bias=False))[0] == NO_KERNEL              # cout_pad % 256 != 0
    assert plan(desc(fmt=2, cout_pad=256, force_bn=128, bias=False))[0] == NO_KERNEL
    assert plan(desc(fmt=2, cout_pad=256, force_bn=128, banded=True, bias=False))[0] == NO_KERNEL
    assert plan(desc(fmt=2, cout_pad=256, force_bn=128, banded=True))[0] == 0       # the same banded conv with a bias


def test_exact_mode_16bit_residual_needs_its_lo_plane():
    """fmt 2 reads the LO plane of a 16-bit residual at o_plane, also when only out32 is written; without it the epilogue
    would add the HI plane twice."""
    kw = dict(fmt=2, cout_pad=64, out16=None, out32=FAKE)
    assert plan(desc(o_plane=0, **kw))[0] == -18
    assert plan(desc(o_plane=64 * 64 * 64 * 2, **kw))[0] == 0
    assert plan(desc(o_plane=0, residual_is_f32=1, **kw))[0] == 0                  # an fp32 residual has no LO plane
    assert plan(desc(o_plane=0, residual=None, **kw))[0] == 0
