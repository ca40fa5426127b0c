"""Every built implicit-GEMM variant (RN_IGEMM_VARIANTS in rn_igemm.cuh, 33 of them) and both epilogue store paths against a
float64 convolution of the very operands the kernel reads, at the edges where the kernel can go wrong.

* One case per variant, plus bf16 cases for every non-split N tile.  Each case pins its plan through rn_conv_plan on the
  descriptor it launches -- (N tile, cluster, M sub-tiles, halo sharing) -- so a heuristic change cannot move it onto
  another variant unnoticed.  Variants are chosen with per-call descriptor fields only.
* Ragged M (W and H not multiples of the tile box, a second M sub-tile partly or wholly below the image, D not a multiple
  of the depth box, B >= 2), ragged N (Cout < cout_pad, Cout % 8 != 0, strided channel views, the o_nsplit address split),
  K blocks of 32, 64 and 128 bytes, 1x1 / 3x3 / halo-shared 3x3 / 3-D taps, max_ctas coprime with the tile count, clusters
  on grids that are rounded down to a multiple of the cluster size.
* Exact-mode (fp16 hi/lo pair) operands carry LO halves that are fp16 subnormals (DESIGN §4).
* Epilogue: the cases run through every activation x residual x output combination on the 16-byte vector path and on the
  scalar path (test_epilogue_matrix_is_covered).
* Checks: out32 against float64 as max |err| / max |ref| (the operands are exact, so this is fp32 accumulation alone);
  16-bit outputs bit for bit against the rounding of out32 (hi = fp16(out32), lo = fp16(out32 - hi) for pairs); NaN
  sentinels before, between and after the output rows, in the channels past Cout, in the columns o_nsplit skips and in
  both planes of a pair, all of which must survive the launch.
"""
import ctypes as C
import itertools
import math

import pytest
import torch

from rendernet_b200._lib import PLAN_FIELDS, check, lib, rn_conv_desc

dev = "cuda"
ACTS, RESS, OUTS = ("none", "prelu", "sigmoid"), ("none", "16", "f32"), ("16", "32", "both")
COMBOS = list(itertools.product(ACTS, RESS, OUTS))
MARGIN = 40                 # elements of NaN before o_base and after the last row


def bar(K):
    """fp32 accumulation error bar, max |err| / max |ref|, for K = taps x input channels: the truncating accumulation adds
    one error per k16 MMA step, so it grows like sqrt(K / 16).  Measured on one H100 80GB HBM3 (700 W power limit), over the
    39 cases of test_variant: at most 2.05e-7 x sqrt(K / 16) (256_1_1_0_0, K = 1152: 1.74e-6; 128_1_2_0_1, K = 864:
    1.05e-6; exact mode at most 9.1e-8 x sqrt(K / 16)); the bar is 3x that."""
    return 6e-7 * math.sqrt(max(K, 16) / 16)

TAPS = {
    "1x1": [(0, 0, 0)],
    "3x3": [(kx - 1, ky - 1, 0) for ky in range(3) for kx in range(3)],          # tap = ky*3 + kx, dy consecutive
    "2x2": [(kx, ky - 1, 0) for ky in range(2) for kx in range(2)],
    "3^3": [(kx - 1, ky - 1, kz - 1) for ky in range(3) for kx in range(3) for kz in range(3)],
    "2^3": [(kx - 1, ky, kz) for ky in range(2) for kx in range(2) for kz in range(2)],
}


class Case:
    def __init__(self, variant, ny=1, fmt=None, ndim=2, B=2, H=16, W=16, D=1, Cin=64, Cout=64, cout_pad=None, taps="3x3",
                 force_bn=0, cluster=0, msub=0, max_ctas=0, tile_w=0, want_ny=0, band=None, pad=0, o_base=MARGIN, nsplit=None):
        f = [int(v) for v in variant.split("_")]
        self.variant = variant
        self.bn, self.cl, self.ms, self.split, self.half = f[:5]
        self.raw = len(f) > 5 and f[5] == 1
        self.ny = ny
        self.fmt = (2 if self.split else 0) if fmt is None else fmt
        self.ndim, self.B, self.H, self.W, self.D, self.Cin, self.Cout = ndim, B, H, W, D, Cin, Cout
        self.cout_pad = cout_pad or Cout
        self.taps = taps
        self.force_bn, self.cluster, self.msub, self.max_ctas, self.tile_w, self.want_ny = (force_bn, cluster, msub, max_ctas,
                                                                                         tile_w, want_ny)
        self.band = band            # (Cin, Cout, z stride) per depth of a depth-folded 3^3 conv3d
        self.pad, self.o_base, self.nsplit = pad, o_base, nsplit
        self.epi = ("none", "none", "32") if self.raw else None
        if band is not None:        # the GEMM of rn_conv3d_banded_same: x [B,H,W,D*bc], N = Do*bo output channels
            bc, bo, sz = band
            zo_n = 128 // bo
            self.kblocks = (((zo_n - 1) * sz + 3) * bc + 63) // 64
            self.Do = -(-D // sz)
            self.pz = max((self.Do - 1) * sz + 3 - D, 0) // 2
            self.Cin = self.kblocks * 64
            self.cout_pad = self.Do * bo
            self.Cout = Cout or self.cout_pad
            self.force_bn = 128

    def id(self):
        return self.variant + ("" if self.fmt != 1 else "_bf16")

    def col(self, n):
        if self.nsplit is None:
            return n
        ns, nhi = self.nsplit
        return (n // ns) * nhi + n % ns

    def ox(self):
        return self.col(self.Cout - 1) + 1 + self.pad

    def vec_ok(self):
        return self.ox() % 8 == 0 and self.o_base % 8 == 0

    def paths(self):
        """Store paths of the epilogue this case runs: 16-column chunks with every column valid on 16-byte aligned rows
        take the vector path, the others the scalar one."""
        p = set()
        if self.vec_ok() and self.Cout >= 16:
            p.add("vector")
        if not self.vec_ok() or self.Cout % 16 != 0:
            p.add("scalar")
        return p


CASES = [
    # ---- fast mode (fp16): N tiles 256 .. 16, clusters, M sub-tiles
    Case("256_1_1_0_0", B=2, H=20, W=24, Cin=128, Cout=250, cout_pad=256, max_ctas=7, pad=6),
    Case("256_2_1_0_0", ndim=3, B=2, H=5, W=6, D=6, Cin=32, Cout=244, cout_pad=256, taps="3^3", cluster=2, max_ctas=5, pad=4),
    Case("256_4_1_0_0", B=4, H=12, W=16, Cin=128, Cout=256, taps="1x1", cluster=4, max_ctas=7, pad=8),
    Case("128_1_1_0_0", B=2, H=18, W=20, Cin=16, Cout=100, cout_pad=128, msub=1, pad=4),
    Case("128_2_1_0_0", B=2, H=16, W=32, Cin=64, Cout=380, cout_pad=384, taps="1x1", force_bn=128, cluster=2, msub=1, pad=4),
    Case("128_4_1_0_0", ny=3, B=2, H=16, W=30, Cin=32, Cout=120, cout_pad=128, cluster=4, msub=1, want_ny=3, max_ctas=6),
    Case("128_1_2_0_0", ny=3, B=2, H=22, W=16, Cin=32, Cout=120, cout_pad=128, msub=2, want_ny=3, pad=8),
    Case("128_2_2_0_0", B=2, H=18, W=24, Cin=32, Cout=200, cout_pad=256, taps="1x1", force_bn=128, cluster=2, msub=2, pad=0),
    Case("128_4_2_0_0", B=4, H=40, W=16, Cin=16, Cout=124, cout_pad=128, cluster=4, msub=2, max_ctas=10, pad=4),
    Case("64_1_1_0_0", B=3, H=9, W=20, Cin=32, Cout=44, cout_pad=64, taps="1x1", msub=1, max_ctas=4, pad=4),
    Case("64_1_2_0_0", ny=3, B=2, H=20, W=16, Cin=64, Cout=64, msub=2, want_ny=3, nsplit=(32, 40), pad=8),
    Case("32_1_1_0_0", B=2, H=11, W=13, Cin=16, Cout=90, cout_pad=96, msub=1),
    Case("32_1_2_0_0", B=2, H=18, W=24, Cin=64, Cout=30, cout_pad=32, taps="1x1", msub=2, pad=2, max_ctas=5),
    Case("16_1_1_0_0", ny=3, B=2, H=12, W=20, Cin=32, Cout=46, cout_pad=48, msub=1, want_ny=3, pad=2),
    Case("16_1_2_0_0", B=2, H=36, W=8, Cin=16, Cout=13, cout_pad=16, taps="2x2", msub=2),
    # ---- exact mode (fp16 hi/lo pairs): single CTAs
    Case("256_1_1_1_0", B=2, H=12, W=20, Cin=64, Cout=252, cout_pad=256, pad=4, max_ctas=5),
    Case("128_1_1_1_0", ndim=3, B=2, H=5, W=6, D=6, Cin=32, Cout=120, cout_pad=128, taps="2^3", pad=8),
    Case("128_1_2_1_0", ny=3, B=2, H=20, W=16, Cin=32, Cout=116, cout_pad=256, force_bn=128, msub=2, want_ny=3, pad=4),
    Case("64_1_1_1_0", B=2, H=10, W=12, Cin=16, Cout=60, cout_pad=64, taps="1x1", msub=1, pad=4),
    Case("64_1_2_1_0", ny=3, B=2, H=26, W=16, Cin=32, Cout=64, msub=2, want_ny=3, nsplit=(32, 48), pad=0, max_ctas=3),
    Case("32_1_1_1_0", B=2, H=9, W=10, Cin=64, Cout=90, cout_pad=96, taps="1x1", msub=1),
    Case("32_1_2_1_0", B=2, H=17, W=16, Cin=32, Cout=24, cout_pad=32, msub=2, pad=0),
    Case("16_1_1_1_0", B=2, H=7, W=9, Cin=16, Cout=44, cout_pad=48, msub=1, pad=4),
    Case("16_1_2_1_0", ny=3, B=2, H=20, W=16, Cin=64, Cout=3, cout_pad=16, msub=2, want_ny=3),
    # ---- depth-folded 3^3 conv3d (banded filter, N tile 128, half-tile K blocks): band = (Cin, Cout, z stride) per depth
    Case("128_1_1_0_1", ny=3, B=2, H=10, W=12, D=8, band=(32, 32, 1), Cout=0, msub=1, want_ny=3),
    Case("128_2_1_0_1", ny=3, B=2, H=8, W=16, D=15, band=(16, 16, 2), Cout=0, cluster=2, msub=1, want_ny=3, pad=8, max_ctas=3),
    Case("128_4_1_0_1", ny=3, B=2, H=16, W=16, D=3, band=(64, 128, 1), Cout=0, cluster=4, msub=1, want_ny=3, o_base=MARGIN + 3),
    Case("128_1_2_0_1", B=2, H=20, W=16, D=4, band=(32, 32, 1), Cout=120, msub=2, pad=8),
    Case("128_2_2_0_1", B=2, H=24, W=16, D=8, band=(8, 16, 1), Cout=0, cluster=2, msub=2, max_ctas=5),
    Case("128_4_2_0_1", B=4, H=20, W=16, D=8, band=(16, 32, 2), Cout=116, cluster=4, msub=2, pad=4),
    Case("128_1_1_1_1", ny=3, B=2, H=10, W=12, D=4, band=(32, 32, 1), Cout=0, msub=1, want_ny=3, pad=8),
    Case("128_1_2_1_1", B=2, H=20, W=16, D=16, band=(16, 16, 2), Cout=124, msub=2, pad=4),
    # ---- raw fp32 output (no bias): the exact-mode per-position GEMM of the Winograd convs, here a 3-D image
    Case("256_1_1_1_0_1", ndim=3, B=2, H=5, W=6, D=6, Cin=64, Cout=256, taps="1x1"),
    # ---- bf16: every non-split N tile
    Case("256_1_1_0_0", fmt=1, B=2, H=10, W=12, Cin=64, Cout=256, pad=8),
    Case("128_1_2_0_0", fmt=1, B=2, H=20, W=16, Cin=32, Cout=124, cout_pad=128, msub=2, pad=4),
    Case("64_1_1_0_0", fmt=1, ndim=3, B=2, H=4, W=6, D=5, Cin=16, Cout=60, cout_pad=64, taps="3^3", pad=4),
    Case("32_1_2_0_0", fmt=1, ny=3, B=2, H=20, W=16, Cin=64, Cout=32, msub=2, want_ny=3, o_base=MARGIN + 1),
    Case("16_1_2_0_0", fmt=1, B=2, H=18, W=24, Cin=32, Cout=13, cout_pad=16, taps="1x1", msub=2),
    Case("128_2_1_0_1", fmt=1, ny=3, B=2, H=8, W=16, D=8, band=(32, 32, 1), Cout=0, cluster=2, msub=1, want_ny=3, pad=8),
]


def _assign_epilogues():
    """Give every non-raw case one activation x residual x output row, greedily, so that every row runs on both store paths."""
    todo = {(c, p) for c in COMBOS for p in ("vector", "scalar")}
    for i, case in enumerate(c for c in CASES if not c.raw):
        paths = case.paths()
        order = COMBOS[i % len(COMBOS):] + COMBOS[:i % len(COMBOS)]         # ties: rotate, so repeats vary
        case.epi = max(order, key=lambda cb: sum((cb, p) in todo for p in paths))
        todo -= {(case.epi, p) for p in paths}


_assign_epilogues()


def test_epilogue_matrix_is_covered():
    """Host-side check of the case table: one case per built variant (plus the bf16 ones), and every activation x residual
    x output row on both the vector and the scalar store path."""
    covered = {(c.epi, p) for c in CASES if not c.raw for p in c.paths()}
    missing = {(cb, p) for cb in COMBOS for p in ("vector", "scalar")} - covered
    assert not missing, sorted(missing)
    assert len({c.variant for c in CASES if c.fmt != 1}) == 33
    assert {c.bn for c in CASES if c.fmt == 1} == {256, 128, 64, 32, 16}
    assert any(c.nsplit for c in CASES) and any(c.Cout % 8 for c in CASES) and any(c.pad for c in CASES)


# --------------------------------------------------------------------------------------------------------------- operands
def _operand(shape, fmt, g, scale=1.0, small=False):
    """(tensor the kernel reads, its float64 value).  fmt 2: [2, *shape] hi/lo planes; `small` scales half of the entries by
    1/16 so that their LO halves are fp16 subnormals."""
    v = torch.randn(shape, generator=g) * scale
    if small:
        v = torch.where(torch.rand(shape, generator=g) < 0.5, v / 16, v)
    if fmt == 0:
        t = v.half()
        return t.to(dev), t.double().to(dev)
    if fmt == 1:
        t = v.bfloat16()
        return t.to(dev), t.double().to(dev)
    hi = v.half()
    lo = (v - hi.float()).half()
    return torch.stack([hi, lo]).contiguous().to(dev), (hi.double() + lo.double()).to(dev)


class Layout:
    """Element offsets of the output (and residual) rows: o_base + b*o_b + y*o_y + x*o_x + z*o_z + col(n)."""

    def __init__(self, c):
        ox = c.ox()
        if c.ndim == 2:
            D = 1
            self.o = (c.o_base, c.H * c.W * ox, c.W * ox, ox, 0)
        else:
            D = c.D
            self.o = (c.o_base, c.H * c.W * D * ox, c.W * D * ox, D * ox, ox)
        ob, o_b, o_y, o_x, o_z = self.o
        ar = lambda n: torch.arange(n, device=dev, dtype=torch.long)
        cols = torch.tensor([c.col(n) for n in range(c.Cout)], device=dev, dtype=torch.long)
        self.idx = (ob + ar(c.B).view(-1, 1, 1, 1, 1) * o_b + ar(c.H).view(1, -1, 1, 1, 1) * o_y +
                    ar(c.W).view(1, 1, -1, 1, 1) * o_x + ar(D).view(1, 1, 1, -1, 1) * o_z + cols.view(1, 1, 1, 1, -1))
        self.total = ob + c.B * o_b + MARGIN
        flat = self.idx.reshape(-1)
        assert flat.unique().numel() == flat.numel()
        self.guard = torch.ones(self.total, device=dev, dtype=torch.bool)
        self.guard[flat] = False


def _shifted(x5, dx, dy, dz, Do, zs):
    """x5[b, y+dy, x+dx, zs*z+dz] with zeros outside, for z < Do."""
    B, H, W, D, Cn = x5.shape
    ys, xs, zz = torch.arange(H, device=dev) + dy, torch.arange(W, device=dev) + dx, torch.arange(Do, device=dev) * zs + dz
    g = x5[:, ys.clamp(0, H - 1)][:, :, xs.clamp(0, W - 1)][:, :, :, zz.clamp(0, D - 1)]
    m = (((ys >= 0) & (ys < H)).view(-1, 1, 1) & ((xs >= 0) & (xs < W)).view(1, -1, 1) & ((zz >= 0) & (zz < D)).view(1, 1, -1))
    return g * m.view(1, H, W, Do, 1)


def reference_acc(x5, taps, wt, Do=None, zs=1):
    """float64 tap-list convolution: out[b,y,x,z,n] = sum_t sum_c x5[b, y+dy_t, x+dx_t, zs*z+dz_t, c] * wt[t, n, c]."""
    Do = x5.shape[3] if Do is None else Do
    out = 0
    for t, (dx, dy, dz) in enumerate(taps):
        out = out + torch.einsum("bhwdc,nc->bhwdn", _shifted(x5, dx, dy, dz, Do, zs), wt[t])
    return out


def epilogue_ref(acc, c, bias, alpha, res):
    v = acc
    if bias is not None:
        v = v + bias
    if c.epi[0] == "prelu":
        v = v.clamp(min=0) + alpha * v.clamp(max=0)
    elif c.epi[0] == "sigmoid":
        v = 1 / (1 + torch.exp(-v))
    return v if res is None else v + res


class Setup:
    """Operands, float64 reference pieces and output layout of one case."""

    def __init__(self, c, seed):
        g = torch.Generator().manual_seed(seed)
        self.c = c
        fmt = c.fmt
        if c.band is None:
            taps = TAPS[c.taps]
            D = c.D if c.ndim == 3 else 1
            self.x, self.x64 = _operand((c.B, c.H, c.W, D, c.Cin) if c.ndim == 3 else (c.B, c.H, c.W, c.Cin), fmt, g,
                                        small=fmt == 2)
            self.x5 = self.x64.reshape(c.B, c.H, c.W, D, c.Cin)
            K = len(taps) * c.Cin
            self.w, w64 = _operand((len(taps), c.cout_pad, c.Cin), fmt, g, scale=K ** -0.5, small=fmt == 2)
            self.taps, self.wt, self.K, self.Do, self.zs = taps, w64[:, :c.Cout], K, D, 1
        else:
            from rendernet_b200 import ops
            bc, bo, sz = c.band
            self.x, self.x64 = _operand((c.B, c.H, c.W, c.D * bc), fmt, g, small=fmt == 2)
            self.x5 = self.x64.reshape(c.B, c.H, c.W, c.D, bc)
            K = 27 * bc
            wv = torch.randn((3, 3, 3, bc, bo), generator=g) * K ** -0.5
            if fmt == 2:
                wv = torch.where(torch.rand(wv.shape, generator=g) < 0.5, wv / 16, wv)
                hi = wv.half()
                w64 = hi.double() + (wv - hi.float()).half().double()
            else:
                wv = wv.half().float() if fmt == 0 else wv.bfloat16().float()
                w64 = wv.double()
            L = ops.BandedConv3d(wv, None, dtype=torch.bfloat16 if fmt == 1 else torch.float16, sz=sz, fmt=fmt)
            self.L, self.w = L, L.w
            self.taps = [(kx - 1, ky - 1, kz - c.pz) for ky in range(3) for kx in range(3) for kz in range(3)]
            self.wt = torch.stack([w64[ky, kx, kz].T for ky in range(3) for kx in range(3) for kz in range(3)]).to(dev)
            self.K, self.Do, self.zs = K, c.Do, sz
        self.lay = Layout(c)
        self.bias = None if c.raw else (torch.randn(c.cout_pad, generator=g) * 0.5).to(dev)
        self.alpha = (torch.rand(c.cout_pad, generator=g) * 2 - 0.5).to(dev)          # PReLU slopes in [-0.5, 1.5]
        self.res, self.res64 = None, None
        if c.epi[1] != "none":          # the layer's 16-bit format or fp32, NaN between the rows the epilogue reads
            n = self.lay.idx.numel()
            if c.epi[1] == "16":
                vals, v64 = _operand((n,), fmt, g, small=True)
            else:
                vals = torch.randn(n, generator=g).to(dev)
                v64 = vals.double()
            flat = self.lay.idx.reshape(-1)
            if c.epi[1] == "16" and fmt == 2:
                self.res = torch.full((2, self.lay.total), float("nan"), device=dev, dtype=torch.float16)
                self.res[:, flat] = vals
            else:
                self.res = torch.full((self.lay.total,), float("nan"), device=dev, dtype=vals.dtype)
                self.res[flat] = vals
            self.res64 = v64.view(self.lay.idx.shape)
        self.acc = self.reference_acc()

    def reference_acc(self, x5=None, taps=None):
        c = self.c
        a = reference_acc(self.x5 if x5 is None else x5, self.taps if taps is None else taps, self.wt, self.Do, self.zs)
        B, H, W = c.B, c.H, c.W
        if c.band is not None:          # [B,H,W,Do,bo] -> the folded GEMM columns n = zo*bo + co
            a = a.reshape(B, H, W, 1, -1)[..., :c.Cout]
        return a

    def reference(self, acc=None, res64=None):
        c = self.c
        b = None if self.bias is None else self.bias[:c.Cout].double()
        return epilogue_ref(self.acc if acc is None else acc, c, b, self.alpha[:c.Cout].double(),
                            self.res64 if res64 is None else res64)

    def descriptor(self, want16, want32, **over):
        c = self.c
        d = rn_conv_desc()
        d.ndim, d.B, d.H, d.W, d.D = c.ndim, c.B, c.H, c.W, (c.D if c.ndim == 3 else 1)
        d.Cin, d.Cout, d.cout_pad = c.Cin, c.Cout, c.cout_pad
        taps = TAPS[c.taps] if c.band is None else [(kx - 1, ky - 1, 0) for ky in range(3) for kx in range(3)]
        arr = (C.c_int8 * (3 * len(taps)))(*[v for t in taps for v in t])
        d.ntaps, d.taps = len(taps), C.cast(arr, C.c_void_p)
        d._taps = arr
        d.x, d.w_packed = self.x.data_ptr(), self.w.data_ptr()
        d.bias = None if self.bias is None else self.bias.data_ptr()
        d.alpha = self.alpha.data_ptr()
        d.act = ACTS.index(c.epi[0])
        d.residual = None if self.res is None else self.res.data_ptr()
        d.residual_is_f32 = 1 if c.epi[1] == "f32" else 0
        o16 = o32 = None
        if want16:
            shape = (2, self.lay.total) if c.fmt == 2 else (self.lay.total,)
            o16 = torch.full(shape, float("nan"), device=dev, dtype=torch.bfloat16 if c.fmt == 1 else torch.float16)
            d.out16 = o16.data_ptr()
        if want32:
            o32 = torch.full((self.lay.total,), float("nan"), device=dev)
            d.out32 = o32.data_ptr()
        d.o_base, d.o_b, d.o_y, d.o_x, d.o_z = self.lay.o
        if c.nsplit is not None:
            d.o_nsplit, d.o_nhi = c.nsplit
        d.fmt = c.fmt
        d.force_bn, d.max_ctas, d.cluster, d.msub, d.ny, d.tile_w = c.force_bn, c.max_ctas, c.cluster, c.msub, c.want_ny, c.tile_w
        if c.fmt == 2:
            d.x_plane, d.w_plane, d.o_plane = self.x.numel() // 2, self.w.numel() // 2, self.lay.total
        if c.band is not None:
            bc, bo, sz = c.band
            d.x_channels, d.a_c_base, d.a_c_ntile, d.w_banded = c.D * bc, -c.pz * bc, (128 // bo) * sz * bc, 1
            d.band_cin, d.band_cout, d.band_sz = bc, bo, sz
        for k, v in over.items():
            setattr(d, k, v)
        return d, o16, o32

    def launch(self, want16, want32, expect=None, **over):
        """Plan (pinned to `expect` = (bn, cluster, msub, ny), default the case's variant), launch, return (out16, out32)."""
        c = self.c
        d, o16, o32 = self.descriptor(want16, want32, **over)
        out = (C.c_int * 16)()
        assert lib.rn_conv_plan(C.byref(d), out, 16) == 0
        p = dict(zip(PLAN_FIELDS, out))
        want = expect or (c.bn, c.cl, c.ms, c.ny)
        assert (p["bn"], p["cluster"], p["msub"], p["ny"]) == want, f"plan {p} is not the variant {want}"
        if d.max_ctas and p["cluster"] == 1:
            assert p["grid"] < p["tiles"] and p["tiles"] % p["grid"] != 0     # CTAs run several tiles, the last round is partial
        if p["cluster"] > 1 and d.max_ctas:
            assert d.max_ctas % p["cluster"] != 0 and p["grid"] == d.max_ctas - d.max_ctas % p["cluster"]
        check(lib.rn_conv_igemm(C.byref(d), torch.cuda.current_stream().cuda_stream), "rn_conv_igemm")
        torch.cuda.synchronize()
        return o16, o32, p

    def gather(self, buf):
        """Values at the output positions; asserts that every guard element still holds its NaN."""
        planes = buf.view(-1, self.lay.total)
        for q in planes:
            assert bool(torch.isnan(q[self.lay.guard]).all()), "a store landed outside the output rows"
        vals = planes[:, self.lay.idx.reshape(-1)]
        assert bool(torch.isfinite(vals).all()), "output elements left unwritten"
        return vals.view(-1, *self.lay.idx.shape)


def same_bits(a, b):
    """Bit equality, NaN guards included."""
    ints = {torch.float32: torch.int32, torch.float16: torch.int16, torch.bfloat16: torch.int16}
    return torch.equal(a.view(ints[a.dtype]), b.view(ints[b.dtype]))


def rel_err(got, ref):
    return float((got.double() - ref).abs().max()) / float(ref.abs().max())


def check_16bit(c, o16, o32):
    """16-bit output == the round-to-nearest of the fp32 output of the same epilogue (pairs: hi = fp16(v), lo = fp16(v - hi))."""
    if c.fmt == 2:
        hi = o32.half()
        lo = (o32 - hi.float()).half()
        assert torch.equal(o16[0], hi), "HI plane is not fp16(out32)"
        assert torch.equal(o16[1], lo), "LO plane is not fp16(out32 - hi)"
    else:
        assert torch.equal(o16[0], o32.half() if c.fmt == 0 else o32.bfloat16())


def run_case(c, seed):
    s = Setup(c, seed)
    out = c.epi[2]
    if out == "16":             # out16 alone; its fp32 twin comes from a second launch with out32 alone
        o16, _, p = s.launch(True, False)
        _, o32, _ = s.launch(False, True)
    else:
        o16, o32, p = s.launch(out == "both", True)
    v32 = s.gather(o32)[0]
    if out != "32":
        check_16bit(c, s.gather(o16), v32)
    return s, v32, p


@pytest.mark.gpu
@pytest.mark.parametrize("c", CASES, ids=[c.id() for c in CASES])
def test_variant(c):
    s, v32, p = run_case(c, seed=CASES.index(c) + 1)
    err = rel_err(v32, s.reference())
    print(f"{c.id()}: epilogue {c.epi}, paths {sorted(c.paths())}, K = {s.K}: out32 error {err:.2e} of max |ref| "
          f"(bar {bar(s.K):.1e})")
    assert err <= bar(s.K), f"{c.id()}: out32 error {err:.2e} > bar {bar(s.K):.2e}"
    if c.fmt == 2 and c.band is None:
        lo = s.x[1]
        sub = ((lo != 0) & (lo.float().abs() < 2.0 ** -14)).float().mean()
        assert float(sub) > 0.2            # LO halves that are fp16 subnormals are part of the operands


@pytest.mark.gpu
def test_banded_descriptor_matches_the_wrapper():
    """The banded cases above fill the descriptor themselves (strided outputs, guards); it must be the one
    rn_conv3d_banded_same builds: the same bits as ops.conv3d_banded on a plain output."""
    from rendernet_b200 import ops
    c = Case("128_1_1_0_1", ny=3, B=2, H=10, W=12, D=8, band=(32, 32, 1), Cout=0, msub=1, want_ny=3)
    c.epi = ("prelu", "none", "32")
    s = Setup(c, seed=99)
    L = s.L                     # the wrapper expands a per-channel bias and slope over the output depths
    L.bias = s.bias[:32].clone()
    al = s.alpha[:32].clone()
    s.bias.copy_(L.bias.repeat(c.D))
    s.alpha.copy_(al.repeat(c.D))
    _, o32, _ = s.launch(False, True)
    got = s.gather(o32)[0].reshape(c.B, c.H, c.W, c.D, 32)
    y = ops.conv3d_banded(s.x.view(c.B, c.H, c.W, c.D, 32), L, act="prelu", alpha=al, want16=False, want32=True,
                          tune=dict(msub=1))
    assert torch.equal(y, got)


BIT_IDENTICAL = {
    # banded: cluster 1 / 2 / 4 (halo sharing on), msub 1 / 2 (off); every case: a few CTAs that run several tiles each / one
    # CTA per tile
    "banded": (Case("128_1_1_0_1", ny=3, B=4, H=16, W=16, D=8, band=(32, 32, 1), Cout=0, msub=1, want_ny=3),
               [dict(cluster=c, expect=(128, c, 1, 3)) for c in (2, 4)] + [dict(max_ctas=5, expect=(128, 1, 1, 3))]),
    "banded_msub": (Case("128_1_1_0_1", B=2, H=20, W=16, D=8, band=(32, 32, 1), Cout=0, msub=1),
                    [dict(msub=2, expect=(128, 1, 2, 1)), dict(msub=2, cluster=2, expect=(128, 2, 2, 1)),
                     dict(max_ctas=5, expect=(128, 1, 1, 1))]),
    "banded_exact": (Case("128_1_1_1_1", B=2, H=20, W=16, D=4, band=(32, 32, 1), Cout=0, msub=1),
                     [dict(msub=2, expect=(128, 1, 2, 1)), dict(max_ctas=5, expect=(128, 1, 1, 1))]),
    "split_bn64": (Case("64_1_1_1_0", ny=3, B=2, H=26, W=16, Cin=32, Cout=60, cout_pad=64, msub=1, want_ny=3),
                   [dict(msub=2, expect=(64, 1, 2, 3)), dict(max_ctas=3, expect=(64, 1, 1, 3))]),
    "split_bn16": (Case("16_1_1_1_0", B=3, H=18, W=24, Cin=16, Cout=13, cout_pad=16, msub=1),
                   [dict(msub=2, expect=(16, 1, 2, 1)), dict(max_ctas=4, expect=(16, 1, 1, 1))]),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(BIT_IDENTICAL))
def test_same_accumulation_order_same_bits(name):
    """Cluster size, M sub-tiles and the CTA count change which CTA computes a tile, never the order of its sums: the same
    bits, also for the banded and exact-mode variants (tests/test_gpu_kernels.py covers the plain fast-mode ones)."""
    c, others = BIT_IDENTICAL[name]
    c.epi = ("prelu", "16", "both")
    s = Setup(c, seed=7)
    o16, o32, _ = s.launch(True, True)
    for kw in others:
        kw = dict(kw)
        expect = kw.pop("expect")
        p16, p32, _ = s.launch(True, True, expect=expect, **kw)
        assert same_bits(p32, o32) and same_bits(p16, o16), f"{name}: {kw}"
    assert rel_err(s.gather(o32)[0], s.reference()) <= bar(s.K)


@pytest.mark.gpu
def test_bars_discriminate():
    """The checks fail against a reference that is subtly wrong: the LO plane of x dropped, one tap shifted by one pixel,
    the residual's LO plane taken from its HI plane (an epilogue reading o_plane = 0), a 16-bit output without its LO
    plane.  Measured on the H100 (K = 288, bar 2.5e-6): 8.2e-5, 0.20 and 0.45 of max |ref|."""
    c = Case("128_1_2_1_0", ny=3, B=2, H=20, W=16, Cin=32, Cout=116, cout_pad=256, force_bn=128, msub=2, want_ny=3, pad=4)
    c.epi = ("none", "16", "both")
    s = Setup(c, seed=5)
    o16, o32, _ = s.launch(True, True)
    v32 = s.gather(o32)[0]
    assert rel_err(v32, s.reference()) <= bar(s.K)
    hi_x = s.x[0].double().reshape(s.x5.shape)
    e_lo = rel_err(v32, s.reference(acc=s.reference_acc(x5=hi_x)))
    taps = list(s.taps)
    taps[4] = (taps[4][0] + 1,) + tuple(taps[4][1:])
    e_tap = rel_err(v32, s.reference(acc=s.reference_acc(taps=taps)))
    res_hi = s.res[0][s.lay.idx.reshape(-1)].double().view(s.lay.idx.shape)
    e_res = rel_err(v32, s.reference(res64=2 * res_hi))
    print(f"x LO plane dropped: {e_lo:.2e}; tap 4 shifted by one pixel: {e_tap:.2e}; residual LO = HI: {e_res:.2e} "
          f"(bar {bar(s.K):.1e})")
    assert min(e_lo, e_tap, e_res) > 10 * bar(s.K)
    v16 = s.gather(o16)
    assert bool((v16[1] != 0).any())      # a dropped LO plane (all zeros) would fail check_16bit


@pytest.mark.gpu
def test_conv_igemm_raw_helper_exact_residual_and_raw_output():
    """ops.conv_igemm_raw: an exact-mode hi/lo residual with an fp32 output alone (the LO plane's offset comes from the
    residual), and bias = None (the raw fp32 sums) on a ragged position image."""
    from rendernet_b200 import ops
    g = torch.Generator().manual_seed(11)
    B, H, W, Cin, Cout = 2, 9, 17, 64, 256
    x, x64 = _operand((B, H, W, Cin), 2, g, small=True)
    w, w64 = _operand((1, Cout, Cin), 2, g, scale=Cin ** -0.5, small=True)
    acc = reference_acc(x64.unsqueeze(3), [(0, 0, 0)], w64)[:, :, :, 0]
    res, r64 = _operand((B, H, W, Cout), 2, g, small=True)
    bias = torch.zeros(Cout, device=dev)
    y = torch.full((B, H, W, Cout), float("nan"), device=dev)
    ops.conv_igemm_raw(ops.Split16(x), ops.Split16(w), bias, [(0, 0, 0)], 2, B, H, W, 1, Cin, Cout, Cout, out32=y,
                       residual=ops.Split16(res), fmt=2)
    assert rel_err(y, acc + r64) <= bar(Cin)
    buf = torch.full((MARGIN + B * H * W * Cout + MARGIN,), float("nan"), device=dev)
    o = (MARGIN, H * W * Cout, W * Cout, Cout, 0)
    ops.conv_igemm_raw(ops.Split16(x), ops.Split16(w), None, [(0, 0, 0)], 2, B, H, W, 1, Cin, Cout, Cout, out32=buf, o=o, fmt=2)
    assert bool(torch.isnan(buf[:MARGIN]).all()) and bool(torch.isnan(buf[-MARGIN:]).all())
    assert rel_err(buf[MARGIN:-MARGIN].view(B, H, W, Cout), acc) <= bar(Cin)
