"""The exact mode's filter exponent on the host (DESIGN.md §4): the rule that chooses s, that a filter scaled by a power of two
packs to the same bits, the ctypes tables of the rn_*_scaled companions against the header, and the launch planner's check of
w_unscale.  No GPU needed: ops.filter_scales / exact_filter run on CPU tensors as they run on the device."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from rendernet_b200 import ops
from rendernet_b200._lib import SIGNATURES, lib, rn_conv_desc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COMPANIONS = ("rn_conv2d_same", "rn_conv3d_same", "rn_conv3d_banded_same", "rn_conv3d_sliced_same", "rn_winograd_out",
              "rn_conv2d_winograd", "rn_conv2d_transpose_same", "rn_conv2d_transpose_s2_merged", "rn_conv2d_transpose_s1_xfold")


def _split_np(w: torch.Tensor):
    """The exact mode's fp16 hi/lo pair of an fp32 tensor (what rn_pack_* store), as raw bits."""
    hi = w.half()
    lo = (w - hi.float()).half()
    return hi.view(torch.int16), lo.view(torch.int16)


def _exponent(w) -> int:
    up, down = ops.filter_scales(w)
    s = int(np.log2(float(up)))
    assert float(up) == 2.0 ** s and float(down) == 2.0 ** -s
    return s


def test_exponent_rule_is_wino4_exponent_of_max_abs():
    vals = [2.0 ** e for e in range(-60, 40)] + [2.0 ** e * f for e in range(-30, 20) for f in (0.75, 1.0 - 2 ** -24, 1.0 + 2 ** -23)]
    vals += list(np.random.default_rng(0).lognormal(-5, 4, 200))
    for m in vals:
        w = torch.tensor([[m * 0.5, -m], [0.25 * m, 0.0]], dtype=torch.float32)
        s = _exponent(w)
        assert s == ops.wino4_exponent(float(torch.tensor(m, dtype=torch.float32))), m
        top = float(w.abs().max()) * 2.0 ** s
        assert 2.0 ** 11 < top <= 2.0 ** 12 or abs(s) == 100, (m, s, top)
    assert _exponent(torch.zeros(3, 3)) == 100                                   # any s keeps a zero filter zero
    for bad in (float("inf"), float("nan")):
        assert abs(_exponent(torch.tensor([1.0, bad]))) == 100                  # finite scales: the outputs say inf / NaN
    assert _exponent(torch.tensor([1e-38])) == 100                              # clamped like wino4_exponent
    assert _exponent(torch.tensor([3e38])) == -100


@pytest.mark.parametrize("k", [-20, -12, -8, -1, 1, 6])
def test_filter_scaled_by_a_power_of_two_packs_to_the_same_bits(k):
    g = torch.Generator().manual_seed(3 + k)
    w = torch.randn(3, 3, 64, 32, generator=g) * 0.01
    w[0, 0, :4] *= 1e-3                                       # a few entries far below the rest
    p0, u0 = ops.exact_filter(w, 2)
    pk, uk = ops.exact_filter(w * 2.0 ** k, 2)
    assert torch.equal(p0, pk)
    assert all(torch.equal(a, b) for a, b in zip(_split_np(p0), _split_np(pk)))
    assert float(u0) == 2.0 ** -_exponent(w) and float(uk) == float(u0) * 2.0 ** k
    assert torch.equal(p0 * u0, w)                             # 2^s w, undone exactly
    # the point of it: every entry within 2^14 of the largest keeps ~22 significant bits in its hi/lo pair, where unscaled
    # the LO halves of this xavier-sized filter are fp16 subnormals with an absolute step of 2^-25
    def pair_rel_err(v):
        hi = v.half().float()
        return ((v.double() - hi.double() - (v - hi).half().double()).abs() / v.double().abs()).nan_to_num(0.0)
    big = p0.abs() >= p0.abs().max() * 2.0 ** -14
    assert float(pair_rel_err(p0)[big].max()) <= 2.0 ** -22
    assert float(pair_rel_err(w)[big].max()) > 2.0 ** -16


def test_single_16bit_formats_and_the_switch_leave_the_filter_alone(monkeypatch):
    w = torch.randn(4, 4) * 1e-4
    for fmt in (0, 1):
        p, u = ops.exact_filter(w, fmt)
        assert p is w and u is None
    monkeypatch.setattr(ops, "FILTER_EXPONENT", False)
    p, u = ops.exact_filter(w, 2)
    assert p is w and u is None


_CTYPE = {"int": C.c_int, "long long": C.c_longlong, "float": C.c_float}


def _prototype(hdr: str, name: str):
    """[(ctypes type, parameter name)] of `name`'s declaration in the header."""
    m = re.search(r"\bint\s+" + name + r"\s*\(([^;]*?)\);", hdr, re.S)
    assert m, name
    out = []
    for p in m.group(1).split(","):
        p = " ".join(p.split())
        pname = re.findall(r"[A-Za-z_0-9]+$", p)[0]
        ctype = p[: -len(pname)].strip()
        if "*" in ctype:
            out.append(("ptr", pname))
        else:
            out.append((_CTYPE[ctype.replace("const ", "")], pname))
    return out


def _same_kind(ct, declared) -> bool:
    if declared == "ptr":
        return ct is C.c_void_p or issubclass(ct, C._Pointer)
    return ct is declared


@pytest.mark.parametrize("name", COMPANIONS)
def test_companion_tables_match_the_header(name):
    hdr = open(os.path.join(ROOT, "include", "rendernet_b200.h")).read()
    plain, scaled = _prototype(hdr, name), _prototype(hdr, name + "_scaled")
    at = [p for _, p in scaled].index("w_unscale")
    assert scaled[at][0] == "ptr" and at in (1, 2)
    assert [t for t, _ in scaled[:at] + scaled[at + 1:]] == [t for t, _ in plain]      # only grows, by one pointer
    for decl in (plain, scaled):
        args = SIGNATURES[name if decl is plain else name + "_scaled"][1]
        assert len(args) == len(decl)
        for ct, (t, pname) in zip(args, decl):
            assert _same_kind(ct, t), (name, pname, ct, t)
    assert rn_conv_desc._fields_[-1] == ("w_unscale", C.c_void_p)


def _desc(fmt, bias=True):
    taps = [(kx - 1, ky - 1, 0) for ky in range(3) for kx in range(3)]
    d = rn_conv_desc()
    d.ndim, d.B, d.H, d.W, d.D = 2, 1, 16, 16, 1
    d.Cin, d.Cout, d.cout_pad, d.ntaps = 64, 64, 64, len(taps)
    arr = (C.c_int8 * (3 * len(taps)))(*[v for t in taps for v in t])
    d.taps, d._taps = C.cast(arr, C.c_void_p), arr
    d.x = d.w_packed = d.out32 = 0x10000                      # rn_conv_plan never dereferences pointers
    d.bias = 0x10000 if bias else None
    d.o_b, d.o_y, d.o_x = 16 * 16 * 64, 16 * 64, 64
    d.fmt = fmt
    if fmt == 2:
        d.x_plane = d.w_plane = d.o_plane = 8
    return d


def test_plan_takes_w_unscale_in_the_exact_epilogue_only():
    out = (C.c_int * 16)()
    for fmt in (0, 1, 2):
        assert lib.rn_conv_plan(C.byref(_desc(fmt)), out, 16) == 0
    d = _desc(2)
    d.w_unscale = 0x20000
    assert lib.rn_conv_plan(C.byref(d), out, 16) == 0
    for fmt in (0, 1):
        d = _desc(fmt)
        d.w_unscale = 0x20000
        assert lib.rn_conv_plan(C.byref(d), out, 16) == -26
    d = _desc(2, bias=False)                                   # the raw fp32 sums have no epilogue to apply it in
    d.w_unscale = 0x20000
    assert lib.rn_conv_plan(C.byref(d), out, 16) == -26
