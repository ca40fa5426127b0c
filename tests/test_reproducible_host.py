"""Host tests of the fixed-order twins' plumbing (DESIGN §8b), no GPU: the fixed-point exponent of the resampler twins (its
overflow bound and resolution over every binade of fp32), which C entry point each wrapper calls with
torch.use_deterministic_algorithms off and on (a recording stand-in for the library; CPU tensors stand in for device memory, and
the stand-in never touches them), and the ops without a twin raising or warning under the flag.  The flag is process-global:
the `flag` fixture restores it, warn_only included."""
from fractions import Fraction

import numpy as np
import pytest
import torch

from rendernet_b200 import ops
from rendernet_b200._lib import lib


@pytest.fixture
def flag():
    was, warn_only = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    yield torch.use_deterministic_algorithms
    torch.use_deterministic_algorithms(was, warn_only=warn_only)


# ------------------------------------------------------------------------------------------------ fixed-point exponent
def _probe_values():
    f32 = np.float32
    vals = [f32(0.0), np.nextafter(f32(0), f32(1)), f32(2.0 ** -140), f32(1.17549421e-38), np.finfo(f32).tiny,
            np.finfo(f32).max]
    for e in range(-149, 128):
        p = f32(2.0 ** e)
        vals += [p, np.nextafter(p, f32(0)), f32(p * f32(1.5)) if np.isfinite(p * f32(1.5)) else p]
    return sorted({float(v) for v in vals})


@pytest.mark.parametrize("new_size", [1, 2, 16, 32, 100, 128, 256])
def test_fixed_point_exponent_never_overflows(new_size):
    """Every sample point adds one contribution |w g| <= max|G| to each of its 8 corners, so a corner's int64 sum is bounded by
    new_size^3 rounded contributions: that bound stays below 2^63 for every max|G| from 0 through subnormals to FLT_MAX, and
    the resolution 2^-k stays within 2^(L - 61) max|G| (2^L >= new_size^3), under 2^-40 max|G| at new_size = 128."""
    n3 = new_size ** 3
    L = max(0, (n3 - 1).bit_length())
    for m in _probe_values():
        k = lib.rn_fixed_point_exponent(m, new_size)
        if m == 0.0:
            assert k == 0
            continue
        q = Fraction(m) * Fraction(2) ** k                      # the largest scaled contribution, exactly
        c = round(q)                                          # rounded to an integer (ties either way: bounded by ceil)
        assert n3 * (c + 1) < 2 ** 63, (m, k)
        assert q >= Fraction(2) ** (61 - L), (m, k)          # resolution: 2^-k <= max|G| 2^(L - 61)
        assert -1022 <= k <= 1023 and -1022 <= -k <= 1023    # 2^k and 2^-k are normal doubles
    if new_size == 128:
        assert lib.rn_fixed_point_exponent(1.0, 128) == 40


def test_fixed_point_exponent_nonfinite():
    for v in (float("inf"), float("nan")):
        assert lib.rn_fixed_point_exponent(v, 128) == 0


# ------------------------------------------------------------------------------------------------ which entry point runs
class _Spy:
    """Stands in for the ctypes library: records (name, args) and returns 0 (64 bytes for workspace queries)."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def fn(*args):
            self.calls.append((name, args))
            return 64 if name.endswith("_workspace") else 0
        return fn

    def names(self):
        return [n for n, _ in self.calls]


@pytest.fixture
def spy(monkeypatch):
    s = _Spy()
    monkeypatch.setattr(ops, "lib", s)
    monkeypatch.setattr(ops, "_cuda", lambda t, dtype=None: t.contiguous())
    monkeypatch.setattr(ops, "_stream", lambda: 0)
    return s


def _t(*shape, dtype=torch.float32):
    return torch.rand(shape, dtype=dtype)


def _phong_args():
    n = _t(2, 4, 8, 3)
    return n, _t(2, 4, 8, 3), _t(2, 4, 8, 3)


def _run_twinned(spy):
    """Calls the six twinned wrappers once each; returns the tensors they were handed and produced."""
    vox, minv, g = _t(2, 8, 8, 8, 1), _t(2, 3, 4), _t(2, 16, 16, 16, 1)
    r = {"resample": (vox, minv, g, ops.resample_backward(vox, minv, g, True))}
    tex, g5 = _t(2, 8, 8, 8, 4), _t(2, 16, 16, 16, 5)
    r["resample5"] = (vox, tex, minv, g5, ops.resample5_backward(vox, tex, minv, g5))
    a, n, tgt = _phong_args()
    light = torch.tensor([[0.3, 0.4, 1.0]])
    r["recon"] = (a, n, tgt, ops.phong_recon_loss_grad(a, n, tgt, light, torch.ones(1, 3)))
    r["composite"] = (a, tgt, ops.phong_composite_loss_grad(a, tgt, light))
    r["shade"] = (n, a, ops.phong_shade_backward(n, tgt, light, albedo=a))
    r["items"] = (a, tgt, ops.image_loss_grad_items(a, tgt))
    return r


TWINNED = ["rn_resample_backward_f32", "rn_resample5_backward_f32", "rn_phong_recon_loss_grad", "rn_phong_composite_loss_grad",
           "rn_phong_shade_backward", "rn_image_loss_grad_items"]


def test_flag_off_calls_todays_entry_points(spy, flag):
    flag(False)
    r = _run_twinned(spy)
    assert spy.names() == TWINNED
    args = dict(spy.calls)
    vox, minv, g, (dvox, dminv) = r["resample"]
    assert args["rn_resample_backward_f32"] == (vox.data_ptr(), minv.data_ptr(), g.data_ptr(), dvox.data_ptr(), dminv.data_ptr(),
                                                2, 1, 8, 16, 1, 0)
    assert not dvox.any() and not dminv.any()                 # accumulated into: zeroed first
    vox, tex, minv, g5, (dv, dt, dm) = r["resample5"]
    assert args["rn_resample5_backward_f32"] == (vox.data_ptr(), tex.data_ptr(), minv.data_ptr(), g5.data_ptr(), dv.data_ptr(),
                                                 dt.data_ptr(), dm.data_ptr(), 2, 8, 16, 0)
    a, n, tgt, (loss, da, dn, dl) = r["recon"]
    ra = args["rn_phong_recon_loss_grad"]
    assert ra[:3] == (a.data_ptr(), n.data_ptr(), tgt.data_ptr()) and ra[5:9] == (0.0, 1.0, 0, 1)
    assert ra[9:] == (loss.data_ptr(), da.data_ptr(), dn.data_ptr(), dl.data_ptr(), 2, 4, 8, 0)
    assert not loss.any() and not dl.any()
    img, tgt, (loss, dimg, dl) = r["composite"]
    ca = args["rn_phong_composite_loss_grad"]
    assert ca[:2] == (img.data_ptr(), tgt.data_ptr()) and ca[4:] == (pytest.approx(0.1), pytest.approx(0.9), 0, 1, loss.data_ptr(),
                                                                       dimg.data_ptr(), dl.data_ptr(), 2, 4, 8, 0)
    n, a, (dn, da, dl) = r["shade"]
    sa = args["rn_phong_shade_backward"]
    assert sa[:2] == (n.data_ptr(), a.data_ptr()) and sa[4:9] == (0.0, 1.0, 1, 1, 1)
    assert sa[10:] == (dn.data_ptr(), da.data_ptr(), dl.data_ptr(), 2, 4, 8, 0)
    img, tgt, (loss, dimg) = r["items"]
    assert args["rn_image_loss_grad_items"] == (img.data_ptr(), tgt.data_ptr(), dimg.data_ptr(), loss.data_ptr(), 32, 3, 2, 0, 0)


def test_flag_on_calls_the_twins(spy, flag):
    flag(True)
    r = _run_twinned(spy)
    twins = [n for n in spy.names() if not n.endswith("_workspace")]
    assert twins == [n.replace("_f32", "") + "_fixed" + ("_f32" if n.endswith("_f32") else "") for n in TWINNED]
    assert all(n.endswith("_workspace") for n in spy.names() if n not in twins)
    args = dict(spy.calls)
    vox, minv, g, (dvox, dminv) = r["resample"]
    assert args["rn_resample_backward_fixed_f32"][:11] == (vox.data_ptr(), minv.data_ptr(), g.data_ptr(), dvox.data_ptr(),
                                                          dminv.data_ptr(), 2, 1, 8, 16, 1, args["rn_resample_backward_fixed_f32"][10])
    assert args["rn_resample_backward_fixed_f32"][11:] == (64, 0)
    assert args["rn_resample_backward_fixed_workspace"] == (2, 1, 8, 16, 1)
    assert args["rn_resample5_backward_fixed_workspace"] == (2, 8, 16, 1, 1)
    assert args["rn_image_loss_grad_items_fixed_workspace"] == (32, 3, 2)


def test_flag_on_warn_only_still_calls_the_twins(spy, flag):
    flag(True, warn_only=True)
    _run_twinned(spy)
    assert "rn_resample_backward_fixed_f32" in spy.names() and "rn_resample_backward_f32" not in spy.names()


def test_shade_backward_without_light_grad_needs_no_workspace(spy, flag):
    flag(True)
    n, a, g = _phong_args()
    ops.phong_shade_backward(n, g, (0.0, 0.0, 1.0), want_light_grad=False)
    (name, args), = spy.calls
    assert name == "rn_phong_shade_backward_fixed" and args[12] is None and args[-3:] == (None, 0, 0)


# ------------------------------------------------------------------------------------------------ ops without a twin
def _untwinned():
    h = dict(dtype=torch.float16)
    vox, tex, minv = _t(1, 8, 8, 8, 1), _t(1, 8, 8, 8, 4), _t(1, 3, 4)
    return {
        "rn_conv2d_weight_grad": lambda: ops.conv2d_weight_grad(_t(1, 4, 4, 8, **h), _t(1, 4, 4, 16, **h), 3, 3),
        "rn_conv_weight_grad_direct": lambda: ops.conv_weight_grad_direct(_t(1, 4, 4, 8, **h), _t(1, 4, 4, 8, **h), (3, 3),
                                                                          (1, 1), (1, 1)),
        "rn_bias_grad_16": lambda: ops.bias_grad(_t(64, 16, **h)),
        "rn_prelu_alpha_grad": lambda: ops.prelu_alpha_grad(_t(64, 16, **h), _t(64, 16, **h)),
        "rn_prelu_grad_f32": lambda: ops.prelu_grad_f32(_t(64, 4), _t(64, 4), _t(4)),
        "rn_image_loss_grad": lambda: ops.image_loss_grad(_t(2, 4, 4, 3), _t(2, 4, 4, 3)),
        "rn_resample5_backward_window_f32": lambda: ops.resample5_backward(vox, tex, minv, _t(1, 16, 16, 16, 5),
                                                                           window=(0, 0, 16, 16)),
    }


@pytest.mark.parametrize("op", sorted(_untwinned()))
def test_untwinned_op_raises_under_flag(spy, flag, op):
    flag(True)
    with pytest.raises(RuntimeError, match=op):
        _untwinned()[op]()
    assert op not in spy.names()


@pytest.mark.parametrize("op", sorted(_untwinned()))
def test_untwinned_op_warns_under_warn_only(spy, flag, op):
    flag(True, warn_only=True)
    with pytest.warns(UserWarning, match=op):
        _untwinned()[op]()
    assert spy.names()[-1] == op


@pytest.mark.parametrize("op", sorted(_untwinned()))
def test_untwinned_op_silent_without_flag(spy, flag, op, recwarn):
    flag(False)
    _untwinned()[op]()
    assert spy.names()[-1] == op and not [w for w in recwarn if op in str(w.message)]
