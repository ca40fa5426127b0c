"""The loss-scale chooser of the 16-bit backward pass (rendernet_b200/backward.py), on the CPU: choose_loss_scale at the edges of
fp32, the loss_scale argument's modes, and which output heads _choose_scale reads.  tests/test_gpu_gradient_range.py checks on
the GPU that whole backward passes are exact under the power-of-two scales it returns."""
import math
import types

import numpy as np
import pytest
import torch

from rendernet_b200.backward import (LOSS_SCALE_TARGET, _InputGradients, _key, _loss_scale_mode, choose_loss_scale)

F32_TINY = float(np.finfo(np.float32).tiny)             # 2^-126
F32_SUB = float(np.finfo(np.float32).smallest_subnormal)  # 2^-149
F32_MAX = float(np.finfo(np.float32).max)


def _is_pow2(v):
    m, _ = math.frexp(v)
    return v > 0 and m == 0.5


@pytest.mark.parametrize("amax", [1.0, 0.25, 3.0, 4096.0, 65504.0, 1e-3, 6.1e-5, 2.5e-6, 1.1e-7, 3.2e-8, 1e-20, F32_TINY,
                                  F32_SUB, 3 * F32_SUB, 1e30, F32_MAX, math.nextafter(1.0, 2.0), math.nextafter(1.0, 0.0)])
@pytest.mark.parametrize("target", [LOSS_SCALE_TARGET, 2.0 ** 12, 2.0 ** 14, 3000.0])
def test_scale_is_the_largest_power_of_two_within_the_target(amax, target):
    """scale = 2^floor(log2(target / amax)): a power of two with scale * amax <= target < 2 scale * amax, unless the clamp to
    [2^-126, 2^126] (scale and 1 / scale normal fp32 numbers) binds, which only fp32's extreme magnitudes reach."""
    s = choose_loss_scale(amax, target)
    assert _is_pow2(s), s
    assert 2.0 ** -126 <= s <= 2.0 ** 126
    e = math.log2(s)
    if -126 < e < 126:
        assert s * amax <= target < 2 * s * amax, (amax, target, s)
    elif e == 126:
        assert 2.0 ** 126 * amax <= target                  # a subnormal amax would want a larger scale than fp32 holds
    else:
        assert 2.0 ** -126 * amax > target / 2


def test_scale_edges():
    assert choose_loss_scale(2.0 ** -20, 2.0 ** 12) == 2.0 ** 32       # exact powers of two land on the target
    assert choose_loss_scale(2.0 ** 12, 2.0 ** 12) == 1.0
    assert choose_loss_scale(math.nextafter(2.0 ** 12, 1e9), 2.0 ** 12) == 0.5
    assert choose_loss_scale(F32_SUB) == 2.0 ** 126                     # clamped
    assert choose_loss_scale(F32_MAX) == 2.0 ** math.floor(math.log2(LOSS_SCALE_TARGET) - 128)
    assert choose_loss_scale(0.0) == 1.0                                 # a zero gradient: nothing to scale
    for bad in (math.inf, -math.inf, math.nan):
        with pytest.raises(FloatingPointError):
            choose_loss_scale(bad)
    for bad in (0.0, -1.0, math.inf, math.nan):
        with pytest.raises(ValueError):
            choose_loss_scale(1.0, bad)


def test_loss_scale_modes():
    """None and "auto" choose per call; a number is a fixed scale, passed through unchanged (no rounding to a power of two)."""
    assert _loss_scale_mode(None) is None and _loss_scale_mode("auto") is None
    for v in (4096.0, 3000.0, 1, 2.0 ** -20):
        assert _loss_scale_mode(v) == float(v)
    for bad in (0.0, -4096.0, math.inf, math.nan, "fixed"):
        with pytest.raises(ValueError):
            _loss_scale_mode(bad)


def _fake(loss_scale, target=LOSS_SCALE_TARGET):
    """Two sigmoid heads (albedo, normal), a hidden PReLU layer and an fp32 decoder layer with a sigmoid (the shape decoder's
    g_conv5) on a tape of CPU tensors."""
    rng = np.random.default_rng(0)
    y1 = torch.from_numpy(rng.uniform(0.01, 0.99, (2, 4, 4, 3)).astype(np.float32))
    y2 = torch.from_numpy(rng.uniform(0.01, 0.99, (2, 4, 4, 3)).astype(np.float32))
    h = torch.zeros(2, 4, 4, 8)
    v = torch.from_numpy(rng.uniform(0.01, 0.99, (2, 8, 8, 8, 1)).astype(np.float32))
    tape = [dict(op="conv", act="prelu", y=h), dict(op="conv", act="sigmoid", y=y1), dict(op="conv", act="sigmoid", y=y2),
            dict(op="conv_f32", act="sigmoid", y=v)]
    self = types.SimpleNamespace(loss_scale=_loss_scale_mode(loss_scale), scale_target=target, tape=tape)
    return self, y1, y2, v


def test_choose_scale_reads_every_reached_sigmoid_head():
    self, y1, y2, v = _fake(None)
    g1 = torch.full(tuple(y1.shape), 1e-7)
    g2 = torch.full(tuple(y2.shape), 3e-7).reshape(2, -1)              # a reshaped view of the head, as the walk may see it
    big = torch.full(tuple(v.shape), 1e6)                                # fp32 walk: never scaled, so never read
    want = float((g2.reshape(y2.shape) * y2 * (1 - y2)).abs().max())
    got = _InputGradients._choose_scale(self, {_key(y1): g1, _key(y2): g2, _key(v): big})
    assert got == choose_loss_scale(want)
    assert _InputGradients._choose_scale(self, {_key(y1): g1}) == choose_loss_scale(float((g1 * y1 * (1 - y1)).max()))
    assert _InputGradients._choose_scale(self, {_key(v): big}) == 1.0   # no 16-bit head reached
    fixed, y1, _, _ = _fake(3000.0)
    assert _InputGradients._choose_scale(fixed, {_key(y1): torch.full(tuple(y1.shape), 1e-7)}) == 3000.0
