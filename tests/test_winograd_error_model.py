"""The CPU error model of the exact-mode Winograd trunk convolution (scripts/winograd_error_model.py) at the trunk's C = 1024:
F(4x4, 3x3) with the shipped points and power-of-two scales stays well inside the trunk's 2.5e-5 bar, also at |x| ~ 1e4, while
the textbook points would not.  No GPU needed."""
import pytest

from scripts.winograd_error_model import inputs, measure, variants

SHIPPED = "F(4x4) points 0, +-1, +-1/2, V/2, U 2^s (shipped)"


@pytest.mark.parametrize("scale,uniform", [(3.0, False), (1.0e4, True)])
def test_f4x4_emulated_error_at_c1024(scale, uniform):
    x, w = inputs(hw=16, C=1024, cout=8, scale=scale, seed=3, uniform=uniform)
    r = measure(x, w, **variants()[SHIPPED])
    print(f"F(4x4) emulated, |x| ~ {scale:g}: max {r['max_err']:.2e}, rel-rms {r['rel_rms']:.2e}, |V|/|x| {r['v_over_x']:.2f}")
    assert r["finite"] and r["max_err"] < 1.5e-5
    assert r["v_over_x"] <= 4.5


def test_textbook_points_are_outside_the_bar():
    x, w = inputs(hw=16, C=1024, cout=8, scale=3.0, seed=3)
    assert measure(x, w, **variants()["F(4x4) points 0, +-1, +-2"])["max_err"] > 2.5e-5
