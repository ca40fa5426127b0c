"""CPU checks of the shading entry points: malformed arguments are refused before anything reaches a device."""
import numpy as np
import pytest
import torch


def test_phong_shade_refuses_malformed_input():
    from rendernet_b200 import ops
    n = torch.rand(3, 8, 8, 3)
    with pytest.raises(ValueError):
        ops.phong_shade(n, torch.ones(2, 3))                                  # light_dir rows not in {1, B}
    with pytest.raises(ValueError):
        ops.phong_shade(n, torch.ones(3, 3), light_col=np.ones((2, 3)))
    with pytest.raises(ValueError):
        ops.phong_shade(n, torch.ones(1, 3), composite="opengl")
    with pytest.raises(ValueError):
        ops.phong_shade(n, torch.ones(1, 3), albedo=torch.rand(3, 8, 8, 1))   # albedo / normal shape mismatch
    with pytest.raises(ValueError):
        ops.phong_shade(torch.rand(3, 8, 8), torch.ones(1, 3))
    with pytest.raises(RuntimeError):                                         # well formed, but no CPU path
        ops.phong_shade(n, torch.ones(1, 3))


def test_phong_shade_c_entry_checks_its_arguments():
    from rendernet_b200._lib import RN_PHONG_TF, lib
    fake = 256                                                                # never dereferenced: the checks come first
    assert lib.rn_phong_shade(None, None, fake, fake, 0.0, 1.0, RN_PHONG_TF, 1, 1, fake, None, None, 1, 4, 4, None) == -1
    assert lib.rn_phong_shade(fake, None, fake, fake, 0.0, 1.0, 2, 1, 1, fake, None, None, 1, 4, 4, None) == -1
    assert lib.rn_phong_shade(fake, None, fake, fake, 0.0, 1.0, RN_PHONG_TF, 1, 1, None, None, None, 1, 4, 4, None) == -1
    assert lib.rn_phong_shade(fake, None, fake, fake, 0.0, 1.0, RN_PHONG_TF, 1, 1, fake, None, None, 0, 4, 4, None) == -1


def test_texture_engine_refuses_malformed_options():
    from rendernet_b200.engine import TextureRenderEngine
    L = np.array([[0.0, 0.0, 1.0]], np.float32)
    with pytest.raises(ValueError):
        TextureRenderEngine(None, 3, phong=dict(light_dir=np.ones((2, 3), np.float32)))
    with pytest.raises(ValueError):
        TextureRenderEngine(None, 3, phong=dict(light_dir=L, composite="opengl"))
    with pytest.raises(ValueError):
        TextureRenderEngine(None, 3, phong=dict(light_col=(1.0, 1.0, 1.0)))     # no light_dir
    with pytest.raises(ValueError):
        TextureRenderEngine(None, 3, phong=dict(light_dir=L, lightdir=L))        # misspelt key
    with pytest.raises(ValueError):
        TextureRenderEngine(None, 3, model="shader")
    with pytest.raises(ValueError):
        TextureRenderEngine(None, 3, model="pretrained")
