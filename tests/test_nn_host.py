"""CPU tests of rendernet_b200.nn: the TF name <-> parameter key map and the argument checks that run before any launch."""
import numpy as np
import pytest
import torch

from oracle import rendernet_oracle as orc


@pytest.mark.parametrize("net,count", [("shader", 166), ("texture", 186)])
def test_parameter_keys_round_trip(net, count):
    """Every TF variable name of the Shader (166) and the Texture+Normal network (186) is a parameter key of an nn.ParameterDict
    whose state_dict key is "params.<tf name>", unique, and maps back to the name."""
    from rendernet_b200.nn import param_key, tf_name_of
    W = orc.init_shader_weights(seed=1) if net == "shader" else orc.init_texture_weights(seed=1)
    assert len(W) == count
    m = torch.nn.Module()
    m.params = torch.nn.ParameterDict({k: torch.nn.Parameter(torch.zeros(1)) for k in W})
    keys = list(m.state_dict())
    assert len(set(keys)) == count
    assert sorted(keys) == sorted(param_key(k) for k in W)
    assert sorted(tf_name_of(k) for k in keys) == sorted(W)
    with pytest.raises(KeyError):
        tf_name_of("encoder/e_conv1/e_conv1/weights")


def _bare(cls):
    """A module without its gradient objects: forward's argument checks run before anything touches the device."""
    m = cls.__new__(cls)
    torch.nn.Module.__init__(m)
    return m


def test_shader_renderer_refuses_malformed_input():
    from rendernet_b200.nn import ShaderRenderer
    m = _bare(ShaderRenderer)
    vp = np.zeros((2, 3), np.float32)
    with pytest.raises(TypeError):
        m(torch.zeros(2, 64, 64, 64, 1), vp)                                # voxels on the host
    with pytest.raises(TypeError):
        m(np.zeros((2, 64, 64, 64, 1), np.float32), vp)


def test_texture_renderer_refuses_pretrained_training_and_bad_models():
    from rendernet_b200.nn import TextureRenderer
    with pytest.raises(ValueError, match="constant"):
        TextureRenderer({}, model="pretrained", trainable=True)
    with pytest.raises(ValueError):
        TextureRenderer(None, model="opengl")
    m = _bare(TextureRenderer)
    with pytest.raises(TypeError):
        m(torch.zeros(1, 64, 64, 64, 1), np.zeros((1, 199), np.float32), np.zeros((1, 3), np.float32))


def test_voxel_and_row_shape_checks():
    """Shapes are checked before the device: a malformed grid raises ValueError wherever it lives, a well-formed one on the
    host TypeError."""
    from rendernet_b200 import nn as rnn
    for shape in ((2, 64, 64, 32, 1), (2, 64, 64, 64, 3), (64, 64, 64), (0, 64, 64, 64)):
        with pytest.raises(ValueError):
            rnn._check_voxels(torch.zeros(shape))
    for shape in ((2, 64, 64, 64, 1), (2, 64, 64, 64)):
        with pytest.raises(TypeError, match="CUDA"):
            rnn._check_voxels(torch.zeros(shape))
    with pytest.raises(TypeError, match="float32"):
        rnn._check_voxels(torch.zeros((1, 64, 64, 64), dtype=torch.float64))
    with pytest.raises(ValueError):
        rnn._rows(np.zeros((3, 3)), 2, 3, "view_params")
    with pytest.raises(ValueError):
        rnn._rows(torch.zeros(2, 198), 2, 199, "texture")


def test_phong_shade_refuses_bad_light_and_host_tensors():
    from rendernet_b200.nn import phong_shade
    n = torch.rand(3, 8, 8, 3)
    for ld in (torch.ones(2, 3), torch.ones(3), torch.ones(3, 4), torch.ones(1, 1, 3)):
        with pytest.raises(ValueError, match="light_dir"):
            phong_shade(n, ld)
    with pytest.raises(ValueError):
        phong_shade(torch.rand(3, 8, 8), torch.ones(1, 3))
    with pytest.raises(ValueError):
        phong_shade(n, torch.ones(1, 3), composite="opengl")
    with pytest.raises(TypeError):
        phong_shade(n, torch.ones(3, 3))                                     # the normal map on the host


def test_phong_shade_backward_c_entry_checks_its_arguments():
    from rendernet_b200._lib import RN_PHONG_TF, lib
    fake = 16                                               # never dereferenced: every call below is refused on its arguments
    args = dict(normal=fake, albedo=None, ld=fake, lc=fake, comp=RN_PHONG_TF, g=fake, dn=fake, B=1, H=4, W=4)

    def call(**kw):
        a = dict(args, **kw)
        return lib.rn_phong_shade_backward(a["normal"], a["albedo"], a["ld"], a["lc"], 0.0, 1.0, a["comp"], 1, 1, a["g"], a["dn"],
                                           None, None, a["B"], a["H"], a["W"], None)
    assert call(normal=None) == -1
    assert call(g=None) == -1
    assert call(dn=None) == -1
    assert call(comp=2) == -1
    assert call(B=0) == -1
    assert call(B=70000) == -2


def test_shape_decoder_refuses_a_latent_of_the_wrong_width():
    from rendernet_b200.nn import ShapeDecoder
    m = _bare(ShapeDecoder)
    for bad in (torch.zeros(2, 199), torch.zeros(200), torch.zeros(0, 200), np.zeros((2, 200), np.float32)):
        with pytest.raises(ValueError, match="200"):
            m(bad)
