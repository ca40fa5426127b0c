"""Host-side logic of fine-tuning the face-reconstruction shape decoder, on the CPU: the walk's new branches in
rendernet_b200/backward.py (a conv_f32 record with ELU / sigmoid, the FC without activation) run with torch emulations of the
CUDA entry points' documented semantics (include/rendernet_b200.h) against torch.autograd through the oracle's layers; the npz
key <-> TF name map of the decoder's 12 variables; nn.ShapeDecoder's argument checks; and the argument checks of the C entry
rn_conv3d_f32_weight_grad (pointers that are never dereferenced).  The kernels themselves are checked on the GPU
(tests/test_gpu_shape_decoder_training.py)."""
import types

import numpy as np
import pytest
import torch

from oracle import rendernet_oracle as orc
from oracle.shape_decoder import CONV_LAYERS, elu, init_shape_decoder_weights
from rendernet_b200 import ops
from rendernet_b200.backward import ShapeDecoderGradients


# ------------------------------------------------------------------------------------------- emulations of the C-ABI semantics
def emu_act_backward_f32(g, y, act):
    """rn_act_backward_f32: ELU y < 0 ? g (y + 1) : g; sigmoid g y (1 - y)."""
    return torch.where(y < 0, g * (y + 1), g) if act == "elu" else g * y * (1 - y)


def emu_conv3d_f32_weight_grad(x, gz, stride, transposed):
    """rn_conv3d_f32_weight_grad: dw, db of sum(gz * conv(x; w) + b), in float64."""
    s = (int(stride),) * 3
    cin, cout = int(x.shape[-1]), int(gz.shape[-1])
    w = torch.zeros((4, 4, 4, cout, cin) if transposed else (4, 4, 4, cin, cout), dtype=torch.float64, requires_grad=True)
    b = torch.zeros(cout, dtype=torch.float64, requires_grad=True)
    f = orc.conv3d_transpose if transposed else orc.conv3d
    (f(x.double(), w, b, s, dtype=torch.float64) * gz.double()).sum().backward()
    return w.grad.float(), b.grad.float()


def emu_conv3d_f32(x, w, bias, stride, transposed, act=None):
    """rn_conv3d_f32 without bias / activation."""
    f = orc.conv3d_transpose if transposed else orc.conv3d
    return f(x, w, None, (int(stride),) * 3, dtype=torch.float64).float()


def emu_fully_connected_param_grad(x, gy, z, alpha, want_gz=False):
    """rn_fully_connected_param_grad with z = alpha = NULL: gz = gy, dW = x^T gy, db = sum_b gy."""
    assert z is None and alpha is None
    return (gy if want_gz else None), (x.double().T @ gy.double()).float(), gy.double().sum(0).float(), None


@pytest.fixture
def emulated_ops(monkeypatch):
    monkeypatch.setattr(ops, "act_backward_f32", emu_act_backward_f32)
    monkeypatch.setattr(ops, "conv3d_f32_weight_grad", emu_conv3d_f32_weight_grad)
    monkeypatch.setattr(ops, "conv3d_f32", emu_conv3d_f32)
    monkeypatch.setattr(ops, "fully_connected_param_grad", emu_fully_connected_param_grad)
    monkeypatch.setattr(ops, "fully_connected_backward_data", lambda g, w: (g.double() @ w.double().T).float())


def _named(t, name):
    t._rn_name = name
    return t


def _rel(got, want):
    return float((got.double() - want.double()).abs().max() / want.double().abs().max())


def _fake():
    f = types.SimpleNamespace(weight_grads={}, _w32=lambda w: w)
    f._f32_conv_weight_step = lambda *a: ShapeDecoderGradients._f32_conv_weight_step(f, *a)
    f._fc_weight_step = lambda *a: ShapeDecoderGradients._fc_weight_step(f, *a)
    return f


@pytest.mark.parametrize("act,stride,xshape,wshape", [("elu", 2, (2, 3, 4, 3, 12), (4, 4, 4, 8, 12)),
                                                      ("sigmoid", 1, (2, 5, 4, 6, 8), (4, 4, 4, 1, 8))])
def test_conv_f32_record_weight_gradients(emulated_ops, act, stride, xshape, wshape):
    """y = act(conv3d_transpose(x) + b), act ELU (g_conv1..4) or sigmoid (g_conv5): dW, db and dx from dL/dy and the stored
    output vs autograd through the oracle's conv3d_transpose."""
    rng = np.random.default_rng(stride)
    x = torch.tensor(rng.standard_normal(xshape).astype(np.float32), requires_grad=True)
    w = torch.tensor((rng.standard_normal(wshape) * 0.2).astype(np.float32), requires_grad=True)
    b = torch.tensor(rng.standard_normal(wshape[3]).astype(np.float32) * 0.1, requires_grad=True)
    z = orc.conv3d_transpose(x, w, b, (stride,) * 3)
    y = elu(z) if act == "elu" else torch.sigmoid(z)
    G = torch.from_numpy(rng.standard_normal(tuple(y.shape)).astype(np.float32))
    (y * G).sum().backward()
    fake = _fake()
    xd = x.detach()
    rec = dict(op="conv_f32", act=act, transposed=True, stride=stride, x=xd, y=y.detach(), alpha=None,
               w=_named(w.detach().clone(), "w"), b=_named(b.detach().clone(), "b"))
    grads = {}
    ShapeDecoderGradients._decoder_weight_step(fake, rec, G, grads)
    wg = fake.weight_grads
    assert tuple(wg["w"].shape) == wshape and tuple(wg["b"].shape) == (wshape[3],)
    errs = {k: _rel(wg[k], t.grad) for k, t in (("w", w), ("b", b))}
    errs["x"] = _rel(grads[xd.data_ptr()], x.grad)
    assert max(errs.values()) < 2e-5, errs


@pytest.mark.parametrize("want_dx", [False, True])
def test_fc_record_without_activation(emulated_ops, want_dx):
    """g_gc1: y = x W + b, no activation: dW and db vs autograd; dL/dx only when asked for."""
    rng = np.random.default_rng(4)
    B, K, N = 3, 200, 256
    x = torch.tensor(rng.standard_normal((B, K)).astype(np.float32), requires_grad=True)
    w = torch.tensor((rng.standard_normal((K, N)) * 0.05).astype(np.float32), requires_grad=True)
    b = torch.tensor(rng.standard_normal(N).astype(np.float32), requires_grad=True)
    y = orc.fully_connected(x, w, b)
    G = torch.from_numpy(rng.standard_normal((B, N)).astype(np.float32))
    (y * G).sum().backward()
    fake = _fake()
    xd = x.detach()
    rec = dict(op="fc", act=None, alpha=None, x=xd, y=y.detach(), w=_named(w.detach().clone(), "w"),
               b=_named(b.detach().clone(), "b"))
    grads = {}
    ShapeDecoderGradients._decoder_weight_step(fake, rec, G, grads, want_dx=want_dx)
    assert _rel(fake.weight_grads["w"], w.grad) < 2e-5 and _rel(fake.weight_grads["b"], b.grad) < 2e-5
    if want_dx:
        assert _rel(grads[xd.data_ptr()], x.grad) < 2e-5
    else:
        assert not grads


def test_layers_without_a_weight_gradient_path_still_refuse():
    """A thin conv without a PReLU slope and a conv_f32 with another activation have no weight-gradient path."""
    with pytest.raises(NotImplementedError):
        ShapeDecoderGradients._decoder_weight_step(_fake(), dict(op="conv_small", act=None, alpha=None, w=None, b=None, x=None),
                                                   None, {})
    with pytest.raises(NotImplementedError):
        ShapeDecoderGradients._decoder_weight_step(_fake(), dict(op="conv_f32", act="relu", alpha=None, w=None, b=None, x=None),
                                                   None, {})


# ------------------------------------------------------------------------------------------- names and argument checks
def test_decoder_npz_keys_and_tf_names_round_trip():
    """The 12 decoder variables: npz key = the TF name's npz spelling (tfcompat._npz_key), the keys of the oracle's weights,
    distinct parameter keys "params.<tf name>" that map back; the fixed shapes are those of the oracle's filters."""
    from rendernet_b200.Reconstruct_RenderNet_Face import DECODER_VARIABLES
    from rendernet_b200.nn import param_key, tf_name_of
    from rendernet_b200.tfcompat import _npz_key
    W = init_shape_decoder_weights(seed=0)
    assert len(DECODER_VARIABLES) == 12
    assert sorted(k for _, k, _ in DECODER_VARIABLES) == sorted(W)
    for tf_name, key, shape in DECODER_VARIABLES:
        assert _npz_key(tf_name) == key
        assert tf_name_of(param_key(tf_name)) == tf_name
        assert shape is None or tuple(W[key].shape) == shape
    assert len({param_key(t) for t, _, _ in DECODER_VARIABLES}) == 12
    assert {k for _, k, s in DECODER_VARIABLES if s is not None} == {n + sfx for n, _, _ in CONV_LAYERS
                                                                     for sfx in ("_weights", "_biases")}


def test_shape_decoder_checks_its_arguments_before_the_device():
    from rendernet_b200.nn import ShapeDecoder
    W = init_shape_decoder_weights(seed=0)
    with pytest.raises(TypeError):
        ShapeDecoder(W, trainable="yes")
    with pytest.raises(TypeError):
        ShapeDecoder([("g_conv5_weights", W["g_conv5_weights"])])
    Wm = dict(W)
    del Wm["g_conv4_g_conv4_biases"]
    with pytest.raises(KeyError, match="g_conv4_g_conv4_biases"):
        ShapeDecoder(Wm, trainable=True)
    Wb = dict(W, g_conv2_g_conv2_weights=np.zeros((4, 4, 4, 128, 64), np.float32))
    with pytest.raises(ValueError, match="g_conv2_g_conv2_weights"):
        ShapeDecoder(Wb)


def test_conv3d_f32_weight_grad_c_entry_checks_its_arguments():
    from rendernet_b200._lib import lib
    fake = 16                                               # never dereferenced: every call below is refused on its arguments
    args = dict(x=fake, gz=fake, dw=fake, db=fake, work=fake, B=5, H=32, W=32, D=32, Cin=32, Ho=64, Wo=64, Do=64, Cout=16, k=4,
                s=2, tr=1)

    def call(**kw):
        a = dict(args, **kw)
        return lib.rn_conv3d_f32_weight_grad(a["x"], a["gz"], a["dw"], a["db"], a["work"], a["B"], a["H"], a["W"], a["D"],
                                             a["Cin"], a["Ho"], a["Wo"], a["Do"], a["Cout"], a["k"], a["s"], a["tr"], None)
    assert call(x=None) == -1 and call(gz=None) == -1 and call(dw=None) == -1 and call(db=None) == -1
    assert call(k=3) == -1
    assert call(B=33) == -1 and call(B=0) == -1
    assert call(Cin=0) == -1 and call(Cout=513) == -1
    assert call(s=3) == -2
    assert call(Ho=32) == -2 and call(Do=63) == -2              # gz is not the layer's output grid
    assert call(work=None) == -4
    for B in (1, 5, 32):
        for name, shape, s in CONV_LAYERS:
            side = {256: 4, 128: 8, 64: 16, 32: 32, 16: 64}[shape[4]]
            assert lib.rn_conv3d_f32_weight_grad_workspace(B, side, side, side, shape[4], shape[3], s, 1) > 0, (name, B)
    assert lib.rn_conv3d_f32_weight_grad_workspace(33, 4, 4, 4, 256, 128, 2, 1) < 0
    # the FC entry: z, alpha and dalpha are NULL together (no activation) or not at all
    fc = lambda z, a, da: lib.rn_fully_connected_param_grad(fake, fake, z, a, None, fake, fake, da, 2, 200, 16384, None)  # noqa: E731
    assert fc(None, fake, None) == -1 and fc(fake, None, fake) == -1 and fc(None, None, fake) == -1
