"""Host-side logic of the Texture+Normal training step, on the CPU: the weight-gradient formulas of rendernet_b200/backward.py for
the records that only this network has -- the fused resample5 + e_conv1 record (5-channel grid re-materialised and concatenated),
and the texture decoder's fp32 layers (`_decoder_weight_step`: 3-D transposed convs at stride 1 and 2, the 4^3 conv, the FC with
its per-column PReLU) -- run with torch emulations of the CUDA entry points' documented semantics (include/rendernet_b200.h) and
compared with torch.autograd through the oracle's layers.  The kernels themselves are checked on the GPU
(tests/test_gpu_texture_training.py).  Also: `texture_dropout`, which runs the oracle's Texture+Normal forward as the
training graph (dropout at its twelve sites), for the GPU tests' references."""
import contextlib
import types
import zlib

import numpy as np
import pytest
import torch

from oracle import rendernet_oracle as orc
from rendernet_b200 import ops
from rendernet_b200.backward import TextureInputGradients

from test_training_host import emu_bias_grad, emu_conv_weight_grad_direct


# ------------------------------------------------------------------------------------------- emulations of the C-ABI semantics
def emu_fully_connected_param_grad(x, gy, z, alpha, want_gz=False):
    """rn_fully_connected_param_grad: gz = gy (z > 0 ? 1 : alpha), dW = x^T gz, db = sum_b gz, dalpha = sum_{z<0} gy z."""
    x, gy, z, a = x.double(), gy.double(), z.double(), alpha.double()
    gz = torch.where(z > 0, gy, gy * a)
    return (gz.float() if want_gz else None), (x.T @ gz).float(), gz.sum(0).float(), (gy * z * (z < 0)).sum(0).float()


def emu_prelu_grad_f32(gy, z, alpha):
    """rn_prelu_grad_f32: gz = gy (z > 0 ? 1 : alpha[c]), db[c] = sum gz, dalpha[c] = sum_{z<0} gy z."""
    C = gy.shape[-1]
    gy, z, a = gy.double(), z.double(), alpha.double()
    gz = torch.where(z > 0, gy, gy * a)
    return gz.float(), gz.reshape(-1, C).sum(0).float(), (gy * z * (z < 0)).reshape(-1, C).sum(0).float()


def emu_conv3d_small(x, w, bias, alpha, stride, transposed, want32=True):
    """rn_conv3d_small without bias / activation: TF conv3d_transpose (transposed) or conv3d, SAME."""
    s = (int(stride),) * 3
    f = orc.conv3d_transpose if transposed else orc.conv3d
    return f(x, w, None, s, dtype=torch.float64).float()


@pytest.fixture
def emulated_ops(monkeypatch):
    monkeypatch.setattr(ops, "conv_weight_grad_direct", emu_conv_weight_grad_direct)
    monkeypatch.setattr(ops, "bias_grad", emu_bias_grad)
    monkeypatch.setattr(ops, "fully_connected_param_grad", emu_fully_connected_param_grad)
    monkeypatch.setattr(ops, "prelu_grad_f32", emu_prelu_grad_f32)
    monkeypatch.setattr(ops, "conv3d_small", emu_conv3d_small)
    monkeypatch.setattr(ops, "concat_channels", lambda a, b: torch.cat([a, b], -1))


def _named(t, name):
    t._rn_name = name
    return t


def _rel(got, want):
    return float((got.double() - want.double()).abs().max() / want.double().abs().max())


def _fake():
    return types.SimpleNamespace(weight_grads={}, _alpha=lambda alpha, n: alpha, _w32=lambda w: w)


def test_resample5_conv1_weight_gradient(emulated_ops, monkeypatch):
    """e_conv1 of the Texture+Normal network (5^3 s2, 5 -> 8): the grid is the concatenation of the two resamplings; dW and db
    from g = dL/d(pre-activation) vs autograd through orc.conv3d."""
    rng = np.random.default_rng(7)
    N, B = 12, 2
    geom = torch.from_numpy(rng.standard_normal((B, N, N, N, 1)).astype(np.float32))
    tex = torch.from_numpy(rng.standard_normal((B, N, N, N, 4)).astype(np.float32))
    vox_g, vox_t = object(), object()                 # stand-ins for the voxel grids the resampler reads
    monkeypatch.setattr(ops, "resample", lambda vox, minv, n, tr: {id(vox_g): geom, id(vox_t): tex}[id(vox)])
    w = torch.tensor((rng.standard_normal((5, 5, 5, 5, 8)) * 0.1).astype(np.float32), requires_grad=True)
    b = torch.zeros(8, requires_grad=True)
    y = orc.conv3d(torch.cat([geom, tex], -1), w, b, (2, 2, 2))
    G = torch.from_numpy(rng.standard_normal(tuple(y.shape)).astype(np.float32))
    (y * G).sum().backward()
    fake = types.SimpleNamespace(weight_grads={}, new_size=N)
    grid = types.SimpleNamespace(geom=types.SimpleNamespace(voxel=vox_g), tex=types.SimpleNamespace(voxel=vox_t), minv=None)
    rec = dict(op="resample5_conv1", w=_named(w.detach().clone(), "w"), b=_named(b.detach().clone(), "b"), stride=[2, 2, 2],
               grid=grid)
    TextureInputGradients._weight_grads_of(fake, rec, G * 4.0, 0.25, True)          # g carries a loss scale of 4
    dw, db = fake.weight_grads["w"], fake.weight_grads["b"]
    assert tuple(dw.shape) == tuple(w.shape)
    assert _rel(dw, w.grad) < 2e-5 and _rel(db, b.grad) < 2e-5


DECODER_CASES = [
    # name, transposed, filter shape (TF layout), input shape, stride
    ("e_tex_conv0", True, (4, 4, 4, 4, 4), (2, 6, 5, 7, 4), 1),
    ("e_tex_conv1", True, (4, 4, 4, 8, 4), (2, 5, 6, 4, 4), 2),
    ("e_tex_conv2", False, (4, 4, 4, 8, 4), (2, 9, 8, 7, 8), 1),
]


@pytest.mark.parametrize("name,transposed,wshape,xshape,stride", DECODER_CASES)
def test_decoder_conv_weight_gradients(emulated_ops, name, transposed, wshape, xshape, stride):
    """A decoder layer y = prelu(conv(x) + b; alpha), slopes of both signs: dW, db, dalpha and dx from dL/dy and the kept
    pre-activation vs autograd through the oracle's conv3d / conv3d_transpose."""
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    x = torch.tensor(rng.standard_normal(xshape).astype(np.float32), requires_grad=True)
    w = torch.tensor((rng.standard_normal(wshape) * 0.2).astype(np.float32), requires_grad=True)
    C = wshape[3] if transposed else wshape[4]
    b = torch.tensor(rng.standard_normal(C).astype(np.float32) * 0.1, requires_grad=True)
    a = torch.tensor(rng.uniform(-0.4, 0.4, C).astype(np.float32), requires_grad=True)
    s3 = (stride,) * 3
    z = orc.conv3d_transpose(x, w, b, s3) if transposed else orc.conv3d(x, w, b, s3)
    y = orc.prelu(z, a)
    G = torch.from_numpy(rng.standard_normal(tuple(y.shape)).astype(np.float32))
    (y * G).sum().backward()
    fake = _fake()
    xd, zd = x.detach(), z.detach()
    rec = dict(op="conv_small", act="prelu", transposed=transposed, stride=stride, x=xd, y=y.detach(),
               w=_named(w.detach().clone(), "w"), b=_named(b.detach().clone(), "b"), alpha=_named(a.detach().clone(), "a"),
               rerun=lambda: zd)
    grads = {}
    TextureInputGradients._decoder_weight_step(fake, rec, G, grads)
    wg = fake.weight_grads
    assert tuple(wg["w"].shape) == wshape
    errs = {k: _rel(wg[k], t.grad) for k, t in (("w", w), ("b", b), ("a", a))}
    errs["x"] = _rel(grads[xd.data_ptr()], x.grad)
    assert max(errs.values()) < 2e-5, errs


def test_fully_connected_weight_gradients(emulated_ops):
    """e_tex_fc1 (199 -> N, per-column PReLU): dW, db, dalpha vs autograd; the texture vector's gradient is not produced."""
    rng = np.random.default_rng(3)
    B, K, N = 5, 199, 256
    x = torch.from_numpy(rng.standard_normal((B, K)).astype(np.float32))
    w = torch.tensor((rng.standard_normal((K, N)) * 0.05).astype(np.float32), requires_grad=True)
    b = torch.tensor(rng.standard_normal(N).astype(np.float32) * 0.1, requires_grad=True)
    a = torch.tensor(rng.uniform(-0.4, 0.4, N).astype(np.float32), requires_grad=True)
    z = orc.fully_connected(x, w, b)
    y = orc.prelu(z, a)
    G = torch.from_numpy(rng.standard_normal((B, N)).astype(np.float32))
    (y * G).sum().backward()
    fake = _fake()
    zd = z.detach()
    rec = dict(op="fc", act="prelu", x=x, y=y.detach(), w=_named(w.detach().clone(), "w"), b=_named(b.detach().clone(), "b"),
               alpha=_named(a.detach().clone(), "a"), rerun=lambda: zd)
    grads = {}
    TextureInputGradients._decoder_weight_step(fake, rec, G, grads)
    wg = fake.weight_grads
    assert not grads
    for k, t in (("w", w), ("b", b), ("a", a)):
        assert tuple(wg[k].shape) == tuple(t.shape) and _rel(wg[k], t.grad) < 2e-5, k


def test_decoder_weight_step_refuses_layers_without_a_prelu_slope():
    rec = dict(op="conv_small", act=None, alpha=None, w=None, b=None, x=None)
    with pytest.raises(NotImplementedError):
        TextureInputGradients._decoder_weight_step(_fake(), rec, None, {})


# ------------------------------------------------------------------------------------------- dropout in the oracle's forward
# The twelve tf.nn.dropout sites of RenderNet_Texture_Face_Normal.py:55,60,65,101,116-125,133-142, in the mirror's call order
# (rendernet_b200/RenderNet_Texture_Face_Normal.py): each follows the PReLU of these layers.
TEXTURE_DROPOUT_SITES = (["encoder/e_conv1/alpha", "encoder/e_conv2/alpha", "encoder/e_conv3/alpha", "encoder/e_conv5/alpha"]
                         + [f"encoder/{h}/e_conv{k}_{s}/alpha" for h, s in (("Image", 1), ("Normal", 2)) for k in (6, 7, 8, 9)])


@contextlib.contextmanager
def texture_dropout(W, dropout):
    """Inside the block, `orc.rendernet_texture(x, W)` runs the training graph: after the PReLU of each dropout site (identified,
    like oracle/frozen_kinks.py does, by the identity of its slope among the "/alpha" values of W) the output goes through
    dropout(call_index, tensor), call_index counting the sites in the mirror's order.  Composes with frozen_kinks.prelu_kinks
    entered first."""
    names = {id(W[n]): n for n in TEXTURE_DROPOUT_SITES}
    inner = orc.prelu
    calls = [0]

    def prelu(x, alpha, *args):
        y = inner(x, alpha, *args)
        name = names.get(id(alpha))
        if name is None:
            return y
        assert name == TEXTURE_DROPOUT_SITES[calls[0]], (name, calls[0])
        y = dropout(calls[0], y)
        calls[0] += 1
        return y

    orc.prelu = prelu
    try:
        yield calls
    finally:
        orc.prelu = inner


def test_texture_dropout_fires_twelve_times_in_mirror_order():
    """The oracle's Texture+Normal forward with texture_dropout calls the hook at e_conv1, 2, 3, 5, then e_conv6..9 of the Image
    head, then of the Normal head; an identity hook leaves the outputs unchanged, and zeroing the Image head's four sites
    changes only the image."""
    W = orc.init_texture_weights(seed=0)
    x = np.random.default_rng(1).random((1, 4, 4, 128, 5)).astype(np.float32)
    plain = orc.prelu
    seen = []

    def rec(i, t):
        seen.append((i, int(t.shape[-1])))
        return t

    img0, nrm0 = orc.rendernet_texture(x, W)
    with texture_dropout(W, rec) as calls:
        img1, nrm1 = orc.rendernet_texture(x, W)
    assert calls[0] == 12 and [i for i, _ in seen] == list(range(12))
    assert [c for _, c in seen] == [8, 16, 16, 256, 128, 64, 32, 16, 128, 64, 32, 16]
    assert torch.equal(img0, img1) and torch.equal(nrm0, nrm1)
    with texture_dropout(W, lambda i, t: t * 0.0 if 4 <= i < 8 else t):
        img2, nrm2 = orc.rendernet_texture(x, W)
    assert torch.equal(nrm2, nrm0) and not torch.equal(img2, img0)
    assert orc.prelu is plain
