"""Host-side logic of the training step, on the CPU: the weight-gradient formulas of rendernet_b200/backward.py
(`_weight_grads_of`: which tensor is the coarse / fine operand of the strided correlation, the TF SAME pads, the filter-layout
permutes, the block-diagonal extraction of the depth-folded tensor-core gradient) are run with torch emulations of the CUDA
entry points' documented semantics (include/rendernet_b200.h) and compared with torch.autograd through the oracle's layers.
The kernels themselves are checked against the same autograd on the GPU (tests/test_gpu_training.py).  Also: the dropout mask
generator (host restatement exported by the library), the learning-rate schedule, TF's Adam formulation."""
import types
import zlib

import numpy as np
import pytest
import torch

from oracle import rendernet_oracle as orc
from rendernet_b200 import ops


# ------------------------------------------------------------------------------------------- emulations of the C-ABI semantics
def emu_conv_weight_grad_direct(P, Q, ksize, stride, pad, Ca=None, Cb=None, scale=1.0):
    """dW[tap][a][b] = scale * sum_pos P[pos][a] * Q[pos*stride + tap - pad][b], zero outside Q (rn_conv_weight_grad_direct)."""
    P, Q = P.double(), Q.double()
    if P.dim() == 4:
        P, Q = P[:, None], Q[:, None]
        ksize, stride, pad = (1,) + tuple(ksize), (1,) + tuple(stride), (0,) + tuple(pad)
        squeeze = True
    else:
        squeeze = False
    Ca, Cb = Ca or P.shape[-1], Cb or Q.shape[-1]
    P, Q = P[..., :Ca], Q[..., :Cb]
    n = [P.shape[1 + i] for i in range(3)]
    hi = [max(0, (n[i] - 1) * stride[i] + ksize[i] - 1 - pad[i] - (Q.shape[1 + i] - 1)) for i in range(3)]
    Qp = torch.nn.functional.pad(Q, (0, 0, pad[2], hi[2], pad[1], hi[1], pad[0], hi[0]))
    dW = torch.zeros(tuple(ksize) + (Ca, Cb), dtype=torch.float64)
    for kz in range(ksize[0]):
        for ky in range(ksize[1]):
            for kx in range(ksize[2]):
                q = Qp[:, kz:kz + (n[0] - 1) * stride[0] + 1:stride[0], ky:ky + (n[1] - 1) * stride[1] + 1:stride[1],
                       kx:kx + (n[2] - 1) * stride[2] + 1:stride[2]]
                dW[kz, ky, kx] = torch.einsum("nzyxa,nzyxb->ab", P, q)
    dW = dW * scale
    return (dW[0] if squeeze else dW).float()


def emu_conv2d_weight_grad(x, g, kh, kw):
    """dw[ky][kx][ci][co] = sum x[b, y+ky-pb, x+kx-pb, ci] g[b,y,x,co], pb = (k-1)//2 (rn_conv2d_weight_grad)."""
    d = emu_conv_weight_grad_direct(g, x, (kh, kw), (1, 1), ((kh - 1) // 2, (kw - 1) // 2))
    return d.permute(0, 1, 3, 2).contiguous()


def emu_bias_grad(g):
    return g.double().reshape(-1, g.shape[-1]).sum(0).float()


@pytest.fixture
def emulated_ops(monkeypatch):
    monkeypatch.setattr(ops, "conv_weight_grad_direct", emu_conv_weight_grad_direct)
    monkeypatch.setattr(ops, "conv2d_weight_grad", emu_conv2d_weight_grad)
    monkeypatch.setattr(ops, "bias_grad", emu_bias_grad)


def _named(t, name):
    t._rn_name = name
    return t


def _run_case(kind, wshape, xshape, stride, tensor_core, g_pad=0, resample=False):
    """One layer: autograd through the oracle's layer vs backward._weight_grads_of with the emulated kernels."""
    from rendernet_b200.backward import ShaderInputGradients
    rng = np.random.default_rng(zlib.crc32(repr((kind, wshape, stride)).encode()))
    x = torch.from_numpy(rng.standard_normal(xshape).astype(np.float32))
    w = torch.tensor((rng.standard_normal(wshape) * 0.2).astype(np.float32), requires_grad=True)
    cout = wshape[2] if kind == "conv2d_transpose" else wshape[-1]
    b = torch.zeros(cout, requires_grad=True)
    if kind == "conv2d":
        y = orc.conv2d(x, w, b)
        st = 1
    elif kind == "conv3d":
        st3 = tuple(stride) if isinstance(stride, (tuple, list)) else ((1, 1, 1) if stride == 1 else (1, 1, 2))
        y = orc.conv3d(x, w, b, st3)
        st = stride
    else:
        y = orc.conv2d_transpose(x, w, b, (stride, stride))
        st = stride
    G = torch.from_numpy(rng.standard_normal(tuple(y.shape)).astype(np.float32))
    (y * G).sum().backward()
    g = G
    if g_pad:                                       # e_conv11: the gradient tensor carries zero-padded channels
        g = torch.zeros(tuple(G.shape[:-1]) + (g_pad,))
        g[..., :cout] = G
    fake = types.SimpleNamespace(weight_grads={}, new_size=xshape[1])
    wv, bv = _named(w.detach().clone(), "w"), _named(b.detach().clone(), "b")
    if resample:
        rec = dict(op="resample_conv1", w=wv, b=bv, stride=list(stride), grid=types.SimpleNamespace(voxel=None, minv=None))
        import rendernet_b200.ops as O
        O_resample = O.resample
        O.resample = lambda vox, minv, n, tr: x
        try:
            ShaderInputGradients._weight_grads_of(fake, rec, g, 1.0, tensor_core)
        finally:
            O.resample = O_resample
    else:
        rec = dict(op="conv", kind=kind, stride=st, x=x, w=wv, b=bv)
        ShaderInputGradients._weight_grads_of(fake, rec, g, 1.0, tensor_core)
    dw, db = fake.weight_grads["w"], fake.weight_grads["b"]
    assert tuple(dw.shape) == tuple(w.shape) and tuple(db.shape) == tuple(b.shape)
    e_w = float((dw - w.grad).abs().max() / w.grad.abs().max())
    e_b = float((db - b.grad).abs().max() / b.grad.abs().max())
    assert e_w < 2e-5 and e_b < 2e-5, (kind, wshape, stride, tensor_core, e_w, e_b)


@pytest.mark.parametrize("case", [
    ("conv2d", (3, 3, 8, 16), (2, 10, 12, 8), 1, False),             # thin conv2d -> direct kernel
    ("conv2d", (4, 4, 8, 8), (1, 9, 8, 8), 1, False),                # 4x4: asymmetric SAME pads (1 before, 2 after)
    ("conv2d", (4, 4, 128, 128), (1, 6, 6, 128), 1, True),           # wide conv2d -> tensor-core kernel's layout
    ("conv2d", (1, 1, 128, 256), (2, 5, 5, 128), 1, True),           # projection unit
    ("conv3d", (3, 3, 3, 8, 16), (1, 8, 8, 8, 8), 2, False),         # e_conv2: stride [1,1,2]
    ("conv3d", (3, 3, 3, 16, 16), (1, 6, 5, 8, 16), 1, True),        # res1: depth-folded (D*C = 128) tensor-core gradient + band extraction
    ("conv3d", (3, 3, 3, 16, 32), (1, 5, 6, 8, 16), 1, True),        # e_conv3-like: Cin != Cout (D*Cin = 128, D*Cout = 256)
    ("conv3d", (3, 3, 3, 16, 16), (1, 6, 5, 8, 16), 1, False),       # the same layer through the direct kernel
    ("conv2d_transpose", (4, 4, 16, 32), (2, 6, 7, 32), 2, False),   # e_conv7/8/9: stride 2
    ("conv2d_transpose", (4, 4, 16, 16), (1, 8, 8, 16), 1, False),   # e_conv7_1 / e_conv10: stride 1
])
def test_weight_gradient_formulas_match_autograd(emulated_ops, case):
    _run_case(*case)


def test_weight_gradient_of_output_layer_with_padded_gradient_channels(emulated_ops):
    _run_case("conv2d_transpose", (4, 4, 3, 16), (1, 8, 8, 16), 1, False, g_pad=16)


def test_weight_gradient_of_fused_resample_conv1(emulated_ops):
    _run_case("conv3d", (5, 5, 5, 1, 8), (1, 16, 16, 16, 1), (2, 2, 2), False, resample=True)


# ------------------------------------------------------------------------------------------- dropout masks, schedule, Adam
def test_dropout_mask_generator_is_deterministic_and_unbiased():
    m1 = ops.dropout_mask_host(1 << 20, 0.75, seed=7, salt=3)
    m2 = ops.dropout_mask_host(1 << 20, 0.75, seed=7, salt=3)
    m3 = ops.dropout_mask_host(1 << 20, 0.75, seed=7, salt=4)
    assert np.array_equal(m1, m2) and not np.array_equal(m1, m3)
    assert abs(m1.mean() - 0.75) < 2e-3 and abs(m3.mean() - 0.75) < 2e-3
    assert abs(np.mean(m1[:-1] & m1[1:]) - 0.75 ** 2) < 3e-3              # neighbours uncorrelated
    assert abs(np.mean(m1 & m3) - 0.75 ** 2) < 3e-3                       # calls uncorrelated
    assert ops.dropout_mask_host(4096, 1.0, 1, 1).all()
    # independent restatement of the documented generator (rn_dropout_hash.h: SplitMix64 finaliser, top 32 bits)
    i = np.arange(1000, dtype=np.uint64)
    with np.errstate(over="ignore"):
        key = (np.uint64(7) << np.uint64(32)) | np.uint64(3)
        z = (i + np.uint64(1)) * np.uint64(0x9E3779B97F4A7C15) + key * np.uint64(0xD1B54A32D192ED03)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
    want = ((z >> np.uint64(32)) < np.uint64(int(0.75 * 2 ** 32))).astype(np.uint8)
    assert np.array_equal(m1[:1000], want)


def test_same_pad_before_matches_oracle():
    for n in (7, 8, 64, 128):
        for k in (1, 3, 4, 5):
            for s in (1, 2):
                assert ops.same_pad_before(n, k, s) == orc.same_pads(n, k, s)[0]


def test_trainer_needs_cuda_and_schedule_formula():
    from rendernet_b200.training import ShaderTrainer
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError):
            ShaderTrainer(None, 1)
    sched = ShaderTrainer.learning_rate
    fake = types.SimpleNamespace(e_eta=1e-5, decay_rate=0.96, decay_steps=100000, global_step=0)
    assert sched(fake, 0) == 1e-5 and sched(fake, 99999) == 1e-5
    assert abs(sched(fake, 100000) - 0.96e-5) < 1e-18 and abs(sched(fake, 250000) - 1e-5 * 0.96 ** 2) < 1e-18


def test_dropout_is_refused_outside_the_training_path_and_gradient_allreduce_is_a_noop_without_a_group():
    """tf.nn.dropout(keep < 1) without a seeded store is the inference path misused: loud error, nothing launched; keep == 1 is
    the identity.  all_reduce_gradients without an initialised process group returns the gradients untouched."""
    from rendernet_b200 import tfcompat as tf
    from rendernet_b200.parallel import all_reduce_gradients
    x = torch.ones(2, 3)
    assert tf.nn.dropout(x, 1.0) is x
    with pytest.raises(NotImplementedError):
        tf.nn.dropout(x, 0.75)
    g = {"a": torch.ones(3), "b": torch.zeros(2, 2)}
    assert all_reduce_gradients(g) is g and torch.equal(g["a"], torch.ones(3))


def test_frozen_kink_prelu_reproduces_the_oracle_with_its_own_masks():
    """oracle.frozen_kinks, which the whole-network gradient tests use to give the oracle the device's PReLU branches: on a
    narrow Shader net, masks taken from the oracle's own pre-activations reproduce its image and the autograd gradients of all
    variables bit for bit (the two forms differ only at a pre-activation of exactly 0, where there is none here), and a mask of
    the wrong shape or a slope it does not know is an error."""
    from oracle.frozen_kinks import kink_flips, prelu_kinks
    W = orc.init_shader_weights(seed=4, width=8, depth=8, alpha_range=(-0.2, 0.3), bias_jitter=0.05)   # 64 features: e_conv10 -> 1
    x = torch.from_numpy(np.random.default_rng(0).random((2, 8, 8, 32, 1)).astype(np.float32))
    G = torch.from_numpy(np.random.default_rng(1).standard_normal((2, 32, 32, 3)).astype(np.float32))

    def run(masks=None, record=None):
        Wt = {n: torch.tensor(v, requires_grad=True) for n, v in W.items()}
        with prelu_kinks(Wt, masks=masks, record=record):
            img = orc.rendernet_shader(x, Wt)
        grads = torch.autograd.grad((img * G).sum(), [Wt[n] for n in sorted(Wt)])
        return img.detach(), dict(zip(sorted(Wt), grads))

    plain = orc.prelu
    signs = {}
    img0, g0 = run(record=signs)
    assert len(signs) == 36                                   # every PReLU of the graph, projection unit included
    plain_img = orc.rendernet_shader(x, W)
    assert torch.equal(img0, plain_img)                       # recording changes nothing
    img1, g1 = run(masks=signs)
    assert kink_flips(signs, signs) == (0, sum(int(m.numel()) for m in signs.values()))
    assert torch.equal(img1, img0)
    assert all(torch.equal(g1[n], g0[n]) for n in g0), [n for n in g0 if not torch.equal(g1[n], g0[n])][:3]
    flipped = {n: m.clone() for n, m in signs.items()}
    flipped["encoder/e_conv5/alpha"].view(-1)[:7] ^= True
    img2, g2 = run(masks=flipped)
    assert not torch.equal(img2, img0) or not torch.equal(g2["encoder/e_conv5/alpha"], g0["encoder/e_conv5/alpha"])
    bad = dict(signs)
    bad["encoder/e_conv3/alpha"] = bad["encoder/e_conv3/alpha"][:1]
    with pytest.raises(ValueError):
        run(masks=bad)
    with pytest.raises(KeyError):
        with prelu_kinks({}, masks={}):
            orc.rendernet_shader(x, W)
    assert orc.prelu is plain
