"""GPU parity of the training step (SURVEY §8 f-4 stage 2; RenderNet_Shader.py:154-167): every kernel of rn_train.cu against
torch / NumPy restatements, the gradients of ALL variables of the full-size network (dropout on) against torch.autograd through
the CPU oracle, and two optimiser steps against the oracle driven by the same Adam formulas."""
import math
import os
import zlib

import numpy as np
import pytest
import torch

from oracle import rendernet_oracle as orc

pytestmark = pytest.mark.gpu
dev = "cuda"


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def _rms(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.sqrt(((a - b) ** 2).mean() / max((b ** 2).mean(), 1e-300)))


def _cos(a, b):
    a, b = np.asarray(a, np.float64).ravel(), np.asarray(b, np.float64).ravel()
    return float((a * b).sum() / max(np.linalg.norm(a) * np.linalg.norm(b), 1e-300))


# ------------------------------------------------------------------------------------------------ kernels
DIRECT_CASES = [
    # kind, filter shape (TF layout), input shape, stride
    ("conv2d", (3, 3, 8, 16), (2, 20, 24, 8), 1),
    ("conv2d", (4, 4, 40, 24), (1, 17, 16, 40), 1),                 # channel counts that do not fill the 32 x 32 tile
    ("conv3d", (3, 3, 3, 8, 16), (1, 16, 16, 16, 8), (1, 1, 2)),    # e_conv2
    ("conv3d", (3, 3, 3, 32, 32), (1, 12, 10, 8, 32), (1, 1, 1)),   # res1 layer through the direct kernel
    ("conv3d", (5, 5, 5, 1, 8), (1, 32, 32, 32, 1), (2, 2, 2)),     # e_conv1 (fp32 fine operand)
    ("conv2d_transpose", (4, 4, 32, 64), (2, 12, 14, 64), 2),       # e_conv9
    ("conv2d_transpose", (4, 4, 16, 32), (1, 16, 16, 32), 1),       # e_conv10
    ("conv2d_transpose", (4, 4, 3, 16), (1, 24, 24, 16), 1),        # e_conv11: gradient padded to 16 channels
]


@pytest.mark.parametrize("kind,wshape,xshape,stride", DIRECT_CASES)
def test_direct_weight_gradient_kernel_matches_autograd(kind, wshape, xshape, stride):
    """rn_conv_weight_grad_direct driven exactly as backward._weight_grads_of drives it, vs torch.autograd through the oracle's
    layer; both 16-bit formats (exact: 2e-5 of the gradient scale; fast: fp16 operand rounding, 2e-3)."""
    from rendernet_b200 import ops
    rng = np.random.default_rng(zlib.crc32(repr((kind, wshape)).encode()))
    x = rng.standard_normal(xshape).astype(np.float32)
    w = torch.tensor((rng.standard_normal(wshape) * 0.2).astype(np.float32), requires_grad=True)
    if kind == "conv2d":
        y = orc.conv2d(x, w)
    elif kind == "conv3d":
        y = orc.conv3d(x, w, None, stride)
    else:
        y = orc.conv2d_transpose(x, w, None, (stride, stride))
    G = rng.standard_normal(tuple(y.shape)).astype(np.float32)
    (y * torch.from_numpy(G)).sum().backward()
    want = w.grad.numpy()
    for name, fmt, tol in (("exact", 2, 2e-5), ("fast", 0, 2e-3)):
        xd = torch.from_numpy(x).to(dev)
        x16 = xd if (kind == "conv3d" and wshape[0] == 5) else ops.cast_to_16(xd, fmt=fmt)        # e_conv1 reads the fp32 grid
        cout = wshape[2] if kind == "conv2d_transpose" else wshape[-1]
        Gd = torch.from_numpy(G).to(dev) * 16.0                                                     # a loss scale
        if cout < 16:                                                                               # e_conv11: 3 of 16 channels
            Gp = torch.zeros(tuple(G.shape[:-1]) + (16,), device=dev)
            Gp[..., :cout] = Gd
            Gd = Gp
        g16 = ops.cast_to_16(Gd.contiguous(), fmt=fmt)
        if kind == "conv2d":
            kh, kw, ci, co = wshape
            pad = (ops.same_pad_before(xshape[1], kh, 1), ops.same_pad_before(xshape[2], kw, 1))
            got = ops.conv_weight_grad_direct(g16, x16, (kh, kw), (1, 1), pad, Ca=co, Cb=ci, scale=1 / 16).permute(0, 1, 3, 2)
        elif kind == "conv3d":
            ks = wshape[:3]
            pad = tuple(ops.same_pad_before(xshape[1 + i], ks[i], stride[i]) for i in range(3))
            got = ops.conv_weight_grad_direct(g16, x16, ks, stride, pad, Ca=wshape[4], Cb=wshape[3], scale=1 / 16).permute(0, 1, 2, 4, 3)
        else:
            kh, kw, co, ci = wshape
            pad = (ops.same_pad_before(xshape[1] * stride, kh, stride), ops.same_pad_before(xshape[2] * stride, kw, stride))
            got = ops.conv_weight_grad_direct(x16, g16, (kh, kw), (stride, stride), pad, Ca=ci, Cb=co, scale=1 / 16).permute(0, 1, 3, 2)
        e = _rel(got.cpu().numpy(), want)
        print(f"[{name}] direct wgrad {kind} {wshape} s{stride}: rel err {e:.2e}")
        assert tuple(got.shape) == tuple(wshape) and e < tol, (name, kind, wshape, e)


def test_depth_folded_tensor_core_weight_gradient_equals_direct_kernel():
    """res1 layer, real shape (B=1, 64x64x32, 32 -> 32): the wgmma gradient of the depth-folded conv + block-diagonal extraction
    vs the direct kernel vs autograd."""
    from rendernet_b200 import ops
    from rendernet_b200.backward import ShaderInputGradients
    import types
    rng = np.random.default_rng(3)
    x = (rng.standard_normal((1, 64, 64, 32, 32)) * (rng.random((1, 64, 64, 32, 32)) < 0.5)).astype(np.float32)
    w = torch.tensor((rng.standard_normal((3, 3, 3, 32, 32)) * 0.05).astype(np.float32), requires_grad=True)
    y = orc.conv3d(x, w)
    G = rng.standard_normal(tuple(y.shape)).astype(np.float32)
    (y * torch.from_numpy(G)).sum().backward()
    want = w.grad.numpy()
    for name, fmt, tol in (("exact", 2, 5e-5), ("fast", 0, 3e-3)):
        x16 = ops.cast_to_16(torch.from_numpy(x).to(dev), fmt=fmt)
        g16 = ops.cast_to_16(torch.from_numpy(G).to(dev), fmt=fmt)
        wv = w.detach().clone()
        wv._rn_name = "w"
        out = {}
        for tc in (True, False):
            fake = types.SimpleNamespace(weight_grads={}, new_size=128)
            ShaderInputGradients._weight_grads_of(fake, dict(op="conv", kind="conv3d", stride=1, x=x16, w=wv, b=None), g16, 1.0, tc)
            out[tc] = fake.weight_grads["w"].cpu().numpy()
        e_tc, e_d, e_x = _rel(out[True], want), _rel(out[False], want), _rel(out[True], out[False])
        print(f"[{name}] res1 wgrad: tensor-core folded {e_tc:.2e}, direct {e_d:.2e}, tc vs direct {e_x:.2e}")
        assert e_tc < tol and e_d < tol


def test_prelu_alpha_gradient_dropout_loss_and_adam_kernels():
    from rendernet_b200 import ops
    from rendernet_b200 import tfcompat as tf
    rng = np.random.default_rng(9)
    # PReLU slope gradient
    z = rng.standard_normal((2, 9, 7, 5, 24)).astype(np.float32)
    g = rng.standard_normal(z.shape).astype(np.float32)
    want = (g.astype(np.float64) * np.minimum(z.astype(np.float64), 0)).reshape(-1, 24).sum(0)
    for fmt, tol in ((2, 1e-5), (0, 2e-3)):
        got = ops.prelu_alpha_grad(ops.cast_to_16(torch.from_numpy(g * 8).to(dev), fmt=fmt), ops.cast_to_16(torch.from_numpy(z).to(dev), fmt=fmt), 0.125)
        assert _rel(got.cpu().numpy(), want) < tol
    # dropout: device mask == host restatement, kept values scaled by 1/keep, and it is its own backward
    x = rng.standard_normal((3, 11, 13, 16)).astype(np.float32)
    for fmt in (2, 0):
        x16 = ops.cast_to_16(torch.from_numpy(x).to(dev), fmt=fmt)
        y = tf.to_float(ops.dropout(x16, 0.75, seed=123, salt=4)).cpu().numpy()
        mask = ops.dropout_mask_host(x.size, 0.75, 123, 4).reshape(x.shape)
        xq = tf.to_float(x16).cpu().numpy()
        assert np.array_equal(y != 0, (mask == 1) & (xq != 0))
        assert np.abs(y - xq * mask / 0.75).max() < (1e-6 if fmt == 2 else 2e-3)
    # losses
    p = rng.random((2, 32, 32, 3)).astype(np.float32)
    t = rng.random((2, 32, 32, 3)).astype(np.float32)
    pt = torch.tensor(p.astype(np.float64), requires_grad=True)
    mse = ((pt - torch.from_numpy(t).double()) ** 2).mean()
    mse.backward()
    loss, dimg = ops.image_loss_grad(torch.from_numpy(p).to(dev), torch.from_numpy(t).to(dev), "mse")
    assert abs(loss.item() - mse.item()) < 1e-6 * mse.item() and _rel(dimg.cpu().numpy(), pt.grad.numpy()) < 1e-5
    pt = torch.tensor(p.astype(np.float64), requires_grad=True)
    td = torch.from_numpy(t).double()
    bce = (-(td * torch.log(1e-6 + pt) + (1 - td) * torch.log(1e-6 + 1 - pt)).sum(dim=(1, 2, 3))).mean()
    bce.backward()
    loss, dimg = ops.image_loss_grad(torch.from_numpy(p).to(dev), torch.from_numpy(t).to(dev), "bce")
    assert abs(loss.item() - bce.item()) < 1e-5 * bce.item() and _rel(dimg.cpu().numpy(), pt.grad.numpy()) < 1e-4
    # Adam (TF formulation), three steps
    n = 5000
    p0, m0, v0 = rng.standard_normal(n).astype(np.float32), np.zeros(n, np.float32), np.zeros(n, np.float32)
    pd_, md, vd = (torch.from_numpy(a.copy()).to(dev) for a in (p0, m0, v0))
    pr, mr, vr = p0.astype(np.float64), m0.astype(np.float64), v0.astype(np.float64)
    for step in range(1, 4):
        gnp = rng.standard_normal(n).astype(np.float32)
        lr_t = 1e-3 * math.sqrt(1 - 0.999 ** step) / (1 - 0.5 ** step)
        ops.adam_step(pd_, torch.from_numpy(gnp).to(dev), md, vd, lr_t, 0.5, 0.999, 1e-8)
        mr = mr + (gnp - mr) * 0.5
        vr = vr + (gnp.astype(np.float64) ** 2 - vr) * 0.001
        pr = pr - lr_t * mr / (np.sqrt(vr) + 1e-8)
    assert np.abs(pd_.cpu().numpy() - pr).max() < 1e-5 and np.abs(md.cpu().numpy() - mr).max() < 1e-6


# ------------------------------------------------------------------------------------------------ whole network
def _scene(golden_dir):
    bv = np.load(os.path.join(golden_dir, "binvox.npz"))
    vox = np.unpackbits(bv["chair_bits"]).reshape(1, 64, 64, 64, 1).astype(np.float32)
    poses = orc.compute_pose_param(250.0, 60.0, 3.3).astype(np.float32)
    grid = orc.transform_voxel_to_match_image(orc.rotation_resampling(vox, poses)).astype(np.float32)
    # a learnable target: the object's silhouette (any occupied voxel along the depth axis), tinted per channel
    sil = (grid[0, :, :, :, 0].sum(axis=2) > 0.5).astype(np.float32)
    target = np.repeat(np.repeat(sil, 4, 0), 4, 1)[None, :, :, None] * np.array([0.9, 0.6, 0.3], np.float32)
    return vox, poses, grid, np.ascontiguousarray(target, np.float32)


def _oracle_step(grid, Wt, target, keep, seed):
    """Oracle forward (dropout masks restated on the host from the library's generator) + MSE + autograd over every variable."""
    from rendernet_b200 import ops

    def drop(call, t):
        m = ops.dropout_mask_host(t.numel(), keep, seed, call).reshape(tuple(t.shape)).astype(np.float32)
        return t * torch.from_numpy(m) / keep

    img = orc.rendernet_shader(torch.from_numpy(grid), Wt, dropout=drop if keep < 1.0 else None)
    loss = ((img - torch.from_numpy(target)) ** 2).mean()
    grads = torch.autograd.grad(loss, [Wt[n] for n in sorted(Wt)])
    return float(loss), img.detach().numpy(), dict(zip(sorted(Wt), (g.numpy() for g in grads)))


@pytest.mark.parametrize("precision", ["exact", "fast"])
def test_gradients_of_every_variable_match_oracle_autograd(golden_dir, precision):
    """Full-size Shader network, chair, B = 1, dropout keep 0.75, MSE against a random target: loss, image and dL/d(variable) for
    all 166 variables (filters, biases, PReLU slopes) vs torch.autograd through the CPU oracle with the same dropout masks.
    The per-variable bar is the gradient's direction (cosine) and norm: with a coherent (real) loss gradient the PReLU units
    that sit on opposite sides of the kink in the two implementations no longer dominate (they do for the white-noise image
    gradient of tests/test_gpu_backward.py) and the agreement is 1e-4-level in exact precision.
    Element by element, against the same oracle differentiated with the device's PReLU branches (oracle/frozen_kinks.py): every
    variable within 2.2e-4 rel-rms and 3.0e-4 max (exact) / 1.4e-3 and 1.6e-3 (fast), measured on an H100; 790 (exact) and
    41044 (fast) of the 131 M PReLU units sit on opposite sides of the kink in the two implementations."""
    from rendernet_b200.training import ShaderTrainer
    from oracle.frozen_kinks import kink_flips, prelu_kinks, tape_prelu_masks
    vox, poses, grid, target = _scene(golden_dir)
    W = orc.init_shader_weights(seed=1, alpha_range=(-0.1, 0.3), bias_jitter=0.02)     # a quarter of the slopes negative
    tr = ShaderTrainer(W, 1, precision=precision, keep_prob=0.75, seed=5)
    loss, grads = tr.loss_and_gradients(vox, poses, target)
    Wt = {n: torch.tensor(v, requires_grad=True) for n, v in W.items()}
    signs = {}
    with prelu_kinks(Wt, record=signs):
        loss_ref, img_ref, g_ref = _oracle_step(grid, Wt, target, 0.75, tr.dropout_seed(0))
    e_img = float(np.abs(tr.img.cpu().numpy() - img_ref).max())
    print(f"[{precision}] training-mode forward: image max-abs err {e_img:.2e}, loss {loss:.6f} vs {loss_ref:.6f}")
    assert e_img < (1e-3 if precision == "exact" else 5e-3)
    assert abs(loss - loss_ref) < (5e-5 if precision == "exact" else 1e-3) * loss_ref      # measured 1.5e-5 / 3e-4
    assert set(grads) == set(g_ref) and len(grads) == 166
    c_min, worst, rows = 1.0, None, []
    for n in sorted(g_ref):
        got, want = grads[n].cpu().numpy(), g_ref[n]
        assert got.shape == want.shape, n
        c, ratio = _cos(got, want), float(np.linalg.norm(got) / max(np.linalg.norm(want), 1e-30))
        rows.append((c, ratio, n))
        if c < c_min:
            c_min, worst = c, n
    rows.sort()
    for c, ratio, n in rows[:6]:
        print(f"[{precision}]   lowest cosine: {n} cos {c:.5f} norm ratio {ratio:.4f}")
    kinds = {"weights": [], "biases": [], "alpha": []}
    for c, ratio, n in rows:
        kinds[n.rsplit("/", 1)[1]].append((c, ratio))
    for k, v in kinds.items():
        print(f"[{precision}] {k}: {len(v)} variables, cosine min {min(c for c, _ in v):.5f} median {np.median([c for c, _ in v]):.5f}, "
              f"norm ratio {min(r for _, r in v):.4f}..{max(r for _, r in v):.4f}")
    bar = 0.9999 if precision == "exact" else 0.9985
    assert c_min > bar, (worst, c_min)
    assert all(abs(r - 1) < (5e-3 if precision == "exact" else 3e-2) for _, r, _ in rows)      # measured: 4e-4 / 5.4e-3
    # element-wise, against the oracle differentiated with the device's PReLU branches (frozen kinks)
    masks = tape_prelu_masks(tr.tape)
    flips, units = kink_flips(masks, signs)
    with prelu_kinks(Wt, masks=masks):
        g_f = _oracle_step(grid, Wt, target, 0.75, tr.dropout_seed(0))[2]
    errs = sorted(((_rms(grads[n].cpu().numpy(), g_f[n]), _rel(grads[n].cpu().numpy(), g_f[n]), n) for n in g_f), reverse=True)
    print(f"[{precision}] {flips} of {units} PReLU units on opposite sides of the kink (device vs oracle); frozen kinks, "
          f"{len(errs)} variables: rel-rms max {errs[0][0]:.2e} ({errs[0][2]}), max-err max {max(e[1] for e in errs):.2e}")
    for r, m, n in errs[:4]:
        print(f"[{precision}]   largest frozen-kink error: {n} rel-rms {r:.2e} max {m:.2e}")
    assert len(errs) == 166
    if precision == "exact":                       # measured: rel-rms <= 2.2e-4, max <= 3.0e-4 (790 units flipped)
        assert errs[0][0] < 6e-4 and max(e[1] for e in errs) < 9e-4, errs[:3]
    else:                                          # measured: 1.4e-3 / 1.6e-3 (41044 units flipped)
        assert errs[0][0] < 4e-3 and max(e[1] for e in errs) < 4.5e-3, errs[:3]


def test_two_adam_steps_follow_the_oracle(golden_dir):
    """Two optimiser steps (exact precision, no dropout, e_eta = 2e-5: with 237 M variables moving coherently one step already
    changes the loss by ~1e-3 of its value and the gradient's L1 norm by a third): the loss before each step, after the second,
    and the direction of the accumulated update of a sample of variables vs the oracle trained by the same TF-Adam formulas."""
    from rendernet_b200.training import ShaderTrainer
    vox, poses, grid, target = _scene(golden_dir)
    W = orc.init_shader_weights(seed=2, alpha_range=(0.0, 0.0))          # PReLU slopes start at 0 like the reference (layer_util.py:38)
    lr, b1, b2, eps = 2e-5, 0.5, 0.999, 1e-8
    tr = ShaderTrainer(W, 1, precision="exact", keep_prob=1.0, learning_rate=lr)
    losses = [tr.step(vox, poses, target), tr.step(vox, poses, target)]
    final = tr.loss_and_gradients(vox, poses, target, training=False)[0]
    Wt = {n: torch.tensor(v, requires_grad=True) for n, v in W.items()}
    m = {n: torch.zeros_like(v) for n, v in Wt.items()}
    v2 = {n: torch.zeros_like(v) for n, v in Wt.items()}
    ref = []
    for t in (1, 2):
        l, _, g = _oracle_step(grid, Wt, target, 1.0, 0)
        ref.append(l)
        lr_t = lr * math.sqrt(1 - b2 ** t) / (1 - b1 ** t)
        with torch.no_grad():
            for n in Wt:
                gn = torch.from_numpy(g[n])
                m[n] += (gn - m[n]) * (1 - b1)
                v2[n] += (gn * gn - v2[n]) * (1 - b2)
                Wt[n] -= lr_t * m[n] / (v2[n].sqrt() + eps)
    ref_final = _oracle_step(grid, Wt, target, 1.0, 0)[0]
    print(f"loss trajectory: GPU {losses + [final]} vs oracle {ref + [ref_final]}")
    assert abs(losses[0] - ref[0]) < 1e-5 * ref[0]
    drop_ref, drop = ref[0] - ref_final, losses[0] - final
    assert drop_ref > 1e-3 * ref[0], "the step size of this test should move the loss"      # 0.23342 -> 0.23322 -> 0.23261 on the CPU
    assert abs(losses[1] - ref[1]) < 0.1 * abs(ref[0] - ref[1]) + 1e-5 * ref[0]
    assert abs(drop - drop_ref) < 0.1 * drop_ref
    sd = tr.state_dict()
    assert tr.global_step == 2 and set(sd) == set(W)
    # Adam's first steps are sign-like (|update| ~ lr): compare the direction of the total update of the big tensors
    for n in ("encoder/res2_3/con1_3X3/weights", "encoder/res1_4/conv2_3x3/weights", "encoder/e_conv9/e_conv9/weights",
              "encoder/e_conv1/e_conv1/weights", "encoder/e_conv5/alpha", "encoder/e_conv11/biases"):
        du, dr = sd[n] - W[n], Wt[n].detach().numpy() - W[n]
        c = _cos(du, dr)
        print(f"  update of {n}: cosine {c:.4f}, |update| mean {np.abs(du).mean():.2e} vs {np.abs(dr).mean():.2e}")
        assert c > 0.9


def test_greyscale_bce_batch2_gradients_match_oracle_autograd(golden_dir):
    """The configuration the reference ships (config_RenderNet.json: is_greyscale, keep_prob 1.0, batch > 1 allowed): one-channel
    output, binary cross entropy (RenderNet_Shader.py:158-161), B = 2 with two poses.  Loss and the gradients of all variables vs
    torch.autograd through the oracle, exact precision."""
    from rendernet_b200.training import ShaderTrainer
    bv = np.load(os.path.join(golden_dir, "binvox.npz"))
    chair = np.unpackbits(bv["chair_bits"]).reshape(1, 64, 64, 64, 1).astype(np.float32)
    vox = np.concatenate([chair, chair[:, ::-1].copy()], 0)
    poses = np.concatenate([orc.compute_pose_param(250.0, 60.0, 3.3), orc.compute_pose_param(40.0, 75.0, 3.0)]).astype(np.float32)
    grid = orc.transform_voxel_to_match_image(orc.rotation_resampling(vox, poses)).astype(np.float32)
    sil = (grid[..., 0].sum(axis=3) > 0.5).astype(np.float32)                                   # [B,128,128]
    target = np.ascontiguousarray(np.repeat(np.repeat(sil, 4, 1), 4, 2)[..., None])             # [B,512,512,1] in {0,1}
    W = orc.init_shader_weights(seed=3, is_greyscale=True, alpha_range=(-0.05, 0.25), bias_jitter=0.02)
    tr = ShaderTrainer(W, 2, precision="exact", is_greyscale=True, keep_prob=1.0)
    assert tr.loss_kind == "bce"
    loss, grads = tr.loss_and_gradients(vox, poses, target)
    Wt = {n: torch.tensor(v, requires_grad=True) for n, v in W.items()}
    img = orc.rendernet_shader(torch.from_numpy(grid), Wt)
    t = torch.from_numpy(target)
    ref = (-(t * torch.log(1e-6 + img) + (1 - t) * torch.log(1e-6 + 1 - img)).sum(dim=(1, 2, 3))).mean()
    g_ref = dict(zip(sorted(Wt), torch.autograd.grad(ref, [Wt[n] for n in sorted(Wt)])))
    print(f"[greyscale BCE, B=2] loss {loss:.4f} vs {float(ref):.4f}; image err {float(np.abs(tr.img.cpu().numpy() - img.detach().numpy()).max()):.2e}")
    assert abs(loss - float(ref)) < 5e-5 * float(ref)
    assert set(grads) == set(g_ref)
    worst = min((_cos(grads[n].cpu().numpy(), g_ref[n].numpy()), n) for n in g_ref)
    ratios = [float(np.linalg.norm(grads[n].cpu().numpy()) / max(np.linalg.norm(g_ref[n].numpy()), 1e-30)) for n in g_ref]
    print(f"[greyscale BCE, B=2] {len(grads)} variables: lowest cosine {worst[0]:.5f} ({worst[1]}), norm ratio {min(ratios):.4f}..{max(ratios):.4f}")
    assert worst[0] > 0.9995 and all(abs(r - 1) < 1e-2 for r in ratios)
