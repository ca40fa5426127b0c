"""Host-side logic of training on random patches, on the CPU: the crop mirrors of tools/model_util.py:77-161 against the reference's
own output (tests/golden/crop.npz), the trainers' crop origin and patch schedule, the window checks of the op wrappers, and the
windowed e_conv1 gradient formulas of rendernet_b200/backward.py run with torch emulations of the CUDA entry points and compared
with torch.autograd on the sliced grid.  The kernels are checked on the GPU (tests/test_gpu_patch_training.py)."""
import os
import types

import numpy as np
import pytest
import torch

from oracle import rendernet_oracle as orc
from rendernet_b200 import model_util, ops
from rendernet_b200.backward import ShaderInputGradients, TextureInputGradients
from rendernet_b200.resampling_voxel_grid import ConcatResampledGrid, CroppedGrid, ResampledGrid, concat_resampled
from rendernet_b200.training import _Trainer, patch_size_for_epoch

from test_training_host import emu_bias_grad, emu_conv_weight_grad_direct


def _rel(got, want):
    return float((got.double() - want.double()).abs().max() / want.double().abs().max())


# ------------------------------------------------------------------------------------------- crops vs the reference
def test_crop_mirrors_match_the_reference(golden_dir):
    """With the origin the reference drew, the mirrors return the reference's voxel, texture, image and normal patches bit for
    bit: one origin for the batch, the image patch at (image_dim // voxel_dim) x the origin with that factor x P as its edge."""
    g = np.load(os.path.join(golden_dir, "crop.npz"))
    for i in range(int(g["n_cases"])):
        c = {k[len(f"c{i}_"):]: g[k] for k in g.files if k.startswith(f"c{i}_")}
        P = int(c["patch"])
        v, im = model_util.tf_random_crop_voxel_image(c["vox"], c["img"], P, origin=c["origin_a"])
        assert np.array_equal(v, c["a_vox"]) and np.array_equal(im, c["a_img"])
        f = c["img"].shape[1] // c["vox"].shape[1]
        assert im.shape[1] == f * P and np.array_equal(im, c["img"][:, f * c["origin_a"][0]:, f * c["origin_a"][1]:][:, :f * P, :f * P])
        out = model_util.tf_random_crop_voxel_texture_image_normal(c["vox"], c["tex"], c["img"], c["nrm"], P, origin=c["origin_b"])
        for got, key in zip(out, ("b_vox", "b_tex", "b_img", "b_nrm")):
            assert np.array_equal(got, c[key]), (i, key)
        out3 = model_util.tf_random_crop_voxel_texture_image(c["vox"], c["tex"], c["img"], P, origin=c["origin_b"])
        assert all(np.array_equal(a, c[k]) for a, k in zip(out3, ("b_vox", "b_tex", "b_img")))


def test_crop_draws_one_origin_per_batch_and_keeps_the_whole_grid_at_full_size():
    vox = np.arange(2 * 16 * 16 * 2, dtype=np.float32).reshape(2, 16, 16, 2, 1)
    img = np.arange(2 * 64 * 64 * 3, dtype=np.float32).reshape(2, 64, 64, 3)
    seen = set()
    for s in range(200):
        v, im = model_util.tf_random_crop_voxel_image(vox, img, 4, rng=np.random.default_rng(s))
        y0, x0 = (int(t) for t in np.argwhere(vox[0, :, :, 0, 0] == v[0, 0, 0, 0, 0])[0])
        assert np.array_equal(v, vox[:, y0:y0 + 4, x0:x0 + 4]) and np.array_equal(im, img[:, 4 * y0:4 * y0 + 16, 4 * x0:4 * x0 + 16])
        seen.add((y0, x0))
    assert {y for y, _ in seen} == set(range(13)) and {x for _, x in seen} == set(range(13))
    same = model_util.tf_random_crop_voxel_texture_image_normal(vox, vox, img, img, 16)
    assert len(same) == 4 and all(a is b for a, b in zip(same, (vox, vox, img, img)))
    with pytest.raises(ValueError):
        model_util.tf_random_crop_voxel_image(vox, img, 4, origin=(13, 0))


def test_crop_of_a_deferred_grid_is_a_cropped_grid():
    """On the deferred resampled grid the crops return CroppedGrid (nothing is resampled on the host); a (geometry, texture)
    pair cropped at one origin concatenates into one deferred patch of the 5-channel grid, which the fused kernel consumes."""
    minv = torch.zeros(2, 3, 4)
    geom = ResampledGrid(torch.zeros(2, 8, 8, 8, 1), minv, 128, transform=True)
    tex = ResampledGrid(torch.zeros(2, 8, 8, 8, 4), minv, 128, transform=True)
    img = np.zeros((2, 512, 512, 3), np.float32)
    v, t, im, nm = model_util.tf_random_crop_voxel_texture_image_normal(geom, tex, img, img, 32, origin=(16, 96))
    assert isinstance(v, CroppedGrid) and v.window == (16, 96, 32, 32) and v.shape == (2, 32, 32, 128, 1)
    assert im.shape == (2, 128, 128, 3) and nm.shape == (2, 128, 128, 3)
    cat = concat_resampled(v, t)
    assert isinstance(cat, CroppedGrid) and isinstance(cat.grid, ConcatResampledGrid) and cat.shape == (2, 32, 32, 128, 5)
    with pytest.raises(ValueError):
        CroppedGrid(ResampledGrid(torch.zeros(2, 8, 8, 8, 1), minv, 128, transform=False), 0, 0, 32, 32)
    with pytest.raises(ValueError):
        CroppedGrid(geom, 0, 0, 24, 32)


# ------------------------------------------------------------------------------------------- trainer: origin and schedule
def _fake_trainer(seed=0, data_parallel=False, new_size=128):
    t = types.SimpleNamespace(seed=seed, data_parallel=data_parallel, new_size=new_size)
    t._rank = lambda: _Trainer._rank(t)
    return t


def test_crop_origin_is_deterministic_in_range_and_reaches_both_ends():
    t = _fake_trainer(seed=7)
    for P in (16, 32, 64, 112):
        o = [_Trainer.crop_origin(t, s, P) for s in range(3000)]
        assert o == [_Trainer.crop_origin(t, s, P) for s in range(3000)]
        ys, xs = [y for y, _ in o], [x for _, x in o]
        assert min(ys) == 0 and min(xs) == 0 and max(ys) == 128 - P and max(xs) == 128 - P
        assert len(set(o)) > 0.5 * min(3000, (129 - P) ** 2)
    assert _Trainer.crop_origin(t, 5, 128) == (0, 0)
    assert [_Trainer.crop_origin(_fake_trainer(seed=8), s, 32) for s in range(20)] != [_Trainer.crop_origin(t, s, 32) for s in range(20)]
    with pytest.raises(ValueError):
        _Trainer.crop_origin(t, 0, 144)


def test_crop_origin_differs_across_ranks_only_with_data_parallel(monkeypatch):
    monkeypatch.setattr(torch.distributed, "is_available", lambda: True)
    monkeypatch.setattr(torch.distributed, "is_initialized", lambda: True)
    per_rank = {}
    for dp in (False, True):
        for r in (0, 1, 3):
            monkeypatch.setattr(torch.distributed, "get_rank", lambda r=r: r)
            per_rank[dp, r] = [_Trainer.crop_origin(_fake_trainer(seed=3, data_parallel=dp), s, 32) for s in range(16)]
    assert per_rank[False, 0] == per_rank[False, 1] == per_rank[False, 3] == per_rank[True, 0]
    assert per_rank[True, 1] != per_rank[True, 0] and per_rank[True, 3] != per_rank[True, 1]


def test_patch_size_for_epoch_follows_both_schedules():
    assert [patch_size_for_epoch(e, "shader") for e in range(8)] == [32] * 5 + [64] * 3
    assert [patch_size_for_epoch(e, "texture") for e in range(8)] == [32] * 4 + [64] * 4
    assert patch_size_for_epoch(0, "shader", new_size=64) == 16
    with pytest.raises(ValueError):
        patch_size_for_epoch(0, "decoder")


# ------------------------------------------------------------------------------------------- op wrappers: window checks
@pytest.mark.parametrize("window", [(0, 0, 24, 32), (0, 0, 32, 8), (0, 0, 0, 32), (-16, 0, 32, 32), (112, 0, 32, 32),
                                    (0, 97, 32, 32), (0, 0, 144, 16)])
def test_wrappers_reject_bad_windows_before_launching(window):
    """The checks come first: CPU tensors would be refused later (no CPU path), so a ValueError proves nothing was launched."""
    vox, tex, minv = torch.zeros(1, 8, 8, 8, 1), torch.zeros(1, 8, 8, 8, 4), torch.zeros(1, 3, 4)
    w1, w5, b = torch.zeros(5, 5, 5, 1, 8), torch.zeros(5, 5, 5, 5, 8), torch.zeros(8)
    calls = [lambda: ops.resample(vox, minv, 128, True, window=window),
             lambda: ops.resample_conv1(vox, minv, 128, w1, b, None, window=window),
             lambda: ops.resample5_conv1(vox, tex, minv, 128, w5, b, None, window=window),
             lambda: ops.resample5_backward(vox, tex, minv, torch.zeros(1, max(window[2], 1), max(window[3], 1), 128, 5),
                                            window=window)]
    for call in calls:
        with pytest.raises(ValueError):
            call()
    with pytest.raises(RuntimeError):                        # a good window gets past the check (and then needs CUDA)
        ops.resample_conv1(vox, minv, 128, w1, b, None, window=(96, 0, 32, 16))


def test_windowed_resample_needs_the_axis_transform():
    with pytest.raises(ValueError):
        ops.resample(torch.zeros(1, 8, 8, 8, 1), torch.zeros(1, 3, 4), 128, False, window=(0, 0, 32, 32))


# ------------------------------------------------------------------------------------------- windowed e_conv1 gradients
@pytest.fixture
def emulated_ops(monkeypatch):
    monkeypatch.setattr(ops, "conv_weight_grad_direct", emu_conv_weight_grad_direct)
    monkeypatch.setattr(ops, "bias_grad", emu_bias_grad)
    monkeypatch.setattr(ops, "concat_channels", lambda a, b: torch.cat([a, b], -1))


def _named(t, name):
    t._rn_name = name
    return t


def _emulated_resample(full):
    """rn_resample(_window)_f32 on stand-in voxel objects: the whole precomputed grid, or its window."""
    def resample(vox, minv, n, tr, window=None):
        g = full[id(vox)]
        if window is None:
            return g
        y0, x0, ph, pw = window
        return g[:, y0:y0 + ph, x0:x0 + pw].contiguous()
    return resample


@pytest.mark.parametrize("C,window", [(1, (16, 0, 16, 32)), (5, (0, 16, 32, 16)), (5, (16, 16, 16, 16))])
def test_windowed_econv1_weight_gradient(emulated_ops, monkeypatch, C, window):
    """e_conv1 (5^3 s2) on a window of the grid, SAME-padded at the window's borders: dW and db from the windowed re-resampled
    grid vs autograd through orc.conv3d on the sliced grid."""
    rng = np.random.default_rng(C)
    N, B = 32, 2
    y0, x0, ph, pw = window
    geom = torch.from_numpy(rng.standard_normal((B, N, N, N, 1)).astype(np.float32))
    tex = torch.from_numpy(rng.standard_normal((B, N, N, N, 4)).astype(np.float32))
    vox_g, vox_t = object(), object()
    monkeypatch.setattr(ops, "resample", _emulated_resample({id(vox_g): geom, id(vox_t): tex}))
    full = geom if C == 1 else torch.cat([geom, tex], -1)
    w = torch.tensor((rng.standard_normal((5, 5, 5, C, 8)) * 0.1).astype(np.float32), requires_grad=True)
    b = torch.zeros(8, requires_grad=True)
    y = orc.conv3d(full[:, y0:y0 + ph, x0:x0 + pw], w, b, (2, 2, 2))
    assert tuple(y.shape) == (B, ph // 2, pw // 2, N // 2, 8)
    G = torch.from_numpy(rng.standard_normal(tuple(y.shape)).astype(np.float32))
    (y * G).sum().backward()
    fake = types.SimpleNamespace(weight_grads={}, new_size=N)
    if C == 1:
        grid, op, cls = types.SimpleNamespace(voxel=vox_g, minv=None), "resample_conv1", ShaderInputGradients
    else:
        grid = types.SimpleNamespace(geom=types.SimpleNamespace(voxel=vox_g), tex=types.SimpleNamespace(voxel=vox_t), minv=None)
        op, cls = "resample5_conv1", TextureInputGradients
    rec = dict(op=op, w=_named(w.detach().clone(), "w"), b=_named(b.detach().clone(), "b"), stride=[2, 2, 2], grid=grid,
               window=window)
    cls._weight_grads_of(fake, rec, G * 4.0, 0.25, True)             # g carries a loss scale of 4
    assert _rel(fake.weight_grads["w"], w.grad) < 2e-5 and _rel(fake.weight_grads["b"], b.grad) < 2e-5


def test_windowed_texture_input_chain(monkeypatch):
    """The Texture walk on a patch record: e_conv1's data gradient has the window's extents (B, ph, pw, N, 5) and matches
    autograd on the sliced grid; resample5_backward receives it with the record's window, and dL/d(texture volume) goes on."""
    rng = np.random.default_rng(11)
    N, B, window = 32, 1, (16, 0, 16, 32)
    y0, x0, ph, pw = window
    x = torch.tensor(rng.standard_normal((B, ph, pw, N, 5)).astype(np.float32), requires_grad=True)
    w = torch.from_numpy((rng.standard_normal((5, 5, 5, 5, 8)) * 0.1).astype(np.float32))
    y = orc.conv3d(x, w, None, (2, 2, 2))
    G = torch.from_numpy(rng.standard_normal(tuple(y.shape)).astype(np.float32))
    (y * G).sum().backward()

    def emu_bwd_data(g, w32, in_shape, stride, want32=False, out_scale=1.0):
        xin = torch.zeros(tuple(in_shape), requires_grad=True)
        (orc.conv3d(xin, w32, None, tuple(stride)) * g).sum().backward()
        return xin.grad * out_scale

    seen = {}

    def emu_r5b(vox, tex, minv, gout, want_dvox=True, want_dtex=True, want_dminv=True, window=None):
        seen.update(gout=gout, window=window)
        return None, torch.ones(1), None
    monkeypatch.setattr(ops, "conv3d_backward_data_direct", emu_bwd_data)
    monkeypatch.setattr(ops, "resample5_backward", emu_r5b)
    tex_vox = torch.zeros(4)
    grid = types.SimpleNamespace(geom=types.SimpleNamespace(voxel=None), tex=types.SimpleNamespace(voxel=tex_vox), minv=None)
    fake = types.SimpleNamespace(new_size=N, B=B, last_loss_scale=4.0, _want=(False, True, False), _w32=lambda t: t)
    grads = {}
    rec = dict(op="resample5_conv1", w=w, stride=[2, 2, 2], grid=grid, window=window)
    TextureInputGradients._input_chain(fake, rec, G * 4.0, grads)
    assert seen["window"] == window and tuple(seen["gout"].shape) == (B, ph, pw, N, 5)
    assert _rel(seen["gout"], x.grad) < 2e-6
    assert fake._dtex_reached and len(grads) == 1


def test_shader_input_gradients_refuse_a_patch_record():
    fake = types.SimpleNamespace(_need_inputs=True)
    with pytest.raises(NotImplementedError):
        ShaderInputGradients._input_chain(fake, dict(op="resample_conv1", window=(0, 0, 32, 32)), None, {})
