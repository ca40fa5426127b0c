"""The 16-bit backward pass at the gradient magnitudes real losses produce (DESIGN §4).

dL/d(output) is scaled by the loss scale in rn_sigmoid_backward and stored as fp16 (fast) or an fp16 hi/lo pair (exact); from
there on every gradient of the trunk and the heads is 16-bit.  These tests pin
  (a) the window of magnitudes in which each format keeps its bits, and what happens outside it;
  (b) that whole backward passes are exact under power-of-two scaling of dL/d(output), from 2^-40 to 2^20: every step of the
      walk is exact under such a scaling while values stay in range, and the loss scale is chosen per call to keep them there;
  (c) the real losses (Shader MSE at B = 1 and at the B = 24 per-pixel magnitude, the reconstruction objective at a random
      start and near convergence) against the float64 frozen-kink oracle, at the white-noise tests' bars;
  (d) overflow: retried at a lower scale or FloatingPointError, never an inf / NaN result.
Outputs that go through fp32 atomics (dvox, dtex, dM^-1, the weight gradients) differ from run to run in the last bits: (b)
measures that noise by running the unscaled case twice and holds every scale to a small multiple of it.
"""
import math
import os

import numpy as np
import pytest
import torch

from oracle import rendernet_oracle as orc

pytestmark = pytest.mark.gpu
dev = "cuda"
KS = (-40, -30, -20, -10, 0, 10, 20)
NOISE_FLOOR = 2.0 ** -23          # relative: atomics noise of a run that happens to repeat bit for bit
NOISE_MULT = 4.0


def _rel(got, want):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert got.shape == want.shape, (got.shape, want.shape)
    return float(np.abs(got - want).max() / max(np.abs(want).max(), 1e-300))


def _rms(got, want):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    return float(np.sqrt(((got - want) ** 2).mean()) / max(np.sqrt((want ** 2).mean()), 1e-300))


# ----------------------------------------------------------------------------------------- (a) representation vs magnitude
def _probe_values():
    """fp32 magnitudes from 2^-30 to 2^17: exact powers of two, random mantissas per binade, the fp16 subnormal / flush
    boundaries and their half-ulp ties, +-0, and values around 65504 and fp16's overflow threshold 65520."""
    rng = np.random.default_rng(1)
    v = [2.0 ** e for e in range(-30, 18)]
    v += list((2.0 ** rng.uniform(-30, 17, 4000)))
    v += [2.0 ** -25, 2.0 ** -25 * 1.0000001, 2.0 ** -25 * 0.9999999, 3 * 2.0 ** -25, 2.0 ** -24, 1.5 * 2.0 ** -24,
          2.0 ** -14, 2.0 ** -14 - 2.0 ** -25, 2.0 ** -14 + 2.0 ** -25, 2.0 ** -14 - 2.0 ** -24, 2.0 ** -3 - 2.0 ** -20,
          65504.0, 65510.0, 65519.0, np.nextafter(np.float32(65520.0), np.float32(0)), 65520.0, 65536.0, 1e5, 2.0 ** 17]
    v = np.asarray(v, np.float32)
    sgn = np.where(rng.random(v.size) < 0.5, -1.0, 1.0).astype(np.float32)
    return np.concatenate([v * sgn, -v * sgn, np.array([0.0, -0.0], np.float32)])


@pytest.mark.parametrize("fmt", [2, 0], ids=["exact", "fast"])
def test_sigmoid_backward_representation_window(fmt):
    """rn_sigmoid_backward at s = 0.5 (s (1 - s) = 1/4 exactly) and a power-of-two scale, so the fp32 product is exact and only
    the 16-bit store rounds.  float64 bounds: exact |err| <= max(2^-22 |v|, 2^-25) (hi rounding, then lo: relative while lo
    is normal, its subnormal half step 2^-25 below), i.e. 2^-21 relative for |v| >= 2^-3; fast |err| <= max(2^-11 |v|,
    2^-25), 2^-11 relative for |v| >= 2^-14; |v| <= 2^-25 flushes to 0 (the tie goes to the even 0); |v| >= 65520 is +-inf
    in the HI half, never a saturated 65504."""
    from rendernet_b200 import ops
    v = _probe_values()
    C = 3
    n = -(-v.size // C) * C
    vv = np.zeros(n, np.float32)
    vv[:v.size] = v
    scale = 2.0 ** 10
    g = (vv * np.float32(4.0 / scale)).reshape(-1, C)
    assert np.array_equal(g.astype(np.float64) * scale / 4, vv.reshape(-1, C).astype(np.float64))   # the input is exact
    s = np.full_like(g, 0.5)
    out = ops.sigmoid_backward(torch.from_numpy(g).to(dev), torch.from_numpy(s).to(dev), 16, scale, fmt)
    planes = out.planes if fmt == 2 else out[None]
    hi, got = (planes[i][..., :C].double().cpu().numpy().reshape(-1)[:v.size] for i in (0, -1))
    if fmt == 2:
        got = hi + got                                   # the pair's value, summed in float64
    want = v.astype(np.float64)
    a = np.abs(want)
    over = a >= 65520.0
    fin = ~over
    assert np.array_equal(hi[over], np.sign(want[over]) * np.inf), "overflow must give +-inf, not a saturated value"
    assert not np.isfinite(got[over]).any()
    assert np.array_equal(got[a == 65504.0], want[a == 65504.0])
    rel = 2.0 ** -22 if fmt == 2 else 2.0 ** -11
    err = np.abs(got[fin] - want[fin])
    bound = np.maximum(rel * a[fin], 2.0 ** -25)
    print(f"fmt {fmt}: {fin.sum()} finite probes, worst {float((err / bound).max()):.3f} of max({rel:.1e} |v|, 2^-25)")
    assert (err <= bound).all()
    # the window: the claimed relative precision holds above the edge, and the edge is real (broken just below it)
    edge, claim = (2.0 ** -3, 2.0 ** -21) if fmt == 2 else (2.0 ** -14, 2.0 ** -11)
    r = np.where(a[fin] > 0, err / np.maximum(a[fin], 1e-300), 0.0)
    inside = a[fin] >= edge
    below = (a[fin] < edge) & (a[fin] > edge / 64)
    print(f"fmt {fmt}: relative error above 2^{math.log2(edge):.0f}: {r[inside].max():.2e} (claim {claim:.1e}); "
          f"in the six binades below: {r[below].max():.2e}")
    assert r[inside].max() <= claim and r[below].max() > claim
    # flush to zero and the subnormal step
    assert (got[a <= 2.0 ** -25] == 0).all()
    assert (got[(a > 2.0 ** -25) & (a < 2.0 ** -24)] != 0).all()
    assert np.array_equal(np.abs(got[(a > 2.0 ** -25) & (a <= 2.0 ** -24)]), np.full(int(((a > 2.0 ** -25) & (a <= 2.0 ** -24)).sum()), 2.0 ** -24))


# ----------------------------------------------------------------------------------------- (b) power-of-two equivariance
def _max_rel_diff(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-300))


def _check_equivariance(label, run, ks, exact_keys=(), noise_by=None):
    """run(f) -> {name: device tensor} for dL/d(output) multiplied by f = 2^k.  Keys in exact_keys must be bit-identical to the
    unscaled run after dividing by 2^k; the rest within NOISE_MULT times the run-to-run noise of two unscaled runs."""
    base = {n: t.clone() for n, t in run(1.0).items()}
    again = run(1.0)
    noise = {n: _max_rel_diff(again[n], base[n]) for n in base}
    if noise_by is not None:                       # one noise level per kind of output (one kind of reduction kernel)
        level = {}
        for n, v in noise.items():
            level[noise_by(n)] = max(level.get(noise_by(n), 0.0), v)
        noise = {n: level[noise_by(n)] for n in noise}
    for n in exact_keys:
        assert torch.equal(again[n], base[n]), f"{label}: {n} is not reproducible"
    del again
    fails, rows = [], []
    for k in ks:
        f = 2.0 ** k
        out = run(f)
        row = []
        for n, t in out.items():
            back = t * (1.0 / f)
            if not bool(torch.isfinite(t).all()):
                row.append(f"{n} NOT FINITE")
                fails.append((k, n, "not finite"))
            elif n in exact_keys:
                same = torch.equal(back, base[n])
                row.append(f"{n} {'bit-exact' if same else f'{_max_rel_diff(back, base[n]):.1e} NOT bit-exact'}")
                if not same:
                    fails.append((k, n, "not bit-exact"))
            else:
                d = _max_rel_diff(back, base[n])
                row.append(f"{n} {d:.1e}")
                if d > NOISE_MULT * max(noise[n], NOISE_FLOOR):
                    fails.append((k, n, d))
        rows.append(f"k={k:+d}: " + ", ".join(row[:6]) + (f" (+{len(row) - 6} more)" if len(row) > 6 else ""))
    noise_s = ", ".join(f"{n} {v:.1e}" for n, v in list(noise.items())[:6])
    print(f"{label}: run-to-run noise {noise_s}" + "".join(f"\n  {r}" for r in rows))
    assert not fails, (label, fails[:8])


def _chair(B):
    bv = np.load(os.path.join(os.path.dirname(__file__), "golden", "binvox.npz"))
    vox = np.unpackbits(bv["chair_bits"]).reshape(1, 64, 64, 64, 1).astype(np.float32)
    vox = vox * 0.75 + 0.125 * (np.random.default_rng(2).random(vox.shape) < 0.02)
    az = np.linspace(250.0, 250.0 + 360.0, B, endpoint=False)
    poses = np.concatenate([orc.compute_pose_param(a % 360.0, 60.0, 3.3) for a in az]).astype(np.float32)
    return np.ascontiguousarray(np.repeat(vox, B, 0)), poses


def _shader_weights():
    return orc.init_shader_weights(seed=1, alpha_range=(0.05, 0.3), bias_jitter=0.02)


@pytest.mark.parametrize("B", [1, 24])
@pytest.mark.parametrize("precision", ["exact", "fast"])
def test_shader_input_gradients_exact_under_power_of_two_scaling(precision, B):
    """ShaderInputGradients.backward(2^k G), G ~ N(0, 1): dL/dgrid (one thread per voxel, no atomics) is 2^k times the
    unscaled result bit for bit; dvox and dpose (resampler atomics) within the noise."""
    from rendernet_b200.backward import ShaderInputGradients
    vox, poses = _chair(B)
    ig = ShaderInputGradients(_shader_weights(), B, precision=precision)
    ig.forward(vox, poses)
    G = torch.from_numpy(np.random.default_rng(5).standard_normal((B, 512, 512, 3)).astype(np.float32)).to(dev)

    def run(f):
        dvox, dpose = ig.backward(G * f)
        return dict(dgrid=ig.last_dgrid, dvox=torch.from_numpy(dvox), dpose=torch.from_numpy(dpose))
    _check_equivariance(f"Shader {precision} B={B}", run, KS if B == 1 else (-30, 0, 10), exact_keys=("dgrid",))


def test_fixed_loss_scale_leaves_the_window():
    """The old fixed scale 4096: at 2^-30 G the gradients flush in fp16's subnormal range (dL/dgrid no longer 2^-30 times the
    unscaled one), at 2^10 G the output layer overflows, which now raises instead of returning inf / NaN."""
    from rendernet_b200.backward import ShaderInputGradients
    vox, poses = _chair(1)
    ig = ShaderInputGradients(_shader_weights(), 1, precision="exact", loss_scale=4096.0)
    ig.forward(vox, poses)
    G = torch.from_numpy(np.random.default_rng(5).standard_normal((1, 512, 512, 3)).astype(np.float32)).to(dev)
    ig.backward(G)
    base = ig.last_dgrid.clone()
    ig.backward(G * 2.0 ** -30)
    d = _max_rel_diff(ig.last_dgrid * 2.0 ** 30, base)
    print(f"fixed scale 4096 at 2^-30 G: dL/dgrid {d:.2e} from the unscaled result")
    assert d > 1e-3
    with pytest.raises(FloatingPointError):
        ig.backward(G * 2.0 ** 10)
    assert ig.last_loss_scale == 4096.0


def _texture_weights(seed):
    W = orc.init_texture_weights(seed=seed, alpha_range=(-0.3, 0.3), bias_jitter=0.02)
    for k in list(W):                        # residual slopes zero: model="pretrained" (ReLU there) is the same network
        if k.endswith("/alpha") and "/res" in k:
            W[k] = np.zeros_like(W[k])
    return W


def _texture_inputs(B, seed):
    rng = np.random.default_rng(seed)
    vox = ((rng.random((B, 64, 64, 64, 1)) < 0.25) * rng.uniform(0.5, 1.0, (B, 64, 64, 64, 1))).astype(np.float32)
    z = rng.standard_normal((B, 199)).astype(np.float32)
    poses = np.stack([rng.uniform(0, 6.28, B), rng.uniform(0.2, 1.4, B), rng.uniform(2.5, 3.3, B)], 1).astype(np.float32)
    az = rng.uniform(0.2, 2.8, (B, 1)).astype(np.float32)
    return vox, z, poses, az


def _phong_grads(albedo, normal, target, az, el=0.7):
    from rendernet_b200 import ops
    from rendernet_b200.Reconstruct_RenderNet_Face import light_pos
    B = albedo.shape[0]
    loss, da, dn, _ = ops.phong_recon_loss_grad(albedo, normal, target.contiguous(), torch.from_numpy(light_pos(az, el)).to(dev),
                                                torch.ones(B, 3, device=dev), 0.0, 1.0, black_background=False, with_mask=True)
    return loss, da, dn


@pytest.mark.parametrize("precision", ["exact", "fast"])
def test_texture_input_gradients_exact_under_power_of_two_scaling(precision):
    """TextureInputGradients at B = 5, through G ~ N(0, 1) and through the reconstruction objective's image gradients."""
    from rendernet_b200.backward import TextureInputGradients
    B = 5
    vox, z, poses, az = _texture_inputs(B, 3)
    tig = TextureInputGradients(_texture_weights(4), B, precision=precision)
    albedo, normal = tig.forward(vox, z, poses)
    rng = np.random.default_rng(6)
    Ga, Gn = (torch.from_numpy(rng.standard_normal((B, 512, 512, 3)).astype(np.float32)).to(dev) for _ in range(2))
    target = torch.from_numpy(rng.random((B, 512, 512, 3)).astype(np.float32)).to(dev)
    _, da, dn = _phong_grads(albedo, normal, target, az)
    for label, (ga, gn) in (("N(0,1)", (Ga, Gn)), ("reconstruction objective", (da, dn))):
        def run(f):
            dvox, dtex, dpose = tig.backward(ga * f, gn * f)
            return dict(dgrid=tig.last_dgrid, dvox=torch.from_numpy(dvox), dtex=torch.from_numpy(dtex),
                        dpose=torch.from_numpy(dpose))
        _check_equivariance(f"Texture {precision} B={B} {label}", run, KS, exact_keys=("dgrid",))


def test_trainer_weight_gradients_exact_under_power_of_two_scaling():
    """ShaderTrainer.backward(2^k dimg) at B = 2 with dropout: all 166 weight gradients within the noise of the split-K /
    direct weight-gradient atomics."""
    from rendernet_b200 import ops
    from rendernet_b200.training import ShaderTrainer
    vox, poses = _chair(2)
    tr = ShaderTrainer(_shader_weights(), 2, precision="exact", keep_prob=0.75, seed=3)
    img = tr.forward(vox, poses)
    target = (img + 0.3 * torch.randn(img.shape, device=dev, generator=torch.Generator(dev).manual_seed(1))).clamp(0, 1)
    _, dimg = ops.image_loss_grad(img.contiguous(), target.contiguous(), "mse")

    def run(f):
        tr.backward(dimg * f, want_dvox=False, want_dpose=False, want_weight_grads=True)
        assert len(tr.weight_grads) == 166
        return dict(tr.weight_grads)
    _check_equivariance("ShaderTrainer exact B=2, weight gradients", run, (-40, -20, 0, 10, 20),
                        noise_by=lambda n: n.rsplit("/", 1)[1])


def test_face_reconstruction_chain_exact_under_power_of_two_scaling():
    """FaceReconstruction.gradients' chain: TextureInputGradients.backward(2^k image gradients, dvox on the device) ->
    ShapeDecoderGradients.backward -> dL/dlatent."""
    from rendernet_b200.Reconstruct_RenderNet_Face import FaceReconstruction, pretrained_dict_from_texture_weights
    from oracle.shape_decoder import init_shape_decoder_weights
    B = 5
    rec = FaceReconstruction(pretrained_dict_from_texture_weights(_texture_weights(7)), init_shape_decoder_weights(8), batch=B)
    _, z, poses, az = _texture_inputs(B, 9)
    lat = (0.5 + 0.3 * np.random.default_rng(10).standard_normal((B, 200))).astype(np.float32)
    vox = rec.sdg.forward(lat)
    albedo, normal = rec.tig.forward(vox, z, poses)
    target = torch.from_numpy(np.random.default_rng(11).random((B, 512, 512, 3)).astype(np.float32)).to(dev)
    _, da, dn = _phong_grads(albedo, normal, target, az, rec.elevation)

    def run(f):
        dv, dtex, _ = rec.tig.backward(da * f, dn * f, want_dpose=False, dvox_on_device=True)
        return dict(dgrid=rec.tig.last_dgrid, dlatent=torch.from_numpy(rec.sdg.backward(dv)), dtex=torch.from_numpy(dtex))
    _check_equivariance("FaceReconstruction chain exact B=5", run, KS, exact_keys=("dgrid",))


# ----------------------------------------------------------------------------------------- (c) real losses vs float64
@pytest.mark.parametrize("precision", ["exact", "fast"])
def test_shader_mse_gradients_match_frozen_kink_oracle(precision):
    """The Shader network's MSE gradient at B = 1 (|dL/dpixel| ~ 1e-6) and the same divided by 24 (the B = 24 per-pixel
    magnitude; the float64 reference just scales) against the frozen-kink oracle, at the bars of
    tests/test_gpu_backward.py::test_full_size_input_gradients_match_oracle_autograd."""
    from rendernet_b200 import ops, tfcompat as tf
    from rendernet_b200.backward import ShaderInputGradients, pose_matrix_jacobian_vjp
    from oracle.frozen_kinks import prelu_kinks, tape_prelu_masks
    from test_gpu_backward import _oracle_gradients
    vox, poses = _chair(1)
    W = _shader_weights()
    ig = ShaderInputGradients(W, 1, precision=precision)
    img = ig.forward(vox, poses)
    target = (img + 0.3 * torch.randn(img.shape, device=dev, generator=torch.Generator(dev).manual_seed(2))).clamp(0, 1)
    _, dimg = ops.image_loss_grad(img.contiguous(), target.contiguous(), "mse")
    with tf.use_store(ig.store):
        masks = tape_prelu_masks(ig.tape)
    G = dimg.cpu().numpy()
    with prelu_kinks(W, masks=masks):
        _, dvox_f, dminv_f, _, _ = _oracle_gradients(vox, poses, W, G)
    dpose_f = pose_matrix_jacobian_vjp(poses, dminv_f)
    bars = dict(max=3.5e-4, rms=3.5e-4, dpose=2.7e-4) if precision == "exact" else dict(max=7e-3, rms=5e-3, dpose=2.8e-3)
    for div in (1.0, 24.0):
        dvox, dpose = ig.backward(dimg / div)
        e = dict(max=_rel(dvox * div, dvox_f), rms=_rms(dvox * div, dvox_f), dpose=_rel(dpose * div, dpose_f))
        print(f"[{precision}] Shader MSE B=1 / {div:g} (max |dL/dpixel| {float(dimg.abs().max()) / div:.1e}, loss scale "
              f"{getattr(ig, 'last_loss_scale', ig.loss_scale)}) vs frozen-kink oracle: dvox max {e['max']:.2e} rms {e['rms']:.2e}, dpose {e['dpose']:.2e}")
        for n, v in e.items():
            assert v < bars[n], (div, n, v)


@pytest.mark.parametrize("precision", ["exact", "fast"])
def test_reconstruction_gradients_match_frozen_kink_oracle(precision):
    """The reconstruction objective's image gradients at B = 2, at a random start (loss ~0.1) and near convergence (target =
    the state's own shaded image + noise of 0.01: loss ~1e-4, |dL/dpixel| ~ 1e-8) pushed through TextureInputGradients,
    against the frozen-kink oracle, at the bars of test_full_size_texture_input_gradients_match_frozen_kink_oracle."""
    from rendernet_b200 import tfcompat as tf
    from rendernet_b200.backward import TextureInputGradients, pose_matrix_jacobian_vjp
    from rendernet_b200.Reconstruct_RenderNet_Face import light_pos
    from oracle import phong_tf as pt
    from oracle.frozen_kinks import tape_prelu_masks
    from test_gpu_texture_backward import _oracle_texture_gradients
    B = 2
    W = _texture_weights(12)
    vox, z, poses, az = _texture_inputs(B, 13)
    tig = TextureInputGradients(W, B, precision=precision)
    albedo, normal = tig.forward(vox, z, poses)
    with tf.use_store(tig.store):
        masks = tape_prelu_masks(tig.tape)
    shade = pt.tf_phong_composite(normal.double().cpu(), torch.from_numpy(light_pos(az, 0.7)).double(),
                                  torch.ones(B, 3, dtype=torch.float64), 0.0, 1.0)
    rng = np.random.default_rng(14)
    near = (albedo.double().cpu() * shade + 0.01 * torch.from_numpy(rng.standard_normal((B, 512, 512, 3)))).float().to(dev)
    start = torch.from_numpy(rng.random((B, 512, 512, 3)).astype(np.float32)).to(dev)
    bar = 3e-4 if precision == "exact" else 6e-3
    for label, target in (("random start", start), ("near convergence", near)):
        loss, da, dn = _phong_grads(albedo, normal, target, az)
        dvox, dtex, dpose = tig.backward(da, dn)
        dvox_f, dtex_f, dminv_f = _oracle_texture_gradients(vox, z, poses, W, da.cpu().numpy(), dn.cpu().numpy(), masks)
        dpose_f = pose_matrix_jacobian_vjp(poses, dminv_f)
        e = dict(dvox=_rel(dvox, dvox_f), dtex=_rel(dtex, dtex_f), dpose=_rel(dpose, dpose_f))
        print(f"[{precision}] reconstruction {label} (loss {loss.cpu().numpy()}, max |dL/dpixel| "
              f"{max(float(da.abs().max()), float(dn.abs().max())):.1e}, loss scale {getattr(tig, 'last_loss_scale', tig.loss_scale)}) vs frozen-kink "
              f"oracle: " + ", ".join(f"{n} {v:.2e}" for n, v in e.items()))
        for n, v in e.items():
            assert v < bar, (label, n, v)


# ----------------------------------------------------------------------------------------- (d) overflow
def test_input_gradients_retry_or_raise_on_overflow():
    """A headroom target far above fp16's range makes the output layer overflow: the adaptive scale retries 16x lower until
    nothing overflows and returns what that scale, fixed, gives (within the atomics noise); a fixed scale that overflows, or
    an adaptive one out of retries, raises FloatingPointError.  Neither returns inf / NaN.  Both input-gradient classes."""
    from rendernet_b200.backward import LOSS_SCALE_TARGET, ShaderInputGradients, TextureInputGradients
    vox, poses = _chair(1)
    G = torch.from_numpy(np.random.default_rng(5).standard_normal((1, 512, 512, 3)).astype(np.float32)).to(dev)
    tvox, z, tposes, _ = _texture_inputs(1, 15)
    W = _texture_weights(16)
    cases = (("Shader", lambda ls: ShaderInputGradients(_shader_weights(), 1, loss_scale=ls),
              lambda ig: ig.forward(vox, poses), lambda ig: ig.backward(G)),
             ("Texture", lambda ls: TextureInputGradients(W, 1, loss_scale=ls),
              lambda ig: ig.forward(tvox, z, tposes), lambda ig: ig.backward(G, G)))
    for name, make, fwd, bwd in cases:
        ig = make(None)
        fwd(ig)
        bwd(ig)
        sane_scale = ig.last_loss_scale
        ig.scale_target = 2.0 ** 24
        high = [torch.from_numpy(a) for a in bwd(ig)]
        got = ig.last_loss_scale
        print(f"{name}: target 2^24 -> loss scale {got:g} after retries (the default target gives {sane_scale:g})")
        assert got <= 2.0 ** 24 / 16 * sane_scale / LOSS_SCALE_TARGET
        ig.loss_scale = got                                 # the same walk at that scale, fixed: no retry
        ref = [torch.from_numpy(a) for a in bwd(ig)]
        ref2 = [torch.from_numpy(a) for a in bwd(ig)]
        for a, b, c in zip(high, ref, ref2):
            assert bool(torch.isfinite(a).all())
            assert _max_rel_diff(a, b) <= NOISE_MULT * max(_max_rel_diff(c, b), NOISE_FLOOR)
        ig.loss_scale = None
        ig.overflow_retries = 0
        with pytest.raises(FloatingPointError):
            bwd(ig)
        fixed = make(2.0 ** 30)
        fwd(fixed)
        with pytest.raises(FloatingPointError):
            bwd(fixed)


def test_trainer_recovers_from_overflow():
    """ShaderTrainer.step with its headroom target (adaptive) or its fixed loss scale far too high: the step is redone at half
    the value (same dropout masks) until nothing overflows, and the gradient it applies equals that of a trainer started at the
    value it settled on, within the atomics noise of two such trainers.  Without overflows the target grows back toward where
    it started."""
    from rendernet_b200.backward import LOSS_SCALE_TARGET
    from rendernet_b200.training import ShaderTrainer
    vox, poses = _chair(2)
    W = _shader_weights()
    target = np.random.default_rng(17).random((2, 512, 512, 3)).astype(np.float32)

    def stepped(target_=None, **kw):
        tr = ShaderTrainer(W, 2, precision="exact", keep_prob=0.75, seed=4, learning_rate=1e-4, **kw)
        if target_ is not None:
            tr.scale_target = target_
        tr.step(vox, poses, target)
        assert tr.global_step == 1
        return tr

    hot = stepped(2.0 ** 18)
    fixed = stepped(loss_scale=2.0 ** 40)
    print(f"adaptive: target 2^18 -> 2^{math.log2(hot.scale_target):.0f}; fixed: 2^40 -> 2^{math.log2(fixed.loss_scale):.0f}")
    assert hot.scale_target < 2.0 ** 18 and fixed.loss_scale < 2.0 ** 40
    kind = lambda n: n.rsplit("/", 1)[1]                                        # noqa: E731
    worst = {}
    for tag, tr, kw in (("adaptive", hot, dict(target_=hot.scale_target)), ("fixed", fixed, dict(loss_scale=fixed.loss_scale))):
        ref, ref2 = stepped(**kw), stepped(**kw)
        # the noise of one kind of variable (filters, biases, slopes: one kind of reduction kernel) between the two
        noise = {}
        for n in ref.m:
            noise[kind(n)] = max(noise.get(kind(n), NOISE_FLOOR), _max_rel_diff(ref2.m[n], ref.m[n]))
        for n in ref.m:                              # Adam's first moment after one step: (1 - beta1) x the gradient applied
            d = _max_rel_diff(tr.m[n], ref.m[n])
            worst[tag] = max(worst.get(tag, 0.0), d / noise[kind(n)])
            assert d <= NOISE_MULT * noise[kind(n)], (tag, n, d, noise[kind(n)])
        print(f"{tag}: noise of two trainers started at the settled value {noise}")
        del ref, ref2
        torch.cuda.empty_cache()
    print(f"gradient applied vs a trainer started at the settled value, worst over 166 variables in units of the noise: {worst}")
    # grow back: one step without overflow after growth_interval doubles the target, up to its starting value
    tr = hot
    del fixed
    tr.scale_target = LOSS_SCALE_TARGET / 4
    tr.growth_interval = 1
    tr.step(vox, poses, target)
    assert tr.scale_target == LOSS_SCALE_TARGET / 2
    tr.step(vox, poses, target)
    tr.step(vox, poses, target)
    assert tr.scale_target == LOSS_SCALE_TARGET
