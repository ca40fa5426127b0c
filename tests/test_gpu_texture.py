"""GPU tests of the Texture+Normal network's forward path (BASELINE config 4, `bench.py --config 4`) at the batch it is benchmarked
at, B = 24: the texture decoder's kernels against float64, the tiled 4^3 conv against the generic one bit for bit, and the whole
engine at B = 24 against B = 8 shards, B = 1 renders and the oracle.

The float64 reference is the oracle's own decoder code run with dtype=torch.float64 (oracle/rendernet_oracle.py), so it has the
SAME-padding and transposed-conv semantics that tests/test_oracle_golden.py pins to the reference's Python.  Inputs are the fp32
values a kernel actually reads (for 16-bit inputs: after rounding).  Errors are max |kernel - float64| / max |float64|.

A 16-bit output is checked bit for bit against torch's round-to-nearest of the same call's fp32 output, so it carries the fp32
output's measured error plus one rounding.

Bars: about 3x the largest value measured on one H100 80GB HBM3 (400 W power limit).  The kernels reduce in a fixed order (no
atomics), so with these seeded inputs the errors repeat run to run.
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import rendernet_oracle as orc

pytestmark = pytest.mark.gpu
dev = "cuda"
F64 = torch.float64
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# fc_kernel, one fp32 FMA chain of K terms per output: measured <= 6.4e-7 at the decoder's K = 199 (B = 1..32), 9.2e-7 at K = 512
BAR_FC = 3e-6
# conv3d_small_kernel and conv3d_k4_8to4_tiled_kernel, <= 256 terms per output: measured <= 9.2e-7 on the small grids (every
# instantiation and format), 1.1e-6 for e_tex_conv2 at B = 24 (tiled), 6.3e-7 / 2.8e-7 for e_tex_conv0 / e_tex_conv1
BAR_CONV = 3.5e-6
# the whole decoder (FC + three convolutions) on the bench's texture vectors: measured 1.06e-6 (worst of 24 items), item 23 8.5e-7
BAR_DECODER = 3e-6

FMT_NAMES = {0: "fp16", 1: "bf16", 2: "fp16 hi/lo"}


def _weights():
    return orc.init_texture_weights(seed=3, alpha_range=(0.05, 0.3), bias_jitter=0.02)


def _rel(got, ref) -> float:
    got = got.float().cpu().to(F64) if got.dtype != F64 else got.cpu()
    return float((got - ref).abs().max() / ref.abs().max())


def _round16(v: torch.Tensor, fmt: int) -> torch.Tensor:
    """What a kernel must store for the fp32 values v in 16-bit format fmt (torch's round-to-nearest-even, not the library's):
    the tensor, or fmt 2's [2, ...] planes hi = fp16(v), lo = fp16(v - hi)."""
    if fmt == 1:
        return v.bfloat16()
    hi = v.half()
    return hi if fmt == 0 else torch.stack([hi, (v - hi.float()).half()])


def _to16(v: torch.Tensor, fmt: int):
    """An fp32 device tensor as a 16-bit kernel input in format fmt (rounded by torch)."""
    from rendernet_b200.ops import Split16
    return Split16(_round16(v, 2)) if fmt == 2 else _round16(v, fmt)


def _same16(got, v32: torch.Tensor, fmt: int, label: str):
    from rendernet_b200.ops import Split16
    bits = got.planes if isinstance(got, Split16) else got
    want = _round16(v32, fmt)
    assert isinstance(got, Split16) == (fmt == 2) and bits.dtype == want.dtype, (label, type(got), bits.dtype)
    assert torch.equal(bits, want), (label, int((bits != want).sum()))


# ----------------------------------------------------------------------------------------------------- fully_connected
def _check_fc(B, K, N, seed):
    from rendernet_b200 import ops
    rng = np.random.default_rng(seed)
    x = torch.from_numpy(rng.standard_normal((B, K)).astype(np.float32))
    w = torch.from_numpy((rng.standard_normal((K, N)) * 0.02).astype(np.float32))
    b = torch.from_numpy((rng.standard_normal(N) * 0.05).astype(np.float32))
    a = torch.from_numpy(rng.uniform(-0.5, 1.5, N).astype(np.float32))
    assert (a < 0).any() and (a > 1).any()
    xd, wd = x.to(dev), w.to(dev)
    mm = orc.fully_connected(x, w, dtype=F64)
    errs = []
    for bias in (None, b):
        for alpha in (None, a):
            ref = mm if bias is None else orc.fully_connected(x, w, bias, dtype=F64)
            if alpha is not None:
                ref = orc.prelu(ref, alpha, dtype=F64)
            bd = None if bias is None else bias.to(dev)
            ad = None if alpha is None else alpha.to(dev)
            got = ops.fully_connected(xd, wd, bd, ad)
            label = f"fc B={B} K={K} N={N} bias={bias is not None} prelu={alpha is not None}"
            err = _rel(got, ref)
            errs.append(err)
            print(f"{label}: fp32 {err:.2e}, last item {_rel(got[-1], ref[-1]):.2e}")
            assert err < BAR_FC, label
            for fmt in FMT_NAMES:
                _same16(ops.fully_connected(xd, wd, bd, ad, want32=False, fmt=fmt), got, fmt, f"{label} {FMT_NAMES[fmt]}")
    return errs


@pytest.mark.parametrize("B", [1, 8, 9, 24, 32])
def test_fully_connected_decoder_shape(B):
    """e_tex_fc1's shape, K = 199 -> N = 32^3 * 4, at batch sizes on both sides of the fc_kernel<8> / fc_kernel<32> split
    (B <= 8 / 9..32): the bench runs B = 24 through fc_kernel<32>.  With and without bias and PReLU (slopes in [-0.5, 1.5]);
    fp32 output vs float64, the three 16-bit outputs vs the rounded fp32 output."""
    _check_fc(B, 199, 131072, seed=B)


@pytest.mark.parametrize("B,K,N", [(3, 199, 1000), (9, 57, 1001), (32, 384, 1001), (24, 512, 255)])
def test_fully_connected_ragged_shapes(B, K, N):
    """N not a multiple of the 256-thread block (a partial last block) and B * K * 4 at the 48 KB shared-memory limit."""
    _check_fc(B, K, N, seed=100 + B)


def test_fully_connected_rejects_unsupported_shapes():
    from rendernet_b200 import ops
    from rendernet_b200._lib import RenderNetCudaError
    z = lambda *s: torch.zeros(s, device=dev)                                                         # noqa: E731
    with pytest.raises(RenderNetCudaError, match="rc=-2"):                # B > 32: no kernel instantiation
        ops.fully_connected(z(33, 8), z(8, 256), None, None)
    for B, K in ((32, 385), (24, 513), (1, 12289)):                      # B * K * 4 bytes > 48 KB of shared memory
        with pytest.raises(RenderNetCudaError, match="rc=-3"):
            ops.fully_connected(z(B, K), z(K, 256), None, None)


# ----------------------------------------------------------------------------------------------------- conv3d_small
def _conv_ref(x, w, b, a, stride, transposed):
    y = (orc.conv3d_transpose if transposed else orc.conv3d)(x, w, b, (stride,) * 3, dtype=F64)
    return orc.prelu(y, a, dtype=F64)


def _conv_case(B, shape, cin, cout, k, stride, transposed, seed, scale=0.1):
    rng = np.random.default_rng(seed)
    wshape = (k, k, k, cout, cin) if transposed else (k, k, k, cin, cout)
    x = torch.from_numpy(rng.standard_normal((B,) + tuple(shape) + (cin,)).astype(np.float32)).to(dev)
    w = torch.from_numpy((rng.standard_normal(wshape) * scale).astype(np.float32)).to(dev)
    b = torch.from_numpy((rng.standard_normal(cout) * 0.1).astype(np.float32)).to(dev)
    a = torch.from_numpy(rng.uniform(-0.5, 1.5, cout).astype(np.float32)).to(dev)
    return x, w, b, a


def _check_conv(label, x, w, b, a, stride, transposed, formats=True):
    """fp32 in/out vs float64; 16-bit inputs (fp32 out vs float64 of the rounded input, 16-bit out vs the rounded fp32 out);
    fp32 in with 16-bit out.  Returns the fp32 output and the fp32-input error."""
    from rendernet_b200 import ops
    conv = lambda xx, **kw: ops.conv3d_small(xx, w, b, a, stride, transposed, **kw)                # noqa: E731
    cpu = [t.cpu() for t in (w, b, a)]
    got = conv(x)
    ref = _conv_ref(x.cpu(), *cpu, stride, transposed)
    assert got.shape == ref.shape, (label, got.shape, ref.shape)
    err = _rel(got, ref)
    print(f"{label}: fp32 in/out {err:.2e}, last item {_rel(got[-1], ref[-1]):.2e}")
    assert err < BAR_CONV, label
    if not formats:
        return got, err
    for fmt, name in FMT_NAMES.items():
        x16 = _to16(x, fmt)
        got16in = conv(x16)
        e16 = _rel(got16in, _conv_ref(x16.float().cpu(), *cpu, stride, transposed))
        print(f"{label}: {name} in, fp32 out {e16:.2e}")
        assert e16 < BAR_CONV, (label, name)
        _same16(conv(x16, want32=False), got16in, fmt, f"{label} {name} in/out")
        _same16(conv(x, want32=False, fmt=fmt), got, fmt, f"{label} fp32 in, {name} out")
    return got, err


CONV_CASES = [(ci, co, k, s, t) for ci, co in ((4, 4), (4, 8), (8, 4), (2, 3)) for k in (3, 4) for s in (1, 2)
              for t in (False, True)]


@pytest.mark.parametrize("cin,cout,k,stride,transposed", CONV_CASES,
                         ids=[f"{ci}to{co}-k{k}-s{s}-{'T' if t else 'F'}" for ci, co, k, s, t in CONV_CASES])
def test_conv3d_small_instantiations(cin, cout, k, stride, transposed):
    """Every channel instantiation, forward and transposed, strides 1 and 2, 3^3 and 4^3 filters, on a non-cubic grid whose sizes
    are odd and not multiples of 8 (the generic kernel), B = 3; fp32 and all three 16-bit formats in and out."""
    x, w, b, a = _conv_case(3, (9, 7, 11), cin, cout, k, stride, transposed, seed=cin * 100 + cout * 10 + k + stride)
    _check_conv(f"{cin}->{cout} k{k} s{stride} {'transposed' if transposed else 'forward'}", x, w, b, a, stride, transposed)


def test_conv3d_small_unequal_pads_and_rejections():
    """Forward SAME on a non-cubic grid is supported when every dimension gets the same pad-before (4^3 stride 2: 1 for odd
    and even sizes) and rejected otherwise (3^3 stride 2: 1 for odd, 0 for even sizes; rc -2).  Channel pairs without an
    instantiation are rc -4, filters beyond 48 KB of shared memory rc -3."""
    from rendernet_b200 import ops
    from rendernet_b200._lib import RenderNetCudaError
    x, w, b, a = _conv_case(2, (9, 6, 12), 4, 8, 4, 2, False, seed=7)
    _check_conv("4->8 k4 s2 forward on 9x6x12", x, w, b, a, 2, False, formats=False)
    x, w, b, a = _conv_case(2, (9, 6, 12), 4, 8, 3, 2, False, seed=8)
    with pytest.raises(RenderNetCudaError, match="rc=-2"):
        ops.conv3d_small(x, w, b, a, 2, False)
    z = lambda *s: torch.zeros(s, device=dev)                                                         # noqa: E731
    for cin, cout in ((3, 3), (8, 8), (4, 2), (1, 4)):
        for t in (False, True):
            with pytest.raises(RenderNetCudaError, match="rc=-4"):
                ops.conv3d_small(z(1, 4, 4, 4, cin), z(3, 3, 3, *((cout, cin) if t else (cin, cout))), None, None, 1, t)
    with pytest.raises(RenderNetCudaError, match="rc=-3"):                # 8^3 * 8 * 4 * 4 B = 64 KB
        ops.conv3d_small(z(1, 8, 8, 8, 8), z(8, 8, 8, 8, 4), None, None, 1, False)
    with pytest.raises(TypeError):                                       # one 16-bit format in and out: fp16 in, bf16 out
        ops.conv3d_small(z(1, 4, 4, 4, 4).half(), z(3, 3, 3, 4, 4), None, None, 1, False, want32=False, fmt=1)


DECODER_LAYERS = {"e_tex_conv0": ("conv3d_transpose", 4, 4, 1, True, 32), "e_tex_conv1": ("conv3d_transpose", 4, 8, 2, True, 32),
                  "e_tex_conv2": ("conv3d", 8, 4, 1, False, 64)}


@pytest.mark.parametrize("layer", list(DECODER_LAYERS))
def test_conv3d_small_decoder_layers_b24(layer):
    """The decoder's three convolutions at B = 24 with the seeded decoder weights (e_tex_conv2 in fp32 runs the tiled kernel);
    fp32 vs float64, the last item reported on its own, and the three 16-bit outputs (the generic kernel) vs the rounded fp32."""
    from rendernet_b200 import ops
    kind, cin, cout, stride, transposed, n = DECODER_LAYERS[layer]
    W = _weights()
    p = f"texture_encoder/{layer}/{kind}"
    w, b = (torch.from_numpy(W[f"{p}/{v}"]).to(dev) for v in ("weights", "biases"))
    a = torch.from_numpy(W[f"texture_encoder/{layer}/alpha"]).to(dev)
    x = torch.from_numpy(np.random.default_rng(20).standard_normal((24, n, n, n, cin)).astype(np.float32)).to(dev)
    got, _ = _check_conv(f"{layer} B=24 {n}^3", x, w, b, a, stride, transposed, formats=False)
    for fmt, name in FMT_NAMES.items():
        _same16(ops.conv3d_small(x, w, b, a, stride, transposed, want32=False, fmt=fmt), got, fmt, f"{layer} {name} out")


# ----------------------------------------------------------------------------------------------------- tiled vs generic
_CHILD = r"""
import sys
import torch
sys.path.insert(0, sys.argv[1])
from rendernet_b200 import ops
d = torch.load(sys.argv[2])
args = [d[k].cuda() for k in ("x", "w", "b", "a")]
with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]) as prof:
    y = ops.conv3d_small(*args, 1, False)
    torch.cuda.synchronize()
torch.save({"y": y.cpu(), "kernels": sorted({e.key for e in prof.key_averages()})}, sys.argv[3])
"""


def _kernels_of(fn):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    return out, sorted({e.key for e in prof.key_averages()})


@pytest.mark.parametrize("B,H,W,D", [(24, 64, 64, 64), (3, 16, 24, 40)])
def test_tiled_tex_conv_bit_identical_to_generic(tmp_path, B, H, W, D):
    """e_tex_conv2 (4^3 conv 8 -> 4, stride 1) by conv3d_k4_8to4_tiled_kernel in this process and by conv3d_small_kernel<8,4>
    in a child process with RN_TUNE=tiled_tex_conv=0 (read once per process): equal bit for bit.  At the bench's B = 24 on 64^3,
    and at B = 3 on 16 x 24 x 40, where a tile index split that mixes up y, x and z or the batch would show.  The profiler
    confirms which kernel each process ran."""
    from rendernet_b200 import ops
    Wt = _weights()
    p = "texture_encoder/e_tex_conv2"
    w, b, a = (torch.from_numpy(Wt[n]) for n in (f"{p}/conv3d/weights", f"{p}/conv3d/biases", f"{p}/alpha"))
    x = torch.from_numpy(np.random.default_rng(21).standard_normal((B, H, W, D, 8)).astype(np.float32))
    torch.save({"x": x, "w": w, "b": b, "a": a}, tmp_path / "in.pt")
    tiled, names = _kernels_of(lambda: ops.conv3d_small(x.to(dev), w.to(dev), b.to(dev), a.to(dev), 1, False))
    assert any("conv3d_k4_8to4_tiled_kernel" in n for n in names), names
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", _CHILD, ROOT, str(tmp_path / "in.pt"),
                                                                         str(tmp_path / "out.pt")]
    r = subprocess.run(cmd, env=dict(os.environ, RN_TUNE="tiled_tex_conv=0"), capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    child = torch.load(tmp_path / "out.pt")
    assert any("conv3d_small_kernel<8, 4>" in n for n in child["kernels"]), child["kernels"]
    assert not any("tiled" in n for n in child["kernels"]), child["kernels"]
    generic, tiled = child["y"], tiled.cpu()
    diff = generic != tiled
    print(f"tiled vs generic B={B} {H}x{W}x{D}: {int(diff.sum())} of {diff.numel()} values differ")
    assert torch.equal(generic, tiled)
    if B == 3:
        err = _rel(tiled, _conv_ref(x, w, b, a, 1, False))
        print(f"tiled B=3 16x24x40 vs float64: {err:.2e}")
        assert err < BAR_CONV


# ----------------------------------------------------------------------------------------------------- whole decoder
def _decode(W, z):
    from rendernet_b200 import tfcompat as tf
    from rendernet_b200.RenderNet_Texture_Face_Normal import decoder_texture
    with tf.use_store(tf.VariableStore(precision="exact")):
        tf.load_weight_dict(W)
        return tf.realize(decoder_texture(torch.from_numpy(np.ascontiguousarray(z)).to(dev))).cpu()


@pytest.fixture(scope="module")
def decoder24():
    import bench
    W = _weights()
    z = bench.synthetic_texture(24)
    return dict(W=W, z=z, tex=_decode(W, z), ref=orc.decoder_texture(z, W, dtype=F64))


def test_decoder_b24_vs_float64(decoder24):
    """decoder_texture at B = 24 on the bench's texture vectors (bench.synthetic_texture), every voxel vs the float64 decoder, item
    by item (the last item on its own: end-of-batch indexing); and the same items decoded at B = 8 (fc_kernel<8>) and B = 1 equal
    the B = 24 decode (fc_kernel<32>) bit for bit."""
    W, z, tex, ref = (decoder24[k] for k in ("W", "z", "tex", "ref"))
    assert tuple(tex.shape) == (24, 64, 64, 64, 4) and tex.dtype == torch.float32
    errs = [_rel(tex[i], ref[i]) for i in range(24)]
    print(f"decoder B=24 vs float64: all {_rel(tex, ref):.2e}, worst item {max(errs):.2e} (item {int(np.argmax(errs))}), "
          f"item 23 {errs[23]:.2e}")
    assert max(errs) < BAR_DECODER and errs[23] < BAR_DECODER
    assert torch.equal(_decode(W, z[16:24]), tex[16:24])
    assert torch.equal(_decode(W, z[23:24]), tex[23:24])


def test_decoder_bars_discriminate(decoder24):
    """The decoder bar catches a reference built from fp16-rounded decoder weights (what a kernel that silently read 16-bit
    weights computes) and one whose item 23 decodes item 22's texture vector.  Measured: 1.7e-4 (57x the bar) and 0.33."""
    W, z, tex, ref = (decoder24[k] for k in ("W", "z", "tex", "ref"))
    W16 = {k: (v.astype(np.float16).astype(np.float32) if k.startswith("texture_encoder") and k.endswith("/weights") else v)
           for k, v in W.items()}
    ref16 = orc.decoder_texture(z[[0, 23]], W16, dtype=F64)
    for j, i in enumerate((0, 23)):
        e = _rel(tex[i], ref16[j])
        print(f"item {i} vs float64 decoder with fp16-rounded weights: {e:.2e} ({e / BAR_DECODER:.0f}x the bar)")
        assert e > 10 * BAR_DECODER
    e = _rel(tex[23], ref[22])       # the decoder maps each item on its own: item 22's vector in slot 23 decodes to ref[22]
    print(f"item 23 vs float64 decode of item 22's vector: {e:.2e} ({e / BAR_DECODER:.0f}x the bar)")
    assert e > 10 * BAR_DECODER


# ----------------------------------------------------------------------------------------------------- engine at B = 24
@pytest.fixture(scope="module")
def bench_inputs():
    import bench
    vox, poses = bench.synthetic_batch(24)
    W = _weights()
    tex = bench.synthetic_texture(24)
    ref = orc.render_forward_texture(vox[[0, 23]], tex[[0, 23]], poses[[0, 23]], W)
    return W, vox, tex, poses, [r.numpy() for r in ref]


def _equal(got, want, label):
    d = got != want
    if d.any():
        items = sorted({int(i) for i in d.nonzero()[:, 0]})
        print(f"{label}: {int(d.sum())} values differ, items {items}, max |diff| {float((got - want).abs().max()):.3e}")
    assert not d.any(), label


@pytest.mark.parametrize("precision", ["exact", "fast"])
def test_engine_b24_equals_shards_and_single_renders(bench_inputs, precision):
    """TextureRenderEngine(B = 24) on the bench's own inputs (bench.synthetic_batch / synthetic_texture) equals three B = 8 shards
    and B = 1 renders of items 0, 9 and 23, bit for bit (B = 24 decodes through fc_kernel<32>, B = 8 and B = 1 through
    fc_kernel<8>); submit/result equals render; items 0 and 23 meet config 4's bars against the oracle (exact 1e-3, fast 5e-3;
    measured exact 2.7e-5, fast 2.2e-3)."""
    from rendernet_b200.engine import TextureRenderEngine
    W, vox, tex, poses, (ref_img, ref_nrm) = bench_inputs
    eng = TextureRenderEngine(W, 24, precision=precision)
    img, nrm = (t.clone() for t in eng.render(vox, tex, poses))
    assert tuple(img.shape) == tuple(nrm.shape) == (24, 512, 512, 3)
    got = eng.result(eng.submit(vox, tex, poses))
    _equal(got[0], img, "submit/result albedo"); _equal(got[1], nrm, "submit/result normal")
    del eng
    torch.cuda.empty_cache()
    eng = TextureRenderEngine(W, 8, precision=precision)
    for s in range(3):
        sl = slice(8 * s, 8 * s + 8)
        a, n = eng.render(vox[sl], tex[sl], poses[sl])
        _equal(a, img[sl], f"B=8 shard {s} albedo"); _equal(n, nrm[sl], f"B=8 shard {s} normal")
    del eng
    eng = TextureRenderEngine(W, 1, precision=precision)
    for i in (0, 9, 23):
        a, n = eng.render(vox[i:i + 1], tex[i:i + 1], poses[i:i + 1])
        _equal(a, img[i:i + 1], f"B=1 item {i} albedo"); _equal(n, nrm[i:i + 1], f"B=1 item {i} normal")
    del eng
    torch.cuda.empty_cache()
    bar = 1e-3 if precision == "exact" else 5e-3
    for j, i in enumerate((0, 23)):
        e1 = float(np.abs(img[i].numpy() - ref_img[j]).max())
        e2 = float(np.abs(nrm[i].numpy() - ref_nrm[j]).max())
        print(f"engine B=24 [{precision}] item {i} vs oracle: albedo {e1:.3e}, normal {e2:.3e} (bar {bar:g})")
        assert e1 <= bar and e2 <= bar
