"""CPU oracle for RenderNet's forward rendering hot path.  TEST INFRASTRUCTURE ONLY.

This module is a CPU restatement (NumPy fp32 for the resampler / Phong / binvox,
PyTorch-CPU fp32 for the convolutions) of the reference's TF-1 graph.  It is the
*checker*: only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s
``cpu_baseline`` / ``--impl reference`` legs may import it.  Nothing under
``rendernet_b200/`` imports it, and the product path fails loudly without its CUDA
extension.

Pinning status: the reference ships no tests, no golden tensors and no weights, and
TensorFlow-1 cannot be installed here, so this restatement is pinned against
fixtures produced by executing the *reference's own Python source* (from
the reference source tree) over a NumPy shim of the TF-1 primitives it calls
(``oracle/tf1_shim.py`` + ``tests/golden/make_golden.py`` -> ``tests/golden/*.npz``).
TF's own C++ kernels remain unpinned ("parity pinned to reference Python over a TF
shim; TF kernels unpinned").

All file:line citations are into the reference source tree.
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Sequence, Tuple

import numpy as np

try:  # torch is only needed for the conv stack
    import torch
    import torch.nn.functional as F
except Exception:  # pragma: no cover
    torch = None
    F = None
_F32 = torch.float32 if torch is not None else None   # default arithmetic type of the conv stack


# ----------------------------------------------------------------------------------
# binvox reader  (tools/binvox_rw.py:45-93)
# ----------------------------------------------------------------------------------
def read_binvox_header(fp):
    """tools/binvox_rw.py:45-56."""
    line = fp.readline().strip()
    if not line.startswith(b"#binvox"):
        raise IOError("Not a binvox file")
    dims = list(map(int, fp.readline().strip().split(b" ")[1:]))
    translate = list(map(float, fp.readline().strip().split(b" ")[1:]))
    scale = list(map(float, fp.readline().strip().split(b" ")[1:]))[0]
    fp.readline()
    return dims, translate, scale


def read_binvox(fp, fix_coords: bool = True) -> np.ndarray:
    """RLE decode -> bool[dims]; xzy->xyz transpose.  tools/binvox_rw.py:58-93."""
    dims, _, _ = read_binvox_header(fp)
    raw = np.frombuffer(fp.read(), dtype=np.uint8)
    values, counts = raw[::2], raw[1::2]
    data = np.repeat(values, counts).astype(bool).reshape(dims)
    if fix_coords:
        data = np.transpose(data, (0, 2, 1))
    return data


# ----------------------------------------------------------------------------------
# pose  (RenderNet_demo.py:33-38)
# ----------------------------------------------------------------------------------
def compute_pose_param(azimuth: float, elevation: float, radius: float) -> np.ndarray:
    phi = azimuth * math.pi / 180.0
    theta = (90 - elevation) * math.pi / 180
    return np.expand_dims(np.array([phi, theta, 3.3 / radius]), axis=0)


# ----------------------------------------------------------------------------------
# resampler  (tools/resampling_voxel_grid.py:381-614, tools/model_util.py:41-49)
# ----------------------------------------------------------------------------------
def rotation_around_grid_centroid(view_params: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """resampling_voxel_grid.py:515-562.  fp32 throughout; always returns (R, S)
    because the `== 2` test at :551 is a Python `==` on a tensor (always False)."""
    vp = np.asarray(view_params, dtype=np.float32)
    B = vp.shape[0]
    az = vp[:, 0] - np.float32(math.pi * 0.5)                    # :529
    el = vp[:, 1]
    ca, sa = np.cos(az).astype(np.float32), np.sin(az).astype(np.float32)
    ce, se = np.cos(el).astype(np.float32), np.sin(el).astype(np.float32)
    rot_y = np.zeros((B, 4, 4), np.float32)                      # :537-541
    rot_y[:, 0, 0] = ca; rot_y[:, 0, 2] = -sa
    rot_y[:, 1, 1] = 1
    rot_y[:, 2, 0] = sa; rot_y[:, 2, 2] = ca
    rot_y[:, 3, 3] = 1
    rot_z = np.zeros((B, 4, 4), np.float32)                      # :544-548
    rot_z[:, 0, 0] = ce; rot_z[:, 0, 1] = se
    rot_z[:, 1, 0] = -se; rot_z[:, 1, 1] = ce
    rot_z[:, 2, 2] = 1
    rot_z[:, 3, 3] = 1
    R = np.matmul(rot_z, rot_y)                                  # :550
    S = np.zeros((B, 4, 4), np.float32)                          # :556-561
    s = vp[:, 2]
    S[:, 0, 0] = s; S[:, 1, 1] = s; S[:, 2, 2] = s; S[:, 3, 3] = 1
    return R, S


def inverse_total_matrix(R: np.ndarray, S: Optional[np.ndarray], size: int, new_size: int) -> np.ndarray:
    """resampling_voxel_grid.py:579-602: M = T_new_inv (S) R T ; return inv(M)[:, :3, :]."""
    B = R.shape[0]
    T = np.array([[1, 0, 0, -size * 0.5], [0, 1, 0, -size * 0.5],
                  [0, 0, 1, -size * 0.5], [0, 0, 0, 1]], np.float32)
    Tn = np.array([[1, 0, 0, new_size * 0.5], [0, 1, 0, new_size * 0.5],
                   [0, 0, 1, new_size * 0.5], [0, 0, 0, 1]], np.float32)
    T = np.tile(T[None], (B, 1, 1)); Tn = np.tile(Tn[None], (B, 1, 1))
    if S is None:
        M = np.matmul(np.matmul(Tn, R), T)
    else:
        M = np.matmul(np.matmul(np.matmul(Tn, S), R), T)
    Minv = np.linalg.inv(M.astype(np.float32)).astype(np.float32)
    return Minv[:, 0:3, :]


def interpolate(voxel: np.ndarray, x: np.ndarray, y: np.ndarray, z: np.ndarray) -> np.ndarray:
    """tf_interpolate, resampling_voxel_grid.py:381-486.  voxel [B,H,W,D,C]; x,y,z flat
    over (B * n_points).  Returns [B*n_points, C] fp32."""
    B, H, W, D, C = voxel.shape
    n = x.size // B
    x = x.astype(np.float32); y = y.astype(np.float32); z = z.astype(np.float32)
    x0 = np.floor(x).astype(np.int32); x1 = x0 + 1
    y0 = np.floor(y).astype(np.int32); y1 = y0 + 1
    z0 = np.floor(z).astype(np.int32); z1 = z0 + 1
    x0 = np.clip(x0, 0, W - 1); x1 = np.clip(x1, 0, W - 1)        # :417-422 (max_x = width-1)
    y0 = np.clip(y0, 0, H - 1); y1 = np.clip(y1, 0, H - 1)
    z0 = np.clip(z0, 0, D - 1); z1 = np.clip(z1, 0, D - 1)
    base = np.repeat(np.arange(B, dtype=np.int64) * W * H * D, n)   # :427
    base_z0 = base + z0 * W * H; base_z1 = base + z1 * W * H        # :430-431
    b00 = base_z0 + y0 * W; b01 = base_z0 + y1 * W
    b10 = base_z1 + y0 * W; b11 = base_z1 + y1 * W
    idx = [b00 + x0, b01 + x0, b00 + x1, b01 + x1,                   # a b c d  (:440-443)
           b10 + x0, b11 + x0, b10 + x1, b11 + x1]                   # e f g h  (:446-449)
    flat = voxel.reshape(-1, C).astype(np.float32)
    x0f, x1f = x0.astype(np.float32), x1.astype(np.float32)
    y0f, y1f = y0.astype(np.float32), y1.astype(np.float32)
    z0f, z1f = z0.astype(np.float32), z1.astype(np.float32)
    w = [(x1f - x) * (y1f - y) * (z1f - z), (x1f - x) * (y - y0f) * (z1f - z),
         (x - x0f) * (y1f - y) * (z1f - z), (x - x0f) * (y - y0f) * (z1f - z),
         (x1f - x) * (y1f - y) * (z - z0f), (x1f - x) * (y - y0f) * (z - z0f),
         (x - x0f) * (y1f - y) * (z - z0f), (x - x0f) * (y - y0f) * (z - z0f)]
    out = w[0][:, None] * flat[idx[0]]
    for k in range(1, 8):                                            # add_n order a..h (:485)
        out = out + w[k][:, None] * flat[idx[k]]
    return out.astype(np.float32)


def voxel_meshgrid(height: int, width: int, depth: int) -> np.ndarray:
    """tf_voxel_meshgrid homogeneous=True, resampling_voxel_grid.py:488-513.
    Columns are (x=k, y=j, z=i, 1) for flat index n = i*H*W + j*W + k."""
    z_t, y_t, x_t = np.meshgrid(np.arange(depth, dtype=np.float32),
                                np.arange(height, dtype=np.float32),
                                np.arange(width, dtype=np.float32), indexing="ij")
    g = np.stack([x_t.reshape(-1), y_t.reshape(-1), z_t.reshape(-1),
                  np.ones(x_t.size, np.float32)], axis=0)
    return g


def resampling(voxel: np.ndarray, R: np.ndarray, S: Optional[np.ndarray] = None,
               size: int = 64, new_size: int = 128) -> np.ndarray:
    """tf_resampling, resampling_voxel_grid.py:564-614 (the vestigial `params` arg dropped)."""
    voxel = np.asarray(voxel, np.float32)
    B = voxel.shape[0]; C = voxel.shape[4]
    Minv = inverse_total_matrix(R, S, size, new_size)
    grid = voxel_meshgrid(new_size, new_size, new_size)
    pts = np.matmul(Minv, grid[None])                               # [B,3,N]   :605
    out = interpolate(voxel, pts[:, 0].reshape(-1), pts[:, 1].reshape(-1), pts[:, 2].reshape(-1))
    return out.reshape(B, new_size, new_size, new_size, C)


def rotation_resampling(voxel: np.ndarray, view_params: np.ndarray, size: int = 64,
                        new_size: int = 128) -> np.ndarray:
    """tf_rotation_resampling, resampling_voxel_grid.py:616-632."""
    R, S = rotation_around_grid_centroid(view_params)
    return resampling(voxel, R, S, size=size, new_size=new_size)


def transform_voxel_to_match_image(t: np.ndarray) -> np.ndarray:
    """tools/model_util.py:41-49: transpose (0,2,1,3,4) then reverse axis 1."""
    if torch is not None and isinstance(t, torch.Tensor):
        return torch.flip(t.permute(0, 2, 1, 3, 4), dims=(1,))
    return np.transpose(t, (0, 2, 1, 3, 4))[:, ::-1]


# ----------------------------------------------------------------------------------
# layer ops  (tools/layer_util.py) -- channel-last torch tensors, fp32, TF SAME rules
# ----------------------------------------------------------------------------------
def same_pads(n_in: int, k: int, s: int) -> Tuple[int, int]:
    """TF SAME: out=ceil(in/s); total=max((out-1)*s+k-in,0); before=total//2."""
    out = -(-n_in // s)
    total = max((out - 1) * s + k - n_in, 0)
    return total // 2, total - total // 2


def _t(x):
    return x if isinstance(x, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(x))


def conv3d(x, w, b=None, stride=(1, 1, 1), dtype=_F32):
    """tf.nn.conv3d SAME + bias (layer_util.py:228-265).  x [B,D0,D1,D2,Cin], w [k0,k1,k2,Cin,Cout].
    dtype: arithmetic type (torch.float64 gives a high-precision reference of the same op)."""
    x = _t(x).to(dtype); w = _t(w).to(dtype)
    xs = x.permute(0, 4, 1, 2, 3)
    pads = []
    for d in (2, 1, 0):  # F.pad wants last dim first
        pb, pa = same_pads(x.shape[1 + d], w.shape[d], stride[d])
        pads += [pb, pa]
    y = F.conv3d(F.pad(xs, pads), w.permute(4, 3, 0, 1, 2).contiguous(), stride=tuple(stride))
    y = y.permute(0, 2, 3, 4, 1)
    if b is not None:
        y = y + _t(b).to(dtype)
    return y.contiguous()


def conv2d(x, w, b=None, stride=(1, 1)):
    """tf.nn.conv2d / slim.conv2d SAME + bias (layer_util.py:147-184).  x [B,H,W,Cin], w [kh,kw,Cin,Cout]."""
    x = _t(x).float(); w = _t(w).float()
    xs = x.permute(0, 3, 1, 2)
    pads = []
    for d in (1, 0):
        pb, pa = same_pads(x.shape[1 + d], w.shape[d], stride[d])
        pads += [pb, pa]
    y = F.conv2d(F.pad(xs, pads), w.permute(3, 2, 0, 1).contiguous(), stride=tuple(stride))
    y = y.permute(0, 2, 3, 1)
    if b is not None:
        y = y + _t(b).float()
    return y.contiguous()


def conv2d_transpose(x, w, b=None, stride=(1, 1)):
    """tf.nn.conv2d_transpose SAME, out = in*stride (layer_util.py:186-226).
    x [B,H,W,Cin], w [kh,kw,Cout,Cin].  Gradient of the forward SAME conv:
    y[o] += x[i] w[k], o = i*s + k - pb, pb = max(k-s,0)//2."""
    x = _t(x).float(); w = _t(w).float()
    B, H, W, _ = x.shape
    kh, kw = w.shape[0], w.shape[1]
    full = F.conv_transpose2d(x.permute(0, 3, 1, 2), w.permute(3, 2, 0, 1).contiguous(), stride=tuple(stride))
    pbh = max(kh - stride[0], 0) // 2
    pbw = max(kw - stride[1], 0) // 2
    y = full[:, :, pbh:pbh + H * stride[0], pbw:pbw + W * stride[1]].permute(0, 2, 3, 1)
    if b is not None:
        y = y + _t(b).float()
    return y.contiguous()


def conv3d_transpose(x, w, b=None, stride=(1, 1, 1), dtype=_F32):
    """tf.nn.conv3d_transpose SAME (layer_util.py:269-309).  w [k0,k1,k2,Cout,Cin]; dtype as in conv3d."""
    x = _t(x).to(dtype); w = _t(w).to(dtype)
    B, D0, D1, D2, _ = x.shape
    full = F.conv_transpose3d(x.permute(0, 4, 1, 2, 3), w.permute(4, 3, 0, 1, 2).contiguous(), stride=tuple(stride))
    pb = [max(w.shape[d] - stride[d], 0) // 2 for d in range(3)]
    y = full[:, :, pb[0]:pb[0] + D0 * stride[0], pb[1]:pb[1] + D1 * stride[1], pb[2]:pb[2] + D2 * stride[2]]
    y = y.permute(0, 2, 3, 4, 1)
    if b is not None:
        y = y + _t(b).to(dtype)
    return y.contiguous()


def fully_connected(x, w, b=None, dtype=_F32):
    """layer_util.py:311-343; dtype as in conv3d."""
    y = _t(x).to(dtype) @ _t(w).to(dtype)
    if b is not None:
        y = y + _t(b).to(dtype)
    return y


def prelu(x, alpha, dtype=_F32):
    """layer_util.py:27-45: max(0,x) + alpha*min(0,x), alpha per last-axis channel; dtype as in conv3d."""
    x = _t(x).to(dtype); a = _t(np.asarray(alpha, np.float32)) if not isinstance(alpha, torch.Tensor) else alpha
    return torch.clamp(x, min=0) + a.to(dtype) * torch.clamp(x, max=0)


def projection_unit(x, w, b, alpha):
    """layer_util.py:8-22: reshape [B,H,W,D,C]->[B,H,W,D*C] (f=d*C+c), 1x1 conv, PReLU."""
    x = _t(x).float()
    B, H, W, D, C = x.shape
    return prelu(conv2d(x.reshape(B, H, W, D * C), w, b), alpha)


# ----------------------------------------------------------------------------------
# weights: names follow the TF variable scopes (RenderNet_Shader.py:33-129,
# layer_util.py:17,35-36,68-71,142,158-161,238-241)
# ----------------------------------------------------------------------------------
def xavier_uniform(rng: np.random.Generator, shape: Sequence[int], fan_in: int, fan_out: int, gain: float = 1.0):
    limit = gain * math.sqrt(6.0 / (fan_in + fan_out))
    return rng.uniform(-limit, limit, size=shape).astype(np.float32)


def shader_layer_specs(is_greyscale: bool = False, width: int = 32, depth: int = 32):
    """(name, kind, filter shape, bias_init, has_alpha) for every variable group of the
    Shader net.  `width`/`depth` exist only so tests can build narrow nets; the
    reference is width=32 (3-D channels), depth=32 (-> 1024 features)."""
    c1, c2, c3 = width // 4, width // 2, width
    F_ = c3 * depth
    specs = []
    specs.append(("encoder/e_conv1/e_conv1", "conv3d", (5, 5, 5, 1, c1), 0.001, "encoder/e_conv1"))
    specs.append(("encoder/e_conv2/e_conv2", "conv3d", (3, 3, 3, c1, c2), 0.001, "encoder/e_conv2"))
    specs.append(("encoder/e_conv3/e_conv3", "conv3d", (3, 3, 3, c2, c3), 0.001, "encoder/e_conv3"))
    for k in range(1, 11):
        specs.append((f"encoder/res1_{k}/con1_3X3", "conv3d", (3, 3, 3, c3, c3), 0.001, f"encoder/res1_{k}"))
        specs.append((f"encoder/res1_{k}/conv2_3x3", "conv3d", (3, 3, 3, c3, c3), 0.001, None))
    specs.append(("encoder/res1_skip/con1_3X3", "conv3d", (3, 3, 3, c3, c3), 0.001, None))
    specs.append(("encoder/projection_unit/Conv", "conv2d", (1, 1, F_, F_), 0.0, "encoder/projection_unit"))
    for k in range(1, 11):
        specs.append((f"encoder/res2_{k}/con1_3X3", "conv2d", (3, 3, F_, F_), 0.0, f"encoder/res2_{k}"))
        specs.append((f"encoder/res2_{k}/conv2_3x3", "conv2d", (3, 3, F_, F_), 0.0, None))
    specs.append(("encoder/res2_skip/con1_3X3", "conv2d", (3, 3, F_, F_), 0.0, None))
    specs.append(("encoder/e_conv5/e_conv5", "conv2d", (4, 4, F_, F_ // 2), 0.0, "encoder/e_conv5"))
    for k in range(1, 6):
        specs.append((f"encoder/res3_{k}/con1_3X3", "conv2d", (3, 3, F_ // 2, F_ // 2), 0.0, f"encoder/res3_{k}"))
        specs.append((f"encoder/res3_{k}/conv2_3x3", "conv2d", (3, 3, F_ // 2, F_ // 2), 0.0, None))
    specs.append(("encoder/res3_skip/con1_3X3", "conv2d", (3, 3, F_ // 2, F_ // 2), 0.0, None))
    specs.append(("encoder/e_conv6/e_conv6", "conv2d", (4, 4, F_ // 2, F_ // 4), 0.0, "encoder/e_conv6"))
    chain = [("e_conv7", F_ // 4, F_ // 8), ("e_conv7_1", F_ // 8, F_ // 8), ("e_conv8", F_ // 8, F_ // 16),
             ("e_conv9", F_ // 16, F_ // 32), ("e_conv10", F_ // 32, F_ // 64)]
    for nm, cin, cout in chain:
        specs.append((f"encoder/{nm}/{nm}", "conv2d_transpose", (4, 4, cout, cin), 0.0, f"encoder/{nm}"))
    cout = 1 if is_greyscale else 3
    # e_conv11 is created directly under "encoder" (RenderNet_Shader.py:125-129)
    specs.append(("encoder/e_conv11", "conv2d_transpose", (4, 4, cout, F_ // 64), 0.0, None))
    return specs


def _fans(kind: str, shape: Sequence[int]) -> Tuple[int, int]:
    rf = int(np.prod(shape[:-2]))
    return rf * shape[-2], rf * shape[-1]   # TF xavier: fan_in=rf*shape[-2], fan_out=rf*shape[-1]


def init_shader_weights(seed: int = 0, is_greyscale: bool = False, width: int = 32, depth: int = 32,
                        alpha_range: Tuple[float, float] = (0.0, 0.0), gain: float = 1.0,
                        bias_jitter: float = 0.0) -> Dict[str, np.ndarray]:
    """Seeded weights following the reference initialisers (xavier-uniform weights,
    bias 0.001 for layer_util convs / 0 for slim convs, alpha 0).  `alpha_range`,
    `gain`, `bias_jitter` let parity tests use non-degenerate PReLU slopes, unsaturated
    logits and non-constant biases."""
    rng = np.random.default_rng(seed)
    W: Dict[str, np.ndarray] = {}
    for name, kind, shape, bias0, alpha_scope in shader_layer_specs(is_greyscale, width, depth):
        fi, fo = _fans(kind, shape)
        W[name + "/weights"] = xavier_uniform(rng, shape, fi, fo, gain)
        nb = shape[-2] if kind == "conv2d_transpose" else shape[-1]
        bias = np.full((nb,), bias0, np.float32)
        if bias_jitter > 0.0:
            bias = bias + (rng.standard_normal(nb) * bias_jitter).astype(np.float32)
        W[name + "/biases"] = bias
        if alpha_scope is not None:
            lo, hi = alpha_range
            W[alpha_scope + "/alpha"] = (rng.uniform(lo, hi, size=nb).astype(np.float32)
                                         if hi > lo else np.full((nb,), lo, np.float32))
    return W


# ----------------------------------------------------------------------------------
# Shader model fn  (RenderNet_Shader.py:32-131), inference (dropout identity)
# ----------------------------------------------------------------------------------
def rendernet_shader(models_in, W: Dict[str, np.ndarray], return_stages: bool = False, dropout=None):
    """models_in [B,H,W,128,1] (already resampled + axis-transformed).  Returns the
    sigmoid image [B,4H,4W,3|1]; with return_stages also a dict of stage tensors.
    dropout: None (inference, keep_prob 1) or callable(call_index, tensor) -> tensor applied at the ten tf.nn.dropout sites of
    RenderNet_Shader.py:39,43,47,88,103,107,111,115,119,123 in graph order (the training graph; the caller supplies the masks)."""
    g = lambda n: W[n]
    st = {}
    calls = [0]

    def drop(t):
        if dropout is None:
            return t
        t = dropout(calls[0], t)
        calls[0] += 1
        return t

    def c3(x, scope, stride=(1, 1, 1)):
        return conv3d(x, g(scope + "/weights"), g(scope + "/biases"), stride)

    def c2(x, scope):
        return conv2d(x, g(scope + "/weights"), g(scope + "/biases"))

    def ct(x, scope, s):
        return conv2d_transpose(x, g(scope + "/weights"), g(scope + "/biases"), (s, s))

    x = _t(models_in).float()
    enc1 = drop(prelu(c3(x, "encoder/e_conv1/e_conv1", (2, 2, 2)), g("encoder/e_conv1/alpha")))      # :36-39
    enc2 = drop(prelu(c3(enc1, "encoder/e_conv2/e_conv2", (1, 1, 2)), g("encoder/e_conv2/alpha")))   # :40-43
    enc3 = drop(prelu(c3(enc2, "encoder/e_conv3/e_conv3"), g("encoder/e_conv3/alpha")))              # :44-47
    st["enc1"], st["enc2"], st["enc3"] = enc1, enc2, enc3
    h = enc3
    for k in range(1, 11):                                                                     # :51-60
        t = prelu(c3(h, f"encoder/res1_{k}/con1_3X3"), g(f"encoder/res1_{k}/alpha"))
        h = c3(t, f"encoder/res1_{k}/conv2_3x3") + h
    enc3_skip = c3(h, "encoder/res1_skip/con1_3X3") + enc3                                     # :62-64
    st["enc3_skip"] = enc3_skip
    enc4 = projection_unit(enc3_skip, g("encoder/projection_unit/Conv/weights"),
                           g("encoder/projection_unit/Conv/biases"), g("encoder/projection_unit/alpha"))  # :67
    st["enc4"] = enc4
    h = enc4
    for k in range(1, 11):                                                                     # :71-80
        t = prelu(c2(h, f"encoder/res2_{k}/con1_3X3"), g(f"encoder/res2_{k}/alpha"))
        h = c2(t, f"encoder/res2_{k}/conv2_3x3") + h
    enc4_skip = c2(h, "encoder/res2_skip/con1_3X3") + enc4                                     # :82-84
    st["enc4_skip"] = enc4_skip
    enc5 = drop(prelu(c2(enc4_skip, "encoder/e_conv5/e_conv5"), g("encoder/e_conv5/alpha")))         # :86-88
    st["enc5"] = enc5
    h = enc5
    for k in range(1, 6):                                                                      # :91-95
        t = prelu(c2(h, f"encoder/res3_{k}/con1_3X3"), g(f"encoder/res3_{k}/alpha"))
        h = c2(t, f"encoder/res3_{k}/conv2_3x3") + h
    enc5_skip = c2(h, "encoder/res3_skip/con1_3X3") + enc5                                     # :97-99
    st["enc5_skip"] = enc5_skip
    enc6 = drop(prelu(c2(enc5_skip, "encoder/e_conv6/e_conv6"), g("encoder/e_conv6/alpha")))         # :101-103
    enc7 = drop(prelu(ct(enc6, "encoder/e_conv7/e_conv7", 2), g("encoder/e_conv7/alpha")))           # :105-107
    enc7_1 = drop(prelu(ct(enc7, "encoder/e_conv7_1/e_conv7_1", 1), g("encoder/e_conv7_1/alpha")))   # :109-111
    enc8 = drop(prelu(ct(enc7_1, "encoder/e_conv8/e_conv8", 2), g("encoder/e_conv8/alpha")))         # :113-115
    enc9 = drop(prelu(ct(enc8, "encoder/e_conv9/e_conv9", 2), g("encoder/e_conv9/alpha")))           # :117-119
    enc10 = drop(prelu(ct(enc9, "encoder/e_conv10/e_conv10", 1), g("encoder/e_conv10/alpha")))       # :121-123
    st["enc6"], st["enc7"], st["enc7_1"], st["enc8"], st["enc9"], st["enc10"] = enc6, enc7, enc7_1, enc8, enc9, enc10
    logits = ct(enc10, "encoder/e_conv11", 1)                                                  # :125-129
    st["logits"] = logits
    out = torch.sigmoid(logits)                                                                # :127,130
    if return_stages:
        return out, st
    return out


def render_forward(voxel: np.ndarray, view_params: np.ndarray, W: Dict[str, np.ndarray],
                   return_stages: bool = False):
    """Whole graph of RenderNet_Shader.py:139-156 at inference: resample -> axis
    transform -> RenderNet."""
    rot = rotation_resampling(voxel, view_params)
    rot = np.ascontiguousarray(transform_voxel_to_match_image(rot))
    res = rendernet_shader(rot, W, return_stages=return_stages)
    if return_stages:
        res[1]["rotated"] = torch.from_numpy(rot)
    return res


# ----------------------------------------------------------------------------------
# Phong composite (NumPy path of the demo)  tools/Phong_shading.py:138-228,247-253
# ----------------------------------------------------------------------------------
def generate_light_pos(elevation=90, azimuth=90):
    elevation = (np.array([[elevation]])) * math.pi / 180.0
    azimuth = (np.array([[azimuth]])) * math.pi / 180.0
    x = np.multiply(-np.sin(elevation), np.cos(azimuth))
    y = np.cos(elevation)
    z = np.multiply(-np.sin(elevation), np.sin(azimuth))
    return np.hstack((x, y, z))


def np_mask(images_in):
    mask = np.linalg.norm(images_in, axis=3, keepdims=True)
    return 1.0 / (1.0 + np.exp(-(255.0 * mask - 150)))


def np_mask_white(images_in):
    mask = np.linalg.norm(1.0 - images_in, axis=3, keepdims=True)
    return 1.0 / (1.0 + np.exp(-(255.0 * mask - 80)))


def np_phong_shading(img_batch, light_dir, light_col, k_diffuse):
    """Phong_shading.py:162-200 (without mutating the caller's light_dir)."""
    normals_ish_vec = (img_batch - 0.5).reshape([-1, 3])
    normals_vec = normals_ish_vec / np.linalg.norm(normals_ish_vec, axis=1)[:, np.newaxis]
    light_dir = light_dir / np.linalg.norm(light_dir, axis=1).reshape([-1, 1])
    npx = int(np.prod(img_batch.shape[1:3]))
    light_dir = np.repeat(light_dir, npx, 0)
    light_col = np.repeat(light_col, npx, 0)
    diffuse_vec = np.maximum(np.sum(normals_vec * light_dir, axis=1, keepdims=True), 0.0)
    diffuse_col_vec = k_diffuse * np.multiply(np.repeat(diffuse_vec, 3, 1), light_col)
    return np.clip(diffuse_col_vec.reshape(img_batch.shape), 0, 1)


def np_phong_composite(images_in, light_dir, light_col, ambient_in, k_diffuse,
                       background_col="Black", with_mask=True):
    """Phong_shading.py:202-228."""
    diffuse = np_phong_shading(images_in, light_dir, light_col, k_diffuse)
    if with_mask:
        mask = np_mask(images_in) if background_col.lower() == "black" else np_mask_white(images_in)
        compos = mask * (ambient_in + diffuse) + (1 - mask)
    else:
        compos = ambient_in + diffuse
    return np.clip(compos, 0, 1)


def to_uint8(img_phong):
    """RenderNet_demo.py:58."""
    return np.clip(255.0 * img_phong, 0, 255).astype(np.uint8)


# ----------------------------------------------------------------------------------
# Texture + Normal network and texture decoder (BASELINE config 4)
# RenderNet_Texture_Face_Normal.py:34-147, graph wiring :155-179
# ----------------------------------------------------------------------------------
def texture_layer_specs():
    """(name, kind, filter shape, bias_init, alpha scope) of every variable group; scope quirks of the reference
    (SURVEY Appendix B.6: `e_conv7_1` block uses scope 'e_conv7_2', default 'conv2d_transpose' scopes) included."""
    sp = []
    te = "texture_encoder"
    sp.append((f"{te}/e_tex_fc1/fully_connected", "fc", (199, 32 * 32 * 32 * 4), 0.001, f"{te}/e_tex_fc1"))
    sp.append((f"{te}/e_tex_conv0/conv3d_transpose", "conv3d_transpose", (4, 4, 4, 4, 4), 0.001, f"{te}/e_tex_conv0"))
    sp.append((f"{te}/e_tex_conv1/conv3d_transpose", "conv3d_transpose", (4, 4, 4, 8, 4), 0.001, f"{te}/e_tex_conv1"))
    sp.append((f"{te}/e_tex_conv2/conv3d", "conv3d", (4, 4, 4, 8, 4), 0.001, f"{te}/e_tex_conv2"))
    e = "encoder"
    sp.append((f"{e}/e_conv1/e_conv1", "conv3d", (5, 5, 5, 5, 8), 0.001, f"{e}/e_conv1"))
    sp.append((f"{e}/e_conv2/e_conv2", "conv3d", (3, 3, 3, 8, 16), 0.001, f"{e}/e_conv2"))
    sp.append((f"{e}/e_conv3/e_conv3", "conv3d", (3, 3, 3, 16, 16), 0.001, f"{e}/e_conv3"))
    for k in range(1, 11):
        sp.append((f"{e}/res1_{k}/con1_3X3", "conv3d", (3, 3, 3, 16, 16), 0.001, f"{e}/res1_{k}"))
        sp.append((f"{e}/res1_{k}/conv2_3x3", "conv3d", (3, 3, 3, 16, 16), 0.001, None))
    sp.append((f"{e}/res1_skip/con1_3X3", "conv3d", (3, 3, 3, 16, 16), 0.001, None))
    sp.append((f"{e}/projection_unit/Conv", "conv2d", (1, 1, 512, 512), 0.0, f"{e}/projection_unit"))
    for k in range(1, 11):
        sp.append((f"{e}/res2_{k}/con1_3X3", "conv2d", (3, 3, 512, 512), 0.0, f"{e}/res2_{k}"))
        sp.append((f"{e}/res2_{k}/conv2_3x3", "conv2d", (3, 3, 512, 512), 0.0, None))
    sp.append((f"{e}/res2_skip/con1_3X3", "conv2d", (3, 3, 512, 512), 0.001, None))          # layer_util.conv2d
    sp.append((f"{e}/e_conv5/e_conv5", "conv2d", (4, 4, 512, 256), 0.001, f"{e}/e_conv5"))
    for k in range(1, 6):
        sp.append((f"{e}/res3_{k}/con1_3X3", "conv2d", (3, 3, 256, 256), 0.0, f"{e}/res3_{k}"))
        sp.append((f"{e}/res3_{k}/conv2_3x3", "conv2d", (3, 3, 256, 256), 0.0, None))
    sp.append((f"{e}/res3_skip/con1_3X3", "conv2d", (3, 3, 256, 256), 0.001, None))
    for head, sfx in (("Image", "1"), ("Normal", "2")):
        h = f"{e}/{head}"
        sp.append((f"{h}/e_conv6_{sfx}/e_conv6_{sfx}", "conv2d", (4, 4, 256, 128), 0.001, f"{h}/e_conv6_{sfx}"))
        if sfx == "1":   # Image head: scope quirks (:118-127)
            sp.append((f"{h}/e_conv7_1/e_conv7_2", "conv2d_transpose", (4, 4, 64, 128), 0.001, f"{h}/e_conv7_1"))
            sp.append((f"{h}/e_conv8_1/conv2d_transpose", "conv2d_transpose", (4, 4, 32, 64), 0.001, f"{h}/e_conv8_1"))
            sp.append((f"{h}/e_conv9_1/conv2d_transpose", "conv2d_transpose", (4, 4, 16, 32), 0.001, f"{h}/e_conv9_1"))
            sp.append((f"{h}/e_conv10_1/conv2d_transpose", "conv2d_transpose", (4, 4, 3, 16), 0.001, None))
        else:
            sp.append((f"{h}/e_conv7_2/e_conv7_2", "conv2d_transpose", (4, 4, 64, 128), 0.001, f"{h}/e_conv7_2"))
            sp.append((f"{h}/e_conv8_2/e_conv8_2", "conv2d_transpose", (4, 4, 32, 64), 0.001, f"{h}/e_conv8_2"))
            sp.append((f"{h}/e_conv9_2/e_conv9_2", "conv2d_transpose", (4, 4, 16, 32), 0.001, f"{h}/e_conv9_2"))
            sp.append((f"{h}/e_conv10_2/e_conv10_2", "conv2d_transpose", (4, 4, 3, 16), 0.001, None))
    return sp


def init_texture_weights(seed: int = 0, alpha_range=(0.0, 0.0), gain: float = 1.0, bias_jitter: float = 0.0,
                         decoder_std: float = 0.02) -> Dict[str, np.ndarray]:
    """Seeded weights: xavier-uniform for the render net; N(0, 0.02) for the texture decoder (layer_util defaults)."""
    rng = np.random.default_rng(seed)
    W: Dict[str, np.ndarray] = {}
    for name, kind, shape, bias0, alpha_scope in texture_layer_specs():
        if name.startswith("texture_encoder"):
            W[name + "/weights"] = (rng.standard_normal(shape) * decoder_std).astype(np.float32)
        else:
            fi, fo = _fans(kind, shape)
            W[name + "/weights"] = xavier_uniform(rng, shape, fi, fo, gain)
        nb = shape[-2] if kind in ("conv2d_transpose", "conv3d_transpose") else shape[-1]
        bias = np.full((nb,), bias0, np.float32)
        if bias_jitter > 0.0:
            bias = bias + (rng.standard_normal(nb) * bias_jitter).astype(np.float32)
        W[name + "/biases"] = bias
        if alpha_scope is not None:
            lo, hi = alpha_range
            W[alpha_scope + "/alpha"] = (rng.uniform(lo, hi, size=nb).astype(np.float32)
                                         if hi > lo else np.full((nb,), lo, np.float32))
    return W


def decoder_texture(z_in, W, dtype=_F32):
    """RenderNet_Texture_Face_Normal.py:34-46: FC 199->32^3*4, T-conv 4^3 s1 4->4, T-conv 4^3 s2 4->8, conv 4^3 8->4.
    z_in is taken as float32 (what the model is fed); dtype is the arithmetic type, as in conv3d."""
    te = "texture_encoder"
    g = lambda n: W[n]
    z = _t(np.asarray(z_in, np.float32))
    zP = prelu(fully_connected(z, g(f"{te}/e_tex_fc1/fully_connected/weights"), g(f"{te}/e_tex_fc1/fully_connected/biases"),
                               dtype), g(f"{te}/e_tex_fc1/alpha"), dtype)
    x = zP.reshape(z.shape[0], 32, 32, 32, 4)
    c0 = prelu(conv3d_transpose(x, g(f"{te}/e_tex_conv0/conv3d_transpose/weights"),
                                g(f"{te}/e_tex_conv0/conv3d_transpose/biases"), (1, 1, 1), dtype),
               g(f"{te}/e_tex_conv0/alpha"), dtype)
    c1 = prelu(conv3d_transpose(c0, g(f"{te}/e_tex_conv1/conv3d_transpose/weights"),
                                g(f"{te}/e_tex_conv1/conv3d_transpose/biases"), (2, 2, 2), dtype),
               g(f"{te}/e_tex_conv1/alpha"), dtype)
    c2 = prelu(conv3d(c1, g(f"{te}/e_tex_conv2/conv3d/weights"), g(f"{te}/e_tex_conv2/conv3d/biases"), (1, 1, 1), dtype),
               g(f"{te}/e_tex_conv2/alpha"), dtype)
    return c2


def rendernet_texture(models_in, W, return_stages: bool = False):
    """RenderNet_Texture_Face_Normal.py:48-147 at inference.  models_in [B,H,W,128,5] -> (image, normal)."""
    g = lambda n: W[n]
    e = "encoder"
    c3 = lambda x, s, st=(1, 1, 1): conv3d(x, g(s + "/weights"), g(s + "/biases"), st)
    c2 = lambda x, s: conv2d(x, g(s + "/weights"), g(s + "/biases"))
    ct = lambda x, s, k: conv2d_transpose(x, g(s + "/weights"), g(s + "/biases"), (k, k))
    st = {}
    x = _t(models_in).float()
    enc1 = prelu(c3(x, f"{e}/e_conv1/e_conv1", (2, 2, 2)), g(f"{e}/e_conv1/alpha"))
    enc2 = prelu(c3(enc1, f"{e}/e_conv2/e_conv2", (1, 1, 2)), g(f"{e}/e_conv2/alpha"))
    enc3 = prelu(c3(enc2, f"{e}/e_conv3/e_conv3"), g(f"{e}/e_conv3/alpha"))
    h = enc3
    for k in range(1, 11):
        t = prelu(c3(h, f"{e}/res1_{k}/con1_3X3"), g(f"{e}/res1_{k}/alpha"))
        h = c3(t, f"{e}/res1_{k}/conv2_3x3") + h
    enc3_skip = c3(h, f"{e}/res1_skip/con1_3X3") + enc3
    enc4 = projection_unit(enc3_skip, g(f"{e}/projection_unit/Conv/weights"), g(f"{e}/projection_unit/Conv/biases"),
                           g(f"{e}/projection_unit/alpha"))
    h = enc4
    for k in range(1, 11):
        t = prelu(c2(h, f"{e}/res2_{k}/con1_3X3"), g(f"{e}/res2_{k}/alpha"))
        h = c2(t, f"{e}/res2_{k}/conv2_3x3") + h
    enc4_skip = c2(h, f"{e}/res2_skip/con1_3X3") + enc4
    enc5 = prelu(c2(enc4_skip, f"{e}/e_conv5/e_conv5"), g(f"{e}/e_conv5/alpha"))
    h = enc5
    for k in range(1, 6):
        t = prelu(c2(h, f"{e}/res3_{k}/con1_3X3"), g(f"{e}/res3_{k}/alpha"))
        h = c2(t, f"{e}/res3_{k}/conv2_3x3") + h
    enc5_skip = c2(h, f"{e}/res3_skip/con1_3X3") + enc5
    st.update(enc3=enc3, enc3_skip=enc3_skip, enc4=enc4, enc4_skip=enc4_skip, enc5_skip=enc5_skip)
    outs = []
    for head, sfx, names in (("Image", "1", ("e_conv7_1/e_conv7_2", "e_conv8_1/conv2d_transpose", "e_conv9_1/conv2d_transpose",
                                              "e_conv10_1/conv2d_transpose")),
                             ("Normal", "2", ("e_conv7_2/e_conv7_2", "e_conv8_2/e_conv8_2", "e_conv9_2/e_conv9_2",
                                              "e_conv10_2/e_conv10_2"))):
        hh = f"{e}/{head}"
        a6 = prelu(c2(enc5_skip, f"{hh}/e_conv6_{sfx}/e_conv6_{sfx}"), g(f"{hh}/e_conv6_{sfx}/alpha"))
        a7 = prelu(ct(a6, f"{hh}/{names[0]}", 2), g(f"{hh}/e_conv7_{sfx}/alpha"))
        a8 = prelu(ct(a7, f"{hh}/{names[1]}", 2), g(f"{hh}/e_conv8_{sfx}/alpha"))
        a9 = prelu(ct(a8, f"{hh}/{names[2]}", 2), g(f"{hh}/e_conv9_{sfx}/alpha"))
        logits = ct(a9, f"{hh}/{names[3]}", 1)
        st[f"logits_{head}"] = logits
        outs.append(torch.sigmoid(logits))
    if return_stages:
        return outs[0], outs[1], st
    return outs[0], outs[1]


def render_forward_texture(voxel, texture_in, view_params, W):
    """Graph of RenderNet_Texture_Face_Normal.py:155-179 at inference."""
    rot = transform_voxel_to_match_image(rotation_resampling(voxel, view_params))
    tex = decoder_texture(texture_in, W).numpy()
    tex_rot = transform_voxel_to_match_image(rotation_resampling(tex, view_params))
    x = np.ascontiguousarray(np.concatenate([rot, tex_rot], axis=4))
    return rendernet_texture(x, W)
