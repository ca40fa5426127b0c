"""CPU oracle of the face-reconstruction shape decoder (Reconstruct_RenderNet_Face.py:31-75, decoder_3d_pretrained).  TEST
INFRASTRUCTURE ONLY, like oracle/rendernet_oracle.py, whose float32 / float64 layer ops it reuses.

    FC 200 -> 4^3 x 256, conv3d_transpose k4 s2 + ELU x 4 (256 -> 128 -> 64 -> 32 -> 16), conv3d_transpose k4 s1 + sigmoid (16 -> 1)

Weights are keyed as in the reference's npz directories (g_zP_g_gc1_weights, g_conv1_g_conv1_biases, ..., g_conv5_weights).
Pinned to the reference's own decoder_3d_pretrained, run over the TF-1 shim, by tests/golden/shape_decoder.npz
(tests/golden/make_shape_decoder_golden.py).
"""
from __future__ import annotations

from typing import Dict

import numpy as np
import torch

from . import rendernet_oracle as orc

# (npz prefix, filter shape [4,4,4,Cout,Cin], stride)
CONV_LAYERS = (("g_conv1_g_conv1", (4, 4, 4, 128, 256), 2), ("g_conv2_g_conv2", (4, 4, 4, 64, 128), 2),
               ("g_conv3_g_conv3", (4, 4, 4, 32, 64), 2), ("g_conv4_g_conv4", (4, 4, 4, 16, 32), 2),
               ("g_conv5", (4, 4, 4, 1, 16), 1))


def init_shape_decoder_weights(seed: int = 0, z_dim: int = 200, gain: float = 1.0, bias_std: float = 0.05) -> Dict[str, np.ndarray]:
    """Seeded decoder weights in the npz key convention.  Each filter is N(0, gain^2 / fan), fan = the taps x channels one output
    sums (8 Cin for the stride-2 layers, 64 Cin for g_conv5), so activations stay O(1) through the ELUs and the sigmoid's input
    spans a few units; biases N(0, bias_std^2)."""
    rng = np.random.default_rng(seed)
    W = {"g_zP_g_gc1_weights": (rng.standard_normal((z_dim, 4 * 4 * 4 * 256)) * gain / np.sqrt(z_dim)).astype(np.float32),
         "g_zP_g_gc1_biases": (rng.standard_normal(4 * 4 * 4 * 256) * bias_std).astype(np.float32)}
    for name, shape, s in CONV_LAYERS:
        fan = (8 if s == 2 else 64) * shape[4]
        W[name + "_weights"] = (rng.standard_normal(shape) * gain / np.sqrt(fan)).astype(np.float32)
        W[name + "_biases"] = (rng.standard_normal(shape[3]) * bias_std).astype(np.float32)
    return W


def elu(x, dtype=orc._F32):
    """tf.nn.elu as TF-1 computes it: x < 0 ? exp(x) - 1 : x (exp, then subtract)."""
    x = orc._t(x).to(dtype)
    return torch.where(x < 0, torch.exp(x) - 1, x)


def decoder_3d(z, W, dtype=orc._F32, return_stages: bool = False):
    """latent [B,200] -> voxels [B,64,64,64,1] in arithmetic type `dtype` (torch.float64: the high-precision reference; z may be a
    tensor that requires grad).  return_stages: also {layer npz prefix: its output}."""
    z = z.to(dtype) if isinstance(z, torch.Tensor) else orc._t(np.asarray(z, np.float32)).to(dtype)
    h = orc.fully_connected(z, W["g_zP_g_gc1_weights"], W["g_zP_g_gc1_biases"], dtype)
    h = h.reshape(z.shape[0], 4, 4, 4, h.shape[1] // 64)
    st = {"g_zP_g_gc1": h}
    for name, _, s in CONV_LAYERS:
        h = orc.conv3d_transpose(h, W[name + "_weights"], W[name + "_biases"], (s, s, s), dtype)
        h = torch.sigmoid(h) if name == "g_conv5" else elu(h, dtype)
        st[name] = h
    return (h, st) if return_stages else h
