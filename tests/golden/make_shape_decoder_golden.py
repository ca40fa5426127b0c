#!/usr/bin/env python
"""Freeze tests/golden/shape_decoder.npz: the reference's own face-reconstruction shape decoder (Reconstruct_RenderNet_Face.py:31-75,
decoder_3d_pretrained), lifted out of its module with `ast` (the module runs its optimisation at import time) and executed over the
NumPy shim of TF-1 (oracle/tf1_shim.py) with tools/layer_util.py imported unmodified, on seeded weights
(oracle/shape_decoder.init_shape_decoder_weights).  The fixture stores the seed, the latents and a strided sample of the output
(every third voxel along each axis, so all eight output phases of the stride-2 layers are covered) plus full-grid sums; the
weights are regenerated from the seed.  Usage: python tests/golden/make_shape_decoder_golden.py /path/to/RenderNet
"""
import io
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from oracle import tf1_shim  # noqa: E402
from oracle.shape_decoder import init_shape_decoder_weights  # noqa: E402

SEED = 2718


def _elu(x, name=None):
    """tf.nn.elu (TF-1: exp, then subtract 1) -- the one op the decoder needs beyond the shim."""
    x = np.asarray(x, np.float32)
    return tf1_shim._T(np.where(x < 0, np.exp(x) - np.float32(1), x).astype(np.float32))


def latents():
    z = np.empty((2, 200), np.float32)
    z[0] = 0.5                                               # the reconstruction's first-epoch latent (:463)
    z[1] = np.random.default_rng(SEED + 1).standard_normal(200)
    return z


def main(ref):
    from make_golden import _lift_function
    tf = tf1_shim.install()
    tf.nn.elu = _elu
    sys.path.insert(0, ref)
    from tools import layer_util
    ns = dict(tf=tf, fully_connected=layer_util.fully_connected, conv3d_transpose=layer_util.conv3d_transpose)
    decoder_3d_pretrained = _lift_function(os.path.join(ref, "Reconstruct_RenderNet_Face.py"), "decoder_3d_pretrained", ns)
    W = init_shape_decoder_weights(SEED)
    z = latents()
    stdout, sys.stdout = sys.stdout, io.StringIO()          # layer_util prints per layer
    try:
        tf1_shim.reset(provided=None)
        vox = np.asarray(decoder_3d_pretrained(tf.constant(z), W), np.float32)
        names = sorted(tf1_shim.created_variables().keys())
    finally:
        sys.stdout = stdout
    assert vox.shape == (2, 64, 64, 64, 1), vox.shape
    out = dict(seed=np.int64(SEED), latents=z, voxels_sub=np.ascontiguousarray(vox[:, ::3, ::3, ::3]),
               voxels_sum=vox.sum(axis=(1, 2, 3, 4), dtype=np.float64), voxels_abs_dev=np.abs(vox - 0.5).sum(axis=(1, 2, 3, 4),
                                                                                                           dtype=np.float64),
               var_names=np.array(names))
    np.savez_compressed(os.path.join(HERE, "shape_decoder.npz"), **out)
    print("wrote", os.path.join(HERE, "shape_decoder.npz"), "variables:", names)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.environ.get("RENDERNET_REFERENCE", ""))
