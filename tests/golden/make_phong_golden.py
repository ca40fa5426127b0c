#!/usr/bin/env python
"""Freeze tests/golden/phong_tf.npz: the reference's own TensorFlow Phong composite (tools/Phong_shading.py:24-130,
tf_phong_composite and tf_generate_light_pos) executed over the NumPy shim of TF-1 (oracle/tf1_shim.py), with the few
reductions it needs added here.  Holds oracle/phong_tf.py (the differentiable restatement the reconstruction-gradient tests
use) to the reference's forward arithmetic.  Usage: python tests/golden/make_phong_golden.py /path/to/RenderNet
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import tf1_shim  # noqa: E402


def _install(ref):
    tf = tf1_shim.install()
    T = tf1_shim._T
    ones_like = tf.ones_like

    def norm(x, axis=None, keep_dims=False, keepdims=None):
        return T(np.sqrt(np.sum(np.square(np.asarray(x)), axis=axis, keepdims=bool(keep_dims or keepdims))))

    def reduce_sum(x, axis=None, keep_dims=False, keepdims=None):
        return T(np.sum(np.asarray(x), axis=axis, keepdims=bool(keep_dims or keepdims)))

    tf.norm = norm
    tf.reduce_sum = reduce_sum
    tf.reduce_prod = lambda x, axis=None: T(np.prod(np.asarray(x), axis=axis))
    tf.multiply = lambda a, b: T(np.multiply(np.asarray(a), np.asarray(b)))
    tf.sigmoid = lambda x: T((1.0 / (1.0 + np.exp(-np.asarray(x, np.float64)))).astype(np.asarray(x).dtype))
    tf.ones_like = lambda x, dtype=None: ones_like(x) if dtype is None else T(np.ones_like(np.asarray(x), tf1_shim._dt(dtype)))
    sys.path.insert(0, ref)
    return tf


def inputs():
    """Normal maps that hit the kinks exactly, plus random and dark / bright background pixels."""
    rng = np.random.default_rng(17)
    nm = rng.random((2, 16, 16, 3)).astype(np.float32)
    nm[:, :3] *= 0.05                                   # dark rows: black-background mask ~ 0
    nm[:, 3:5] = 0.97 + 0.03 * nm[:, 3:5]               # bright rows: white-background mask ~ 0
    nm[:, 5, :4] = [0.5, 0.5, 0.75]                     # n - 0.5 parallel to light (0,0,1): u.L = 1 exactly
    nm[:, 5, 4:8] = [0.75, 0.5, 0.5]                    # perpendicular: u.L = 0 exactly (maximum(., 0) kink)
    nm[:, 5, 8:12] = [0.5, 0.25, 0.5]                   # opposite side: u.L < 0
    light = np.array([[0.0, 0.0, 2.0], [0.3, -0.4, 0.8]], np.float32)    # item 0: exact (0,0,1) after normalisation
    col = np.array([[1.0, 1.0, 1.0], [0.9, 1.0, 0.7]], np.float32)
    return nm, light, col


def main(ref):
    tf = _install(ref)
    from tools import Phong_shading
    nm, light, col = inputs()
    out = dict(normal_map=nm, light=light, light_col=col, ambient=np.float32(0.1), k_diffuse=np.float32(0.9))
    for name, black, mask in (("white_mask", False, True), ("black_mask", True, True), ("no_mask", False, False)):
        out[name] = np.asarray(Phong_shading.tf_phong_composite(tf.constant(nm), tf.constant(light.copy()), tf.constant(col), 0.1,
                                                                0.9, with_black_background=black, with_mask=mask), np.float32)
    out["exact_light_k1"] = np.asarray(Phong_shading.tf_phong_composite(tf.constant(nm), tf.constant(light.copy()), tf.constant(
        np.ones((2, 3), np.float32)), 0.0, 1.0, with_mask=False), np.float32)      # clip boundaries: diffuse = 1 exactly
    az = np.array([[0.3], [2.1]], np.float32)
    out["light_azimuth"] = az
    out["light_elevation"] = np.float32(0.6)
    out["light_pos"] = np.asarray(Phong_shading.tf_generate_light_pos(tf.constant(az), 0.6, 2), np.float32)
    np.savez_compressed(os.path.join(HERE, "phong_tf.npz"), **out)
    print("wrote", os.path.join(HERE, "phong_tf.npz"))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.environ.get("RENDERNET_REFERENCE", ""))
