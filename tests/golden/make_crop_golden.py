#!/usr/bin/env python
"""Freeze tests/golden/crop.npz: the reference's own random patch crops (tools/model_util.py:77-161,
tf_random_crop_voxel_image and tf_random_crop_voxel_texture_image_normal), imported unmodified from a reference checkout and
executed over the NumPy shim of TF-1 (oracle/tf1_shim.py).  What they need beyond the shim is added here: tf.identity's
`name` argument, and tf.random_uniform as a seeded draw whose values the fixture records, so that the mirror
(rendernet_b200/model_util.py) can be called with the same origin and held to the reference's slices -- the voxel patch and
the image / normal patch at image_dim // voxel_dim times the origin.  Usage: python tests/golden/make_crop_golden.py /path/to/RenderNet
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import tf1_shim  # noqa: E402

SEED = 1618
# (voxel grid [B, V, V, D, C], image edge, patch size): image factors 4 (the networks' 128 -> 512) and 2
CASES = [((2, 8, 8, 3, 1), 32, 4), ((2, 12, 12, 2, 1), 24, 4), ((1, 16, 16, 2, 1), 64, 8)]


def main(ref):
    tf = tf1_shim.install()
    draws = []
    rng = np.random.default_rng(SEED)

    def random_uniform(shape, minval=0, maxval=None, dtype=None, seed=None, name=None):
        """tf.random_uniform for an int32 draw on [minval, maxval): seeded, recorded in call order."""
        v = rng.integers(int(minval), int(maxval), size=tuple(int(s) for s in shape)).astype(np.int32)
        draws.append(v)
        return tf1_shim._T(v)

    tf.random_uniform = random_uniform
    tf.identity = lambda x, name=None: tf1_shim.identity(x)
    sys.path.insert(0, ref)
    from tools import model_util
    out = dict(seed=np.int64(SEED), n_cases=np.int64(len(CASES)))
    for i, (vshape, idim, P) in enumerate(CASES):
        vox = rng.standard_normal(vshape).astype(np.float32)
        tex = rng.standard_normal(vshape[:-1] + (4,)).astype(np.float32)
        img = rng.standard_normal((vshape[0], idim, idim, 3)).astype(np.float32)
        nrm = rng.standard_normal((vshape[0], idim, idim, 3)).astype(np.float32)
        n0 = len(draws)
        v1, i1 = model_util.tf_random_crop_voxel_image(tf.constant(vox), tf.constant(img), P)
        v2, t2, i2, n2 = model_util.tf_random_crop_voxel_texture_image_normal(tf.constant(vox), tf.constant(tex), tf.constant(img),
                                                                             tf.constant(nrm), P)
        assert len(draws) == n0 + 2
        out.update({f"c{i}_vox": vox, f"c{i}_tex": tex, f"c{i}_img": img, f"c{i}_nrm": nrm, f"c{i}_patch": np.int64(P),
                    f"c{i}_origin_a": draws[n0], f"c{i}_origin_b": draws[n0 + 1],
                    f"c{i}_a_vox": np.asarray(v1), f"c{i}_a_img": np.asarray(i1),
                    f"c{i}_b_vox": np.asarray(v2), f"c{i}_b_tex": np.asarray(t2), f"c{i}_b_img": np.asarray(i2),
                    f"c{i}_b_nrm": np.asarray(n2)})
    np.savez_compressed(os.path.join(HERE, "crop.npz"), **out)
    print("wrote", os.path.join(HERE, "crop.npz"), "origins", [d.tolist() for d in draws])


if __name__ == "__main__":
    main(sys.argv[1])
