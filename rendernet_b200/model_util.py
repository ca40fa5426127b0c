"""Mirror of the hot-path part of the reference's tools/model_util.py: the voxel->image axis transform
(:41-49), the npz weight-directory loader (:10-39) and the random patch crops of training (:77-161)."""
from __future__ import annotations

import glob
import os

import numpy as np
import torch

from .resampling_voxel_grid import ConcatResampledGrid, CroppedGrid, ResampledGrid


def get_weight(weight_name, weight_dict):
    """:13-24."""
    if weight_dict is None:
        return None
    return weight_dict.get(weight_name)


def load_weights(weight_dir):
    """:26-39: every `<layer>.txt.npz` in the directory -> {layer_name: arr_0}."""
    out = {}
    for path in glob.glob(os.path.join(weight_dir, "*.txt.npz")):
        with np.load(path) as data:
            out[os.path.basename(path).split('.')[0]] = data['arr_0']
    return out


def tf_transform_voxel_to_match_image(tensor_voxel):
    """:41-49: N[b,p,q,r,c] = T[b,q,P-1-p,r,c].  Fused into the resampling kernel when applied to its
    (deferred) output -- which stays deferred, so that e_conv1 can absorb it too; a plain strided copy otherwise
    (pure data movement)."""
    if isinstance(tensor_voxel, ResampledGrid):
        return tensor_voxel.transformed()
    t = tensor_voxel if isinstance(tensor_voxel, torch.Tensor) else torch.as_tensor(np.asarray(tensor_voxel))
    return torch.flip(t.permute(0, 2, 1, 3, 4), dims=(1,)).contiguous()


def random_crop_origin(voxel_dim: int, patch_size: int, rng=None):
    """tf.random_uniform([2], minval=0, maxval=voxel_dim - patch_size + 1, dtype=tf.int32) (:93): ONE (y0, x0) for the whole
    batch, each uniform on [0, voxel_dim - patch_size].  rng: a numpy Generator (None: a fresh unseeded one)."""
    rng = np.random.default_rng() if rng is None else rng
    y0, x0 = rng.integers(0, voxel_dim - patch_size + 1, size=2)
    return int(y0), int(x0)


def _crop_voxels(v, y0: int, x0: int, patch_size: int):
    """v[:, y0:y0+P, x0:x0+P, :, :]: a CroppedGrid of a deferred resampled grid (the fused e_conv1 runs on the window), a slice
    otherwise."""
    if isinstance(v, (ResampledGrid, ConcatResampledGrid)):
        return CroppedGrid(v, y0, x0, patch_size, patch_size)
    return v[:, y0:y0 + patch_size, x0:x0 + patch_size, :, :]


def _crop_setup(voxels, images, patch_size, origin, rng):
    voxel_dim, image_dim = int(voxels.shape[1]), int(images.shape[1])
    factor = int(image_dim / voxel_dim)                   # tf.to_int32(image_dim / voxel_dim)
    P = int(patch_size)
    if P == voxel_dim:
        return None
    if not 0 < P < voxel_dim:
        raise ValueError(f"patch_size {P} outside (0, {voxel_dim}]")
    y0, x0 = random_crop_origin(voxel_dim, P, rng) if origin is None else (int(origin[0]), int(origin[1]))
    if not (0 <= y0 <= voxel_dim - P and 0 <= x0 <= voxel_dim - P):
        raise ValueError(f"crop origin ({y0}, {x0}) with patch {P} leaves the {voxel_dim}-grid")
    return y0, x0, P, factor


def _crop_image(img, y0, x0, P, factor):
    iy, ix, e = y0 * factor, x0 * factor, factor * P      # the image patch starts at factor x the voxel origin, edge factor*P
    return img[:, iy:iy + e, ix:ix + e, :]


def tf_random_crop_voxel_image(voxels, images, patch_size, origin=None, rng=None):
    """:77-100.  voxels [B,N,N,N,C] (the axis-transformed grid; deferred -> CroppedGrid), images [B,I,I,C] -> (voxel patch
    [B,P,P,N,C], image patch [B,fP,fP,C]) with f = I // N and one origin (y0, x0) for the whole batch; the image patch starts at
    f x the origin.  patch_size == N returns both unchanged.  origin: a fixed (y0, x0); otherwise drawn from rng."""
    c = _crop_setup(voxels, images, patch_size, origin, rng)
    if c is None:
        return voxels, images
    y0, x0, P, f = c
    return _crop_voxels(voxels, y0, x0, P), _crop_image(images, y0, x0, P, f)


def tf_random_crop_voxel_texture_image(voxels, texture, images, patch_size, origin=None, rng=None):
    """:102-131: tf_random_crop_voxel_image with a texture grid of the voxels' spatial shape cropped at the same origin ->
    (voxel patch, texture patch, image patch)."""
    c = _crop_setup(voxels, images, patch_size, origin, rng)
    if c is None:
        return voxels, texture, images
    y0, x0, P, f = c
    return _crop_voxels(voxels, y0, x0, P), _crop_voxels(texture, y0, x0, P), _crop_image(images, y0, x0, P, f)


def tf_random_crop_voxel_texture_image_normal(voxels, texture, images, normals, patch_size, origin=None, rng=None):
    """:133-161: tf_random_crop_voxel_texture_image plus the normal map, cropped like the image -> (voxel patch, texture patch,
    image patch, normal patch).  Always four values: upstream's patch_size == voxel_dim branch returns three (no normals), but
    its only caller (RenderNet_Texture_Face_Normal.py:175, epoch schedule 32 / 64 on a 128 grid) never takes it (SURVEY
    finding 7); here that branch returns the four inputs unchanged."""
    c = _crop_setup(voxels, images, patch_size, origin, rng)
    if c is None:
        return voxels, texture, images, normals
    y0, x0, P, f = c
    return (_crop_voxels(voxels, y0, x0, P), _crop_voxels(texture, y0, x0, P), _crop_image(images, y0, x0, P, f),
            _crop_image(normals, y0, x0, P, f))
