"""Drop-in mirror of the `tf_*` half of the reference's tools/resampling_voxel_grid.py (:370-632): rotate a
voxel grid into the camera frame by inverse-mapped trilinear resampling.  The ~60 TF ops of
tf_resampling + tf_interpolate + tf_voxel_meshgrid collapse into ONE gather kernel (rn_resample_f32) that
also applies tools/model_util.py:41-49's axis transform when that call follows.

Pose -> matrix arithmetic ([B,4,4] fp32, a few hundred flops) stays on the host in NumPy float32, in the
reference's own operation order (:529-602), so the kernel and the oracle sample at identical coordinates.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from . import ops
from .tfcompat import get_store


def _np32(x) -> np.ndarray:
    if isinstance(x, torch.Tensor):
        x = x.detach().cpu().numpy()
    return np.asarray(x, dtype=np.float32)


def tf_rotation_around_grid_centroid(view_params):
    """:515-562.  view_params [B,3] = (azimuth rad, elevation-param rad, scale) -> (R [B,4,4], S [B,4,4]).
    The reference's `== 2` test (:551) is always False in TF1, so the 3-parameter branch always runs."""
    vp = _np32(view_params)
    B = vp.shape[0]
    az = vp[:, 0] - np.float32(math.pi * 0.5)
    el = vp[:, 1]
    ca, sa, ce, se = np.cos(az), np.sin(az), np.cos(el), np.sin(el)
    rot_y = np.zeros((B, 4, 4), np.float32)
    rot_y[:, 0, 0], rot_y[:, 0, 2] = ca, -sa
    rot_y[:, 1, 1] = 1
    rot_y[:, 2, 0], rot_y[:, 2, 2] = sa, ca
    rot_y[:, 3, 3] = 1
    rot_z = np.zeros((B, 4, 4), np.float32)
    rot_z[:, 0, 0], rot_z[:, 0, 1] = ce, se
    rot_z[:, 1, 0], rot_z[:, 1, 1] = -se, ce
    rot_z[:, 2, 2] = 1
    rot_z[:, 3, 3] = 1
    R = np.matmul(rot_z, rot_y)
    if vp.shape[1] == 2:
        return R
    S = np.zeros((B, 4, 4), np.float32)
    S[:, 0, 0] = S[:, 1, 1] = S[:, 2, 2] = vp[:, 2]
    S[:, 3, 3] = 1
    return R, S


def inverse_sampling_matrix(transformation_matrix, Scale_matrix=None, size=64, new_size=128) -> np.ndarray:
    """:579-602: M = T(+new/2).S.R.T(-size/2);  returns inverse(M)[:, :3, :] as fp32 [B,3,4]."""
    R = _np32(transformation_matrix)
    B = R.shape[0]
    T = np.array([[1, 0, 0, -size * 0.5], [0, 1, 0, -size * 0.5], [0, 0, 1, -size * 0.5], [0, 0, 0, 1]], np.float32)
    Tn = np.array([[1, 0, 0, new_size * 0.5], [0, 1, 0, new_size * 0.5], [0, 0, 1, new_size * 0.5], [0, 0, 0, 1]],
                  np.float32)
    T = np.tile(T[None], (B, 1, 1))
    Tn = np.tile(Tn[None], (B, 1, 1))
    if Scale_matrix is None:
        M = np.matmul(np.matmul(Tn, R), T)
    else:
        M = np.matmul(np.matmul(np.matmul(Tn, _np32(Scale_matrix)), R), T)
    return np.ascontiguousarray(np.linalg.inv(M).astype(np.float32)[:, 0:3, :])


class ResampledGrid:
    """Deferred result of tf_resampling, so that a following tf_transform_voxel_to_match_image is fused into the
    gather kernel and -- when the consumer is the Shader net's e_conv1 -- the whole resample+transform+conv becomes
    one kernel that never writes the new_size^3 grid (layer_util.conv3d, SURVEY §8 f-1)."""

    def __init__(self, voxel: torch.Tensor, minv: torch.Tensor, new_size: int, transform: bool = False):
        self.voxel, self.minv, self.new_size, self.transform = voxel, minv, new_size, transform
        B, _, _, _, C = voxel.shape
        self.shape = (B, new_size, new_size, new_size, C)
        self.dtype = torch.float32
        self._value = None

    def transformed(self) -> "ResampledGrid":
        """tools/model_util.py:41-49 applied lazily: N[b,p,q,r,c] = T[b,q,P-1-p,r,c] (cubic grid: same shape)."""
        if self.transform:
            raise ValueError("axis transform already applied")
        return ResampledGrid(self.voxel, self.minv, self.new_size, True)

    def realize(self, transform=None) -> torch.Tensor:
        t = self.transform if transform is None else bool(transform)
        if t != self.transform:
            return ops.resample(self.voxel, self.minv, self.new_size, t)
        if self._value is None:
            self._value = ops.resample(self.voxel, self.minv, self.new_size, t)
        return self._value

    def get_shape(self):
        return list(self.shape)


class ConcatResampledGrid:
    """tf.concat([rotated geometry (C = 1), rotated texture volume (C = 4)], axis=4) of two deferred, axis-transformed
    resamplings that share pose and size (RenderNet_Texture_Face_Normal.py:155-179), still deferred: when the consumer is the
    Texture net's e_conv1 the whole chain runs as ONE kernel (rn_resample5_conv1_fused) and the 128^3 x 5 grid is never written."""

    def __init__(self, geom: ResampledGrid, tex: ResampledGrid):
        if (geom.new_size != tex.new_size or geom.transform != tex.transform or geom.minv.data_ptr() != tex.minv.data_ptr()
                and not torch.equal(geom.minv, tex.minv)):
            raise ValueError("ConcatResampledGrid: the two grids must share pose, size and axis transform")
        if geom.voxel.shape[-1] != 1 or tex.voxel.shape[-1] != 4:
            raise ValueError("ConcatResampledGrid: expects a 1-channel geometry grid and a 4-channel texture volume")
        self.geom, self.tex = geom, tex
        self.minv, self.new_size, self.transform = geom.minv, geom.new_size, geom.transform
        self.shape = tuple(geom.shape[:-1]) + (5,)
        self.dtype = torch.float32
        self._value = None

    def realize(self) -> torch.Tensor:
        if self._value is None:
            self._value = ops.concat_channels(self.geom.realize(), self.tex.realize())
        return self._value

    def get_shape(self):
        return list(self.shape)


class CroppedGrid:
    """A deferred patch of an axis-transformed ResampledGrid (C = 1 or 4) or ConcatResampledGrid: rows [y0, y0+ph), columns
    [x0, x0+pw), every depth -- what tools/model_util.py:77-161 slice out of the rotated grid for training on random patches.
    When the consumer is e_conv1 the fused kernels run on the window alone (rn_resample*_conv1_fused_window; SAME padding at
    the patch's borders, as after a slice), so neither the grid nor the patch is written.  ph and pw are multiples of 16."""

    def __init__(self, grid, y0: int, x0: int, ph: int, pw: int):
        if not isinstance(grid, (ResampledGrid, ConcatResampledGrid)) or not grid.transform or grid._value is not None:
            raise ValueError("CroppedGrid: crops a deferred, axis-transformed resampled grid")
        if isinstance(grid, ResampledGrid) and grid.shape[-1] not in (1, 4):
            raise ValueError("CroppedGrid: a resampled grid of 1 or 4 channels")
        self.window = ops.check_window((y0, x0, ph, pw), grid.new_size)
        self.grid = grid
        self.minv, self.new_size, self.transform = grid.minv, grid.new_size, True
        B, N, C = grid.shape[0], grid.new_size, grid.shape[-1]
        self.shape = (B, int(ph), int(pw), N, C)
        self.dtype = torch.float32
        self._value = None

    def realize(self) -> torch.Tensor:
        if self._value is None:
            g, w = self.grid, self.window
            if isinstance(g, ConcatResampledGrid):
                self._value = ops.concat_channels(ops.resample(g.geom.voxel, g.minv, g.new_size, True, window=w),
                                                  ops.resample(g.tex.voxel, g.minv, g.new_size, True, window=w))
            else:
                self._value = ops.resample(g.voxel, g.minv, g.new_size, True, window=w)
        return self._value

    def get_shape(self):
        return list(self.shape)


def concat_resampled(a, b):
    """tf.concat([a, b], 4): stays deferred for (geometry, texture) pairs of resampled grids, and for pairs of patches of them
    cropped at one window, plain concat otherwise."""
    if isinstance(a, ResampledGrid) and isinstance(b, ResampledGrid) and a._value is None and b._value is None:
        try:
            return ConcatResampledGrid(a, b)
        except ValueError:
            pass
    if (isinstance(a, CroppedGrid) and isinstance(b, CroppedGrid) and a.window == b.window and a._value is None
            and b._value is None and isinstance(a.grid, ResampledGrid) and isinstance(b.grid, ResampledGrid)):
        try:
            return CroppedGrid(ConcatResampledGrid(a.grid, b.grid), *a.window)
        except ValueError:
            pass
    return ops.concat_channels(a.realize() if hasattr(a, "realize") else a, b.realize() if hasattr(b, "realize") else b)


def _to_cuda_f32(x) -> torch.Tensor:
    if hasattr(x, "realize"):          # deferred conv output (texture decoder)
        x = x.realize()
    if not isinstance(x, torch.Tensor):
        x = torch.from_numpy(np.ascontiguousarray(np.asarray(x, dtype=np.float32)))
    y = x.to(device="cuda", dtype=torch.float32).contiguous()
    if y.data_ptr() != x.data_ptr():
        tape = get_store().tape
        if tape is not None:                        # backward.py follows tensors by storage address: map the copy to its source
            tape.append(dict(op="copy", x=x, y=y))
    return y


def tf_resampling(voxel_array, transformation_matrix, params=None, Scale_matrix=None, size=64, new_size=128):
    """:564-614.  `params` is vestigial in the reference (never read) and therefore optional here; the
    shipped tf_rotation_resampling omits it and would raise TypeError (SURVEY finding 4)."""
    minv = inverse_sampling_matrix(transformation_matrix, Scale_matrix, size, new_size)
    return ResampledGrid(_to_cuda_f32(voxel_array), torch.from_numpy(minv).cuda(), new_size)


def tf_interpolate(voxel, x, y, z, out_size):
    """:381-486 as a standalone call: trilinear interpolation of `voxel` [B,S,S,S,C] at the flat coordinate lists x, y, z
    (each B*n points, batch-major) -> [B*n, C] float32; `out_size` = [B, h, w, d, C] is only used, like upstream, for the
    point count per item.  Clamp-then-weight rule reproduced bit for bit (rn_interpolate_f32)."""
    vox = _to_cuda_f32(voxel)
    n = int(out_size[1]) * int(out_size[2]) * int(out_size[3])
    xs, ys, zs = (torch.as_tensor(np.asarray(t, np.float32) if not isinstance(t, torch.Tensor) else t).reshape(-1) for t in (x, y, z))
    if xs.numel() != vox.shape[0] * n:
        raise ValueError(f"tf_interpolate: {xs.numel()} points for out_size {list(out_size)} and batch {vox.shape[0]}")
    return ops.interpolate(vox, xs, ys, zs)


def tf_rotation_resampling(voxel_array, view_params, size=64, new_size=128):
    """:616-632."""
    vp = _np32(view_params)
    if vp.shape[1] == 2:
        M = tf_rotation_around_grid_centroid(vp)
        return tf_resampling(voxel_array, M, size=size, new_size=new_size)
    M, S = tf_rotation_around_grid_centroid(vp)
    return tf_resampling(voxel_array, M, Scale_matrix=S, size=size, new_size=new_size)


tf_rotation_translation_resampling = tf_rotation_resampling   # :634-650 is a verbatim duplicate upstream


def tf_voxel_meshgrid(height, width, depth, homogeneous=False):
    """:488-513: rows (x=k, y=j, z=i[, 1]) for flat index n = i*H*W + j*W + k (host NumPy; the kernel
    generates these coordinates on the fly and never materialises the grid)."""
    z_t, y_t, x_t = np.meshgrid(np.arange(depth, dtype=np.float32), np.arange(height, dtype=np.float32),
                                np.arange(width, dtype=np.float32), indexing='ij')
    rows = [x_t.reshape(1, -1), y_t.reshape(1, -1), z_t.reshape(1, -1)]
    if homogeneous:
        rows.append(np.ones_like(rows[0]))
    return np.concatenate(rows, axis=0)
