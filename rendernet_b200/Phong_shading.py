"""Mirror of the NumPy Phong path of the reference's tools/Phong_shading.py (:138-228, :247-253) used by the
demo (RenderNet_demo.py:54-58), and of its TensorFlow composite (:88-113) used by face reconstruction.  Each composite
runs in one CUDA kernel (rn_phong_composite, rn_phong_shade); NumPy in -> NumPy out, torch CUDA in -> torch CUDA out."""
from __future__ import annotations

import math

import numpy as np
import torch

from . import ops


def generate_light_pos(elevation=90, azimuth=90):
    """:247-253."""
    elevation = (np.array([[elevation]])) * math.pi / 180.0
    azimuth = (np.array([[azimuth]])) * math.pi / 180.0
    x = np.multiply(-np.sin(elevation), np.cos(azimuth))
    y = np.cos(elevation)
    z = np.multiply(-np.sin(elevation), np.sin(azimuth))
    return np.hstack((x, y, z))


def _run(images_in, light_dir, light_col, ambient_in, k_diffuse, white, with_mask, want_u8=False):
    is_np = not isinstance(images_in, torch.Tensor)
    img = torch.as_tensor(np.asarray(images_in, np.float32)) if is_np else images_in
    img = img.to(device="cuda", dtype=torch.float32).contiguous()
    B = img.shape[0]
    ld = torch.as_tensor(np.asarray(light_dir, np.float32)).reshape(-1, 3)
    lc = torch.as_tensor(np.asarray(light_col, np.float32)).reshape(-1, 3)
    if ld.shape[0] not in (1, B) or lc.shape[0] not in (1, B):
        raise ValueError("light_dir / light_col must have 1 or batch_size rows")
    res = ops.phong_composite(img, ld, lc, ambient_in, k_diffuse, background_white=white, with_mask=with_mask,
                              want_u8=want_u8)
    if want_u8:
        out, u8 = res
        return (out.cpu().numpy(), u8.cpu().numpy()) if is_np else (out, u8)
    return res.cpu().numpy() if is_np else res


def tf_phong_composite(images_in, light_dir, light_col, ambient_in, k_diffuse, with_black_background=False, with_mask=True):
    """:88-113, TensorFlow's composite (the shading face reconstruction multiplies the albedo by) in rn_phong_shade: images_in
    [B,H,W,3] normal maps in [0,1], light_dir / light_col 1 or B rows of 3 -> shading [B,H,W,3] float32.  NumPy in -> NumPy out,
    torch CUDA in -> torch CUDA out.  The caller's light_dir is not normalised in place (:58)."""
    is_np = not isinstance(images_in, torch.Tensor)
    img = torch.as_tensor(np.asarray(images_in, np.float32)) if is_np else images_in
    img = img.to(device="cuda", dtype=torch.float32).contiguous()
    shade, _, _ = ops.phong_shade(img, light_dir, light_col, ambient_in, k_diffuse, composite="tf",
                                  background_white=not with_black_background, with_mask=with_mask, want_compos=False,
                                  want_u8=False)
    return shade.cpu().numpy() if is_np else shade


def np_phong_composite(images_in, light_dir, light_col, ambient_in, k_diffuse, background_col="Black",
                       with_mask=True):
    """:202-228.  (Unlike the reference, the caller's light_dir is not normalised in place, :179.)"""
    white = background_col not in ("Black", "black", "BLACK")
    return _run(images_in, light_dir, light_col, ambient_in, k_diffuse, white, with_mask)


def np_phong_composite_uint8(images_in, light_dir, light_col, ambient_in, k_diffuse, background_col="Black",
                             with_mask=True):
    """np_phong_composite followed by RenderNet_demo.py:58's clip(255*x,0,255).astype(uint8), fused."""
    white = background_col not in ("Black", "black", "BLACK")
    return _run(images_in, light_dir, light_col, ambient_in, k_diffuse, white, with_mask, want_u8=True)[1]
