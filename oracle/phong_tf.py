"""Differentiable (torch) restatement of the reference's TensorFlow Phong composite and light position
(tools/Phong_shading.py:24-130) and of the face reconstruction objective (Reconstruct_RenderNet_Face.py:372-383), for testing
rn_phong_recon_loss_grad and Reconstruct_RenderNet_Face.reconstruction_gradients.

Autograd reproduces TF-1's gradient conventions because every kink is written with torch.clamp, whose derivative passes at
the bounds inclusive: tf.maximum(x, 0) passes where x >= 0, clip_by_value where lo <= x <= hi; the norm's derivative is x/|x|.
The forward is held to the reference's own code by tests/golden/phong_tf.npz (tests/golden/make_phong_golden.py).
"""
import math

import torch


def _norm(x, dim):
    return torch.sqrt((x * x).sum(dim, keepdim=True))


def tf_phong_composite(images_in, light_dir, light_col, ambient_in, k_diffuse, with_black_background=False, with_mask=True):
    """images_in [B,H,W,3] in [0,1]; light_dir, light_col [B,3] -> shading [B,H,W,3] (tools/Phong_shading.py:24-113)."""
    B = images_in.shape[0]
    v = images_in - 0.5
    u = v / _norm(v, -1)
    L = light_dir / _norm(light_dir, -1)
    d = (u * L.reshape(B, 1, 1, 3)).sum(-1, keepdim=True)
    diffuse = torch.clamp(k_diffuse * torch.clamp(d, min=0.0) * light_col.reshape(B, 1, 1, 3), 0.0, 1.0)
    if not with_mask:
        return torch.clamp(ambient_in + diffuse, 0.0, 1.0)
    n = _norm(images_in, -1)
    s = 255.0 * n - 80 if with_black_background else 255.0 * (math.sqrt(3) - n) - 80
    mask = torch.sigmoid(s)
    return torch.clamp(mask * (ambient_in + diffuse) + (1 - mask), 0.0, 1.0)


def tf_generate_light_pos(batch_light_azimuth, light_elevation):
    """tools/Phong_shading.py:115-130: [B,1] azimuths, one elevation -> [B,3] light positions."""
    el = torch.full_like(batch_light_azimuth, float(light_elevation))
    return torch.cat([torch.sin(el) * torch.cos(batch_light_azimuth), torch.sin(el) * torch.sin(batch_light_azimuth),
                      torch.cos(el)], 1)


def recon_loss(albedo, normal, target, light_dir, light_col, ambient=0.0, k_diffuse=1.0, with_black_background=False,
               with_mask=True):
    """Reconstruct_RenderNet_Face.py:377-383: per-item mean squared error of albedo * shading against the target."""
    shade = tf_phong_composite(normal, light_dir, light_col, ambient, k_diffuse, with_black_background, with_mask)
    return ((target - albedo * shade) ** 2).mean(dim=(1, 2, 3))
