"""Differentiable (torch) restatement of the reference's NumPy Phong composite (tools/Phong_shading.py:138-228 np_mask /
np_mask_white / np_phong_shading / np_phong_composite, the demo's shading, RenderNet_demo.py:54-58) and of its light position
(:247-253), for testing rn_phong_composite_loss_grad and rendernet_b200.shader_fit in float64.

Every kink is written with torch.clamp, whose derivative passes at the bounds inclusive (max(x, 0) where x >= 0, a clip where
lo <= x <= hi), the convention the device kernel documents.  The forward is held to the reference's own code by
tests/golden/phong.npz (tests/golden/make_golden.py).
"""
import torch


def _norm(x, dim):
    return torch.sqrt((x * x).sum(dim, keepdim=True))


def np_mask_arg(images_in, background_white=False):
    """The argument of the soft mask's sigmoid: 255 |img| - 150 (black background, :138-148) or 255 |1 - img| - 80 (white,
    :150-160)."""
    return 255.0 * _norm(1.0 - images_in, -1) - 80 if background_white else 255.0 * _norm(images_in, -1) - 150


def np_phong_composite(images_in, light_dir, light_col, ambient_in, k_diffuse, background_white=False, with_mask=True,
                       mask_value=None):
    """images_in [B,H,W,3] in [0,1]; light_dir, light_col [B,3] (the direction is normalised here, :179) -> [B,H,W,3].

    mask_value: None, or a [B,H,W,1] tensor the mask takes as its VALUE while its derivative stays the float64 sigmoid's (to
    evaluate the gradient at another implementation's rounded mask)."""
    B = images_in.shape[0]
    v = images_in - 0.5
    u = v / _norm(v, -1)
    L = light_dir / _norm(light_dir, -1)
    d = (u * L.reshape(B, 1, 1, 3)).sum(-1, keepdim=True)
    diffuse = torch.clamp(k_diffuse * torch.clamp(d, min=0.0) * light_col.reshape(B, 1, 1, 3), 0.0, 1.0)
    if not with_mask:
        return torch.clamp(ambient_in + diffuse, 0.0, 1.0)
    mask = torch.sigmoid(np_mask_arg(images_in, background_white))
    if mask_value is not None:
        mask = mask_value.to(mask.dtype) + (mask - mask.detach())
    return torch.clamp(mask * (ambient_in + diffuse) + (1 - mask), 0.0, 1.0)


def generate_light_pos(light):
    """:247-253 in radians: light [B,2] (azimuth, elevation) -> [B,3] = (-sin(el) cos(az), cos(el), -sin(el) sin(az))."""
    az, el = light[:, 0:1], light[:, 1:2]
    return torch.cat([-torch.sin(el) * torch.cos(az), torch.cos(el), -torch.sin(el) * torch.sin(az)], 1)


def fit_loss(images_in, target, light_dir, light_col, ambient_in=0.1, k_diffuse=0.9, background_white=False, with_mask=True,
             mask_value=None):
    """Per-item mean squared error of the composite against the target (the Shader fit's "phong" objective)."""
    out = np_phong_composite(images_in, light_dir, light_col, ambient_in, k_diffuse, background_white, with_mask, mask_value)
    return ((target - out) ** 2).mean(dim=(1, 2, 3))
