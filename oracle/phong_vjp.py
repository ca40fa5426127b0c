"""Closed-form float64 vector-Jacobian products of the two Phong composites: tf_vjp64 (TensorFlow's, oracle/phong_tf.py) and
np_vjp64 (the demo's NumPy one, oracle/phong_np.py), for testing rn_phong_recon_loss_grad, rn_phong_composite_loss_grad and
rn_phong_shade_backward at every pixel a normal map can hold.

The autograd restatements are NaN where the composite has no derivative: at n = (0.5, 0.5, 0.5), where u = v / |v| is 0/0,
and where the mask's d|a|/da = a / |a| is 0/0 (|n| = 0 for TF, |img| = 0 or |1 - img| = 0 for NumPy).  These carry the device
kernels' conventions (rn_phong.cuh tf_phong_pixel_backward / phong_pixel_backward) instead:
  - max(x, 0) passes where x >= 0, a clip where lo <= x <= hi (both inclusive), as torch.clamp's derivative does;
  - at n = (0.5, 0.5, 0.5) the pixel is shaded as unlit, and where max(d, 0) passes nothing the normal's and the light's terms
    are exactly 0;
  - the mask term is 0 where |n| = 0 (TF) or |a| = 0 (NumPy).
The NumPy composite's mask takes its fp32 value (mask32, the value phong_pixel computes) while its derivative is the float64
sigmoid's, as tests/test_gpu_nn.py evaluates oracle/phong_np.py.
"""
import math

import numpy as np


def mask32(n, white):
    """The fp32 mask phong_pixel evaluates, emulated in float64 with one rounding per operation: [..., 3] -> [..., 1]."""
    a = (1.0 - n.astype(np.float64)).astype(np.float32) if white else n
    a = a.astype(np.float64)
    f32 = lambda x: np.asarray(x, np.float64).astype(np.float32).astype(np.float64)   # noqa: E731
    s = f32(a[..., 0] * a[..., 0])
    s = f32(a[..., 1] * a[..., 1] + s)
    s = f32(a[..., 2] * a[..., 2] + s)
    arg = f32(255.0 * f32(np.sqrt(s)) - (80.0 if white else 150.0))
    with np.errstate(over="ignore"):
        return f32(1.0 / f32(1.0 + f32(np.exp(-arg))))[..., None]


def _unit(x):
    """(x / |x|, |x|) over the last axis; x / |x| is 0 where |x| = 0."""
    nrm = np.sqrt((x * x).sum(-1, keepdims=True))
    return np.divide(x, nrm, out=np.zeros_like(x), where=nrm > 0), nrm


def _vjp64(n, light_dir, light_col, ambient, k_diffuse, g, albedo, mask):
    """mask: None, or (s, ds/dn, fp32 mask value or None) with s the sigmoid's argument [..., 1] and ds/dn [..., 3] (0 where
    the norm in it is 0)."""
    n = np.asarray(n, np.float64)
    B = n.shape[0]
    l = np.asarray(light_dir, np.float64).reshape(-1, 3) * np.ones((B, 1))
    lnorm = np.sqrt((l * l).sum(-1, keepdims=True))
    L = l / lnorm
    Lp = L.reshape(B, 1, 1, 3)
    col = (np.asarray(light_col, np.float64).reshape(-1, 3) * np.ones((B, 1))).reshape(B, 1, 1, 3)
    u, vn = _unit(n - 0.5)
    d = (u * Lp).sum(-1, keepdims=True)
    lit = (vn > 0) & (d >= 0)                                  # where max(d, 0) passes; n = 0.5 is unlit
    pre = k_diffuse * np.where(lit, d, 0.0) * col
    dif = np.clip(pre, 0.0, 1.0)
    if mask is None:
        x = ambient + dif
    else:
        s, ds_dn, m32 = mask
        m64 = 1.0 / (1.0 + np.exp(-s))
        m = m64 if m32 is None else m32
        x = m * (ambient + dif) + (1.0 - m)
    shade = np.clip(x, 0.0, 1.0)
    g = np.asarray(g, np.float64)
    d_albedo = None if albedo is None else g * shade
    dshade = g if albedo is None else g * np.asarray(albedo, np.float64)
    dx = np.where((x >= 0) & (x <= 1), dshade, 0.0)
    dpre = np.where((pre >= 0) & (pre <= 1), dx if mask is None else dx * m, 0.0)
    dd = np.where(lit, (dpre * k_diffuse * col).sum(-1, keepdims=True), 0.0)
    d_normal = np.divide(dd * (Lp - d * u), vn, out=np.zeros_like(u), where=lit)   # dd/dv = (L - d u) / |v|
    if mask is not None:
        dm = (dx * (ambient + dif - 1.0)).sum(-1, keepdims=True)
        d_normal = d_normal + dm * m64 * (1.0 - m64) * ds_dn
    dLn = (dd * u).sum(axis=(1, 2))                            # dL/d(l / |l|), then through the normalisation
    d_light = (dLn - L * (L * dLn).sum(-1, keepdims=True)) / lnorm
    return shade, d_normal, d_albedo, d_light


def tf_vjp64(n, light_dir, light_col, ambient, k_diffuse, black, with_mask, g, albedo=None):
    """TensorFlow's composite (tools/Phong_shading.py:24-113): n [B,H,W,3], light_dir / light_col [B,3] or [1,3], g = dL/d(compos)
    with compos = albedo * shading (shading alone when albedo is None).  Returns (shading, dL/dn, dL/dalbedo or None, dL/dl)."""
    mask = None
    if with_mask:
        un, nn_ = _unit(np.asarray(n, np.float64))
        s = 255.0 * nn_ - 80.0 if black else 255.0 * (math.sqrt(3) - nn_) - 80.0
        mask = (s, (255.0 if black else -255.0) * un, None)
    return _vjp64(n, light_dir, light_col, ambient, k_diffuse, g, albedo, mask)


def np_vjp64(img, light_dir, light_col, ambient, k_diffuse, white, with_mask, g, albedo=None):
    """The demo's NumPy composite (tools/Phong_shading.py:138-228), arguments and results as tf_vjp64; the mask's value is
    mask32's, its derivative the float64 sigmoid's."""
    mask = None
    if with_mask:
        img = np.asarray(img, np.float32)
        a = 1.0 - img.astype(np.float64) if white else img.astype(np.float64)
        ua, na = _unit(a)
        s = 255.0 * na - (80.0 if white else 150.0)
        mask = (s, (-255.0 if white else 255.0) * ua, mask32(img, white))
    return _vjp64(img, light_dir, light_col, ambient, k_diffuse, g, albedo, mask)
