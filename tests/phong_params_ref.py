"""Float64 vector-Jacobian products of the two Phong composites with the shading parameters' gradients: oracle/phong_vjp.py's
tf_vjp64 / np_vjp64 (the same arithmetic and the same conventions at the kinks), extended by dL/d light_col [B,3] and
dL/d ambient [B], with the ambient term per item.  For the *_params kernels (rn_phong.cuh phong_param_backward):
  x_c = m (ambient + clip(pre_c, 0, 1)) + (1 - m)  (no mask: ambient + clip(pre_c, 0, 1)),   pre_c = k_d max(d, 0) col_c
  dL/d ambient = sum_{h,w,c} m dx_c,   dL/d col_c = sum_{h,w} dpre_c k_d max(d, 0)
with dx_c the upstream gradient through clip(x, 0, 1) and dpre_c = m dx_c through clip(pre, 0, 1).
"""
import math

import numpy as np

from oracle.phong_vjp import _unit, mask32


def vjp64(n, light_dir, light_col, ambient, k_diffuse, g, albedo, mask):
    """oracle.phong_vjp._vjp64 with ambient a float or [B] and two more results: (shade, d_normal, d_albedo or None, d_light
    [B,3], d_light_col [B,3], d_ambient [B])."""
    n = np.asarray(n, np.float64)
    B = n.shape[0]
    l = np.asarray(light_dir, np.float64).reshape(-1, 3) * np.ones((B, 1))
    lnorm = np.sqrt((l * l).sum(-1, keepdims=True))
    L = l / lnorm
    Lp = L.reshape(B, 1, 1, 3)
    col = (np.asarray(light_col, np.float64).reshape(-1, 3) * np.ones((B, 1))).reshape(B, 1, 1, 3)
    amb = (np.asarray(ambient, np.float64).reshape(-1) * np.ones(B)).reshape(B, 1, 1, 1)
    u, vn = _unit(n - 0.5)
    d = (u * Lp).sum(-1, keepdims=True)
    lit = (vn > 0) & (d >= 0)                                  # where max(d, 0) passes; n = 0.5 is unlit
    dmax = np.where(lit, d, 0.0)
    pre = k_diffuse * dmax * col
    dif = np.clip(pre, 0.0, 1.0)
    if mask is None:
        x = amb + dif
        m = m64 = 1.0
    else:
        s, ds_dn, m32 = mask
        m64 = 1.0 / (1.0 + np.exp(-s))
        m = m64 if m32 is None else m32
        x = m * (amb + dif) + (1.0 - m)
    shade = np.clip(x, 0.0, 1.0)
    g = np.asarray(g, np.float64)
    d_albedo = None if albedo is None else g * shade
    dshade = g if albedo is None else g * np.asarray(albedo, np.float64)
    dx = np.where((x >= 0) & (x <= 1), dshade, 0.0)
    dxm = dx * m
    dpre = np.where((pre >= 0) & (pre <= 1), dxm, 0.0)
    dd = np.where(lit, (dpre * k_diffuse * col).sum(-1, keepdims=True), 0.0)
    d_normal = np.divide(dd * (Lp - d * u), vn, out=np.zeros_like(u), where=lit)
    if mask is not None:
        dm = (dx * (amb + dif - 1.0)).sum(-1, keepdims=True)
        d_normal = d_normal + dm * m64 * (1.0 - m64) * ds_dn
    dLn = (dd * u).sum(axis=(1, 2))
    d_light = (dLn - L * (L * dLn).sum(-1, keepdims=True)) / lnorm
    d_col = (dpre * k_diffuse * dmax).sum(axis=(1, 2))
    d_amb = (dxm * np.ones_like(x)).sum(axis=(1, 2, 3))
    return shade, d_normal, d_albedo, d_light, d_col, d_amb


def tf_vjp64(n, light_dir, light_col, ambient, k_diffuse, black, with_mask, g, albedo=None):
    """oracle.phong_vjp.tf_vjp64 plus (d_light_col, d_ambient)."""
    mask = None
    if with_mask:
        un, nn_ = _unit(np.asarray(n, np.float64))
        s = 255.0 * nn_ - 80.0 if black else 255.0 * (math.sqrt(3) - nn_) - 80.0
        mask = (s, (255.0 if black else -255.0) * un, None)
    return vjp64(n, light_dir, light_col, ambient, k_diffuse, g, albedo, mask)


def np_vjp64(img, light_dir, light_col, ambient, k_diffuse, white, with_mask, g, albedo=None):
    """oracle.phong_vjp.np_vjp64 plus (d_light_col, d_ambient); the mask's value is mask32's."""
    mask = None
    if with_mask:
        img = np.asarray(img, np.float32)
        a = 1.0 - img.astype(np.float64) if white else img.astype(np.float64)
        ua, na = _unit(a)
        s = 255.0 * na - (80.0 if white else 150.0)
        mask = (s, (-255.0 if white else 255.0) * ua, mask32(img, white))
    return vjp64(img, light_dir, light_col, ambient, k_diffuse, g, albedo, mask)
