"""Float64 resampler whose cells are the device's, for differentiating through the trilinear weights.

Trilinear interpolation is continuous in the sample coordinate, but its derivative is not: it jumps across every cell face, and
`floor()` of the coordinate picks the cell.  The device computes the coordinates in fp32 (`sample_coord`, rn_ops.cu: the
oracle's `np.matmul` FMA order, DESIGN §5).  A reference that computes them in float64 puts the points that lie within an ulp of
an integer -- every axis-aligned pose has thousands -- in a different cell, or on the other side of the cube's border, and so
differentiates a different patch than the device does.  Here the coordinates are emulated bit for bit in fp32; the inside test
and the cell come from them, and the weights are float64 functions of `minv` that take the fp32 coordinate's value, so autograd
returns d/dvox and d/dMinv of the very function the device evaluates (one-sided at cell faces: the derivative of the cell the fp32
coordinate falls in).
"""
import numpy as np
import torch


def output_grid(new_size, transform=True):
    """Homogeneous grid points (gx, gy, gz, 1) [4, N^3] float64 in the output's flat order [p, q, r] (resample_kernel): with the
    axis transform (gx, gy, gz) = (r, N-1-p, q), without it (r, q, p)."""
    N = new_size
    p, q, r = np.meshgrid(np.arange(N, dtype=np.float64), np.arange(N, dtype=np.float64), np.arange(N, dtype=np.float64),
                          indexing="ij")
    gy, gz = ((N - 1) - p, q) if transform else (q, p)
    return np.stack([r, gy, gz, np.ones_like(p)], 0).reshape(4, -1)


def _two_sum(a, b):
    """s + e == a + b exactly, s = fl64(a + b)."""
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


def _round32(s, e):
    """fp32 round-to-nearest-even of the exact value s + e (|e| <= half an ulp of s in float64).  fl32(s) is that rounding
    unless s sits exactly halfway between two fp32 values and e != 0: then the side e points to wins."""
    r = s.astype(np.float32)
    d = s - r.astype(np.float64)
    nb = np.nextafter(r, np.where(d > 0, np.float32(np.inf), np.float32(-np.inf)).astype(np.float32))
    halfway = (d != 0) & (s == (r.astype(np.float64) + nb.astype(np.float64)) * 0.5)
    return np.where(halfway & (e != 0) & (np.sign(e) == np.sign(d)), nb, r)


def _fma32(a, b, c):
    """fp32 fmaf(a, b, c) for fp32 a, c and an integer b with |b| < 2^29 (a * b is then exact in float64)."""
    return _round32(*_two_sum(a.astype(np.float64) * b, c.astype(np.float64)))


def sample_coords(minv, g):
    """fp32 sample coordinates [B,3,P] exactly as `sample_coord` computes them: fadd(fma(m2,gz, fma(m1,gy, m0*gx)), m3), one
    rounding per operation.  minv [B,3,4] fp32, g [4,P] integer grid points (output_grid)."""
    m = np.asarray(minv, np.float32)[..., None]                  # [B,3,4,1]
    gx, gy, gz = g[0], g[1], g[2]
    assert np.abs(g[:3]).max() < 2 ** 29 and np.array_equal(g[:3], np.round(g[:3]))
    t = (m[:, :, 0].astype(np.float64) * gx).astype(np.float32)  # the product is exact: one rounding
    t = _fma32(m[:, :, 1], gy, t)
    t = _fma32(m[:, :, 2], gz, t)
    return _round32(*_two_sum(t.astype(np.float64), m[:, :, 3].astype(np.float64)))


def resample(vox, minv, new_size, transform=True, device_cells=True):
    """rn_resample_f32 in float64, differentiable w.r.t. vox [B,S,S,S,C] and minv [B,3,4] (float64 tensors; minv's values must be
    fp32 numbers, as the device receives them) -> [B,N,N,N,C].  Zero outside [0, S-1)^3 (resample_kernel's rule).

    device_cells=False takes the inside test, the cells and the weights from float64 coordinates instead: the same function
    away from cell faces, a different one-sided derivative at them (kept to show what the device-cell form changes)."""
    B, S, C = vox.shape[0], vox.shape[1], vox.shape[-1]
    m64 = minv.detach().numpy()
    g = output_grid(new_size, transform)
    if device_cells:
        if not np.array_equal(m64.astype(np.float32).astype(np.float64), m64):
            raise ValueError("minv must hold fp32 values: the device computes its sample coordinates from fp32 entries")
        cells = torch.from_numpy(sample_coords(m64, g).astype(np.float64))
    else:
        cells = torch.from_numpy(np.matmul(m64, g))
    lim = S - 1
    inside = ((cells >= 0) & (cells < lim)).all(1)                                    # [B,P]
    gt = torch.from_numpy(g)
    out = []
    for b in range(B):
        idx = inside[b].nonzero()[:, 0]
        c = cells[b][:, idx]
        x64 = minv[b] @ gt[:, idx]                                                     # [3,n], carries d/dminv
        x = c + (x64 - x64.detach()) if device_cells else x64                          # value: the (fp32) coordinate
        base = torch.floor(c)
        f = x - base                                                                   # (bx, by, bz); (ax, ay, az) = 1 - f
        i0 = base.long()
        flat = vox[b].reshape(-1, C)
        acc = 0
        for dz in (0, 1):
            wz = f[2] if dz else 1 - f[2]
            for dy in (0, 1):
                wy = f[1] if dy else 1 - f[1]
                for dx in (0, 1):
                    wx = f[0] if dx else 1 - f[0]
                    k = ((i0[2] + dz) * S + (i0[1] + dy)) * S + (i0[0] + dx)
                    acc = acc + (wx * wy * wz).unsqueeze(-1) * flat[k]
        out.append(torch.zeros((new_size ** 3, C), dtype=torch.float64).index_copy(0, idx, acc))
    return torch.stack(out).reshape(B, new_size, new_size, new_size, C)
