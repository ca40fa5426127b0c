"""NumPy-2-safe reader and writer for `#binvox 1` voxel files with the call surface of the reference's tools/binvox_rw.py
(`read_as_3d_array(fp, fix_coords=True)` -> object with `.data/.dims/.translate/.scale/.axis_order`, :45-93; `write(voxel_model,
fp)`, `Voxels.write(fp)` and `save_binvox(data, fname)`, :42-43,175-239, which write the reference's bytes).

Format: an ASCII header (`#binvox 1`, `dim X Y Z`, `translate tx ty tz`, `scale s`, `data`) followed by run-length
(value, count) byte pairs in x-z-y order; `fix_coords` re-orders the axes to x-y-z.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List

import numpy as np


@dataclass
class Voxels:
    data: np.ndarray
    dims: List[int]
    translate: List[float]
    scale: float
    axis_order: str = "xyz"
    meta: dict = field(default_factory=dict)

    def clone(self) -> "Voxels":
        return Voxels(self.data.copy(), list(self.dims), list(self.translate), self.scale, self.axis_order, dict(self.meta))

    def write(self, fp):
        write(self, fp)


def read_header(fp):
    """Parse the five header lines; returns (dims, translate, scale)."""
    magic = fp.readline().strip()
    if not magic.startswith(b"#binvox"):
        raise IOError("Not a binvox file")
    fields = {}
    for _ in range(3):
        key, *vals = fp.readline().split()
        fields[key] = vals
    if fp.readline().strip() != b"data":
        raise IOError("binvox header: 'data' marker missing")
    dims = [int(v) for v in fields[b"dim"]]
    translate = [float(v) for v in fields[b"translate"]]
    scale = float(fields[b"scale"][0])
    return dims, translate, scale


def read_as_3d_array(fp, fix_coords=True) -> Voxels:
    dims, translate, scale = read_header(fp)
    pairs = np.frombuffer(fp.read(), dtype=np.uint8).reshape(-1, 2)
    dense = np.repeat(pairs[:, 0] != 0, pairs[:, 1].astype(np.int64))
    if dense.size != int(np.prod(dims)):
        raise IOError(f"binvox payload decodes to {dense.size} voxels, header says {int(np.prod(dims))}")
    grid = dense.reshape(dims)                     # stored x, z, y
    if fix_coords:
        return Voxels(np.ascontiguousarray(grid.transpose(0, 2, 1)), dims, translate, scale, "xyz")
    return Voxels(grid, dims, translate, scale, "xzy")


def read_rle(fp):
    """Header + the undecoded (value, count) byte pairs: (dims, translate, scale, pairs uint8 [n_runs, 2])."""
    dims, translate, scale = read_header(fp)
    raw = np.frombuffer(fp.read(), dtype=np.uint8)
    if raw.size % 2:
        raise IOError("binvox payload has an odd number of bytes")
    pairs = raw.reshape(-1, 2)
    if int(pairs[:, 1].astype(np.int64).sum()) != int(np.prod(dims)):
        raise IOError(f"binvox payload decodes to {int(pairs[:, 1].astype(np.int64).sum())} voxels, "
                      f"header says {int(np.prod(dims))}")
    return dims, translate, scale, pairs


def _rle(flat: np.ndarray) -> bytes:
    """The (value, count) byte pairs of the reference writer's state machine (tools/binvox_rw.py:206-226): runs of equal values
    split into counts of 255; a run that ends exactly at a multiple of 255 and is followed by another value still emits a
    (value, 0) pair, because the writer dumps its counter when the value changes even after the counter was reset."""
    flat = np.asarray(flat).astype(np.uint8).ravel()
    if flat.size == 0:
        return b""
    starts = np.flatnonzero(np.r_[True, flat[1:] != flat[:-1]])
    lengths = np.diff(np.r_[starts, flat.size])
    out = []
    last = len(starts) - 1
    for k, (s, n) in enumerate(zip(starts.tolist(), lengths.tolist())):
        v = int(flat[s])
        full, rest = divmod(n, 255)
        out.extend((v, 255) * full)
        if rest or k < last:
            out.extend((v, rest))
    return bytes(out)


def write(voxel_model: Voxels, fp) -> None:
    """Write `voxel_model` (dense `data`, axis_order "xyz" or "xzy") as binary binvox, byte for byte as the reference's
    tools/binvox_rw.py:175-226: the header prints dims, translate and scale with str(), the payload runs in x-z-y order."""
    if voxel_model.axis_order not in ("xzy", "xyz"):
        raise ValueError("Unsupported voxel model axis order")
    data = np.asarray(voxel_model.data)
    if data.ndim != 3:
        raise ValueError(f"binvox write: dense 3-D data expected, not shape {data.shape}")
    fp.write(("#binvox 1\n" + "dim " + " ".join(map(str, voxel_model.dims)) + "\n" + "translate " +
              " ".join(map(str, voxel_model.translate)) + "\n" + "scale " + str(voxel_model.scale) + "\n" + "data\n")
             .encode("latin-1"))
    flat = data.ravel() if voxel_model.axis_order == "xzy" else np.transpose(data, (0, 2, 1)).ravel()
    fp.write(_rle(flat))


def save_binvox(data, fname) -> None:
    """Save a dense 3-D occupancy array (x-y-z) as a .binvox file: translate 0, scale 1.0 (tools/binvox_rw.py:228-239)."""
    model = Voxels(data, data.shape, [0.0, 0.0, 0.0], 1.0, "xyz")
    with open(fname, "wb") as f:
        model.write(f)


def read_to_device(fps, fix_coords=True, device="cuda"):
    """Decode one or more binvox files ON THE GPU (`rn_binvox_decode`): only the 6-12 KB run-length payloads cross PCIe
    instead of 1 MiB of float32 per grid.  Returns float32 [n, d0, d2, d1, 1] -- what RenderNet_demo.py:125-127 builds
    with `read_as_3d_array(f).data.astype(float32)` reshaped to (1, 64, 64, 64, 1).  All files must share `dims`."""
    from . import ops
    if not isinstance(fps, (list, tuple)):
        fps = [fps]
    items = [read_rle(fp) for fp in fps]
    dims = items[0][0]
    if any(it[0] != dims for it in items):
        raise ValueError("read_to_device: all files must have the same dims")
    return ops.binvox_decode([it[3] for it in items], dims, fix_coords, device)
