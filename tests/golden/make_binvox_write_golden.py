#!/usr/bin/env python
"""Generate tests/golden/binvox_write.npz: the bytes the REFERENCE'S OWN binvox writer produces.

Needs a checkout of the reference (thunguyenphuoc/RenderNet); the tests only read the stored fixture:
    python tests/golden/make_binvox_write_golden.py /path/to/RenderNet

`tools/binvox_rw.py` is imported unmodified from that checkout, with the NumPy aliases it uses (np.bool, np.int) restored as
make_golden.py does; the grids are passed as 0 / 1 uint8 (see main).  Each case is written with the reference's
`save_binvox(data, fname)`, with `Voxels(...).write(fp)` at a non-default header, and with `write` in x-z-y axis order:
  * the five shapes of tests/golden/binvox.npz;
  * "soft": a soft grid (the chair at 0.75 plus seeded noise, smoothed) thresholded at 0.1, as the reference saves its
    reconstructions (Reconstruct_RenderNet_Face.py:516);
  * "runs": a grid whose x-z-y payload has runs of exactly 255, 510 and 255 followed by a change of value, the case in which
    the reference writer emits a (value, 0) pair, and a last run of exactly 255 (no pair after it).
"""
import io
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = sys.argv[1] if __name__ == "__main__" and len(sys.argv) > 1 else os.environ.get("RENDERNET_REFERENCE", "")

SHAPES = ("bunny", "chair", "suzanne", "table", "teapot")


def soft_grid():
    bv = np.load(os.path.join(HERE, "binvox.npz"))
    chair = np.unpackbits(bv["chair_bits"]).reshape(64, 64, 64).astype(np.float64)
    g = 0.75 * chair + 0.2 * np.random.default_rng(11).random((64, 64, 64))
    for ax in range(3):                                  # a [1, 2, 1] / 4 blur along each axis
        g = 0.25 * np.roll(g, 1, ax) + 0.5 * g + 0.25 * np.roll(g, -1, ax)
    return (g * 0.3).astype(np.float32)


def runs_grid():
    """x-y-z grid whose x-z-y flat payload is 255 zeros, 510 ones, 7 zeros, 255 ones, then zeros ending in 255 ones."""
    n = 64 ** 3
    flat = np.zeros(n, bool)
    flat[255:765] = True
    flat[772:1027] = True
    flat[n - 255:] = True
    return np.ascontiguousarray(flat.reshape(64, 64, 64).transpose(0, 2, 1))


def cases():
    bv = np.load(os.path.join(HERE, "binvox.npz"))
    out = {nm: np.unpackbits(bv[nm + "_bits"]).reshape(64, 64, 64).astype(bool) for nm in SHAPES}
    out["soft"] = soft_grid() > 0.1
    out["runs"] = runs_grid()
    return out


def main():
    if not REF or not os.path.isdir(os.path.join(REF, "tools")):
        raise SystemExit("usage: make_binvox_write_golden.py /path/to/RenderNet (the reference checkout)")
    if not hasattr(np, "bool"):
        np.bool = bool
    if not hasattr(np, "int"):
        np.int = int
    sys.path.insert(0, REF)
    from tools import binvox_rw                          # the reference module
    store = {}
    with tempfile.TemporaryDirectory() as tmp:
        for nm, grid in cases().items():
            # NumPy 2's bool scalars have no __index__, so the writer's chr(state) would raise on a bool array: hand it the
            # same 0 / 1 values as uint8 (identical comparisons and identical bytes)
            data = grid.astype(np.uint8)
            if nm not in SHAPES:
                store[nm + "_bits"] = np.packbits(grid.ravel())
            fname = os.path.join(tmp, nm + ".binvox")
            binvox_rw.save_binvox(data, fname)
            with open(fname, "rb") as f:
                store[nm + "_save"] = np.frombuffer(f.read(), np.uint8)
            buf = io.BytesIO()
            binvox_rw.Voxels(data, [64, 64, 64], [0.5, -1.25, 3.0], 2.5, "xyz").write(buf)
            store[nm + "_write"] = np.frombuffer(buf.getvalue(), np.uint8)
            buf = io.BytesIO()
            binvox_rw.write(binvox_rw.Voxels(np.ascontiguousarray(data.transpose(0, 2, 1)), [64, 64, 64], [0.0, 0.0, 0.0], 1.0,
                                             "xzy"), buf)
            store[nm + "_write_xzy"] = np.frombuffer(buf.getvalue(), np.uint8)
    np.savez_compressed(os.path.join(HERE, "binvox_write.npz"), **store)
    print("wrote", os.path.join(HERE, "binvox_write.npz"), {k: v.shape for k, v in store.items()})


if __name__ == "__main__":
    main()
