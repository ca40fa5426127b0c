"""The dataset's file-naming convention (tools/data_util.py:13-29): an image of a shape rendered at azimuth az, elevation parameter
el and radius r is named `..._p<az>_t<el>_r<r>...` (degrees; el in [10, 170] with the up axis at 0).  The reference's data loaders
are not mirrored here."""
from __future__ import annotations

import math

import numpy as np


def extract_param_from_names(image_path: str) -> np.ndarray:
    """Pose [1,3] (azimuth radians, elevation radians, scale) of a name holding "_p<az>_t<el>_r<r>".

    As the reference: the azimuth is the text between "_p" and "_t", the elevation 90 degrees minus the text between "_t" and
    "_r" (so [10, 170] maps to [80, -80]), and the scale 3.3 over the three characters after "_r" (e.g. "3.3" -> 1.0; a longer
    radius is cut to three characters)."""
    p, t, r = image_path.find("_p"), image_path.find("_t"), image_path.find("_r")
    if min(p, t, r) < 0:
        raise ValueError(f"{image_path!r} does not follow the _p<azimuth>_t<elevation>_r<radius> naming")
    azimuth = float(image_path[p + 2:t]) * math.pi / 180.0
    elevation = (90.0 - float(image_path[t + 2:r])) * math.pi / 180.0
    scale = 3.3 / float(image_path[r + 2:r + 5])
    return np.array([[azimuth, elevation, scale]])
