"""rendernet_b200 -- H100-native (sm_90a) implementation of RenderNet's forward rendering hot path.

Host side mirrors the reference's Python call surface (tools/layer_util.py, tools/resampling_voxel_grid.py,
tools/model_util.py, tools/Phong_shading.py, tools/binvox_rw.py, RenderNet_Shader.py, RenderNet_demo.py);
all arithmetic runs in hand-written CUDA kernels behind the C ABI in include/rendernet_b200.h.
Importing the package loads librendernet_b200.so and fails loudly if it is missing.
"""
from . import _lib  # noqa: F401  (raises ImportError when the CUDA extension is not built)

__version__ = "0.1.0"
