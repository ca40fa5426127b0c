"""Render engines: the forward rendering path as one replayable unit.

An engine owns the device-resident state of one model replica -- its OWN variable store (weights + packed kernel
operands, so several engines with different weights / precisions coexist in a process), fixed-shape input / output
buffers and a CUDA graph of the whole step -- so a step is: H2D(inputs) -> graph replay -> D2H(images).
`RenderEngine` is the Shader network (resample -> 3-D encoder -> projection -> 2-D trunk -> decoder [-> Phong],
RenderNet_Shader.py:139-156); `TextureRenderEngine` the Texture/Normal network (RenderNet_Texture_Face_Normal.py:155-179).
This is the call a user makes for throughput; `RenderNet_demo.Session.run` routes through it too.

precision = "fast":  fp16 operands and stored activations, fp32 accumulation (1x tensor-core work); meets the 1e-3 image
                     bar for the reference's initialisers but not for high-gain weights (DESIGN.md §4).
precision = "exact": fp16 hi/lo operand pairs, three tensor-core products per tap (RN_FMT_F16X2); matches the reference's
                     fp32 convolutions to ~1e-6 relative per layer, whatever the weights.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from . import ops
from . import tfcompat as tf
from .RenderNet_Shader import RenderNet
from .resampling_voxel_grid import (ConcatResampledGrid, ResampledGrid, inverse_sampling_matrix,
                                     tf_rotation_around_grid_centroid)


def pose_to_matrix(view_params, size=64, new_size=128) -> np.ndarray:
    """[B,3] (azimuth, elevation-param, scale) -> [B,3,4] fp32 inverse sampling matrices (host arithmetic in the
    reference's operation order, tools/resampling_voxel_grid.py:515-602)."""
    R, S = tf_rotation_around_grid_centroid(np.asarray(view_params, np.float32))
    return inverse_sampling_matrix(R, S, size, new_size)


class _EngineBase:
    """Shared machinery: private variable store, warm-up + launch counting + CUDA-graph capture of `_forward`, the simple
    synchronous `upload`/`step_device` path and the double-buffered `submit`/`result` pipeline."""

    def __init__(self, weights: Optional[Dict[str, np.ndarray]], precision: str, seed: int, device: str, use_graph: bool,
                 strict: bool = True):
        if not torch.cuda.is_available():
            raise RuntimeError(f"{type(self).__name__} needs a CUDA device (no CPU fallback)")
        self.device = torch.device(device)
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.precision = precision
        self.store = tf.VariableStore(precision=precision, device=str(self.device), seed=seed)
        if weights is not None:
            with tf.use_store(self.store):
                tf.load_weight_dict(weights, strict=strict)
        self.graph: Optional[torch.cuda.CUDAGraph] = None
        self.launches_per_step: Optional[int] = None
        self._use_graph = use_graph
        self._pipe = None
        self._h2d_done: Optional[torch.cuda.Event] = None
        self.inputs: List[torch.Tensor] = []       # device input buffers, in `_host_inputs` order
        self.inputs_host: List[torch.Tensor] = []  # pinned staging of the synchronous path
        self.outputs: List[torch.Tensor] = []      # device outputs of the last step (stable addresses under the graph)

    # ---- subclass interface -----------------------------------------------------------------------
    def _forward(self) -> Sequence[torch.Tensor]:
        raise NotImplementedError

    def _host_inputs(self, *args) -> Sequence[torch.Tensor]:
        """User arguments -> CPU tensors shaped like `self.inputs` (poses become 3x4 matrices here)."""
        raise NotImplementedError

    @staticmethod
    def _light_rows(t, B, what) -> torch.Tensor:
        t = torch.as_tensor(np.asarray(t.cpu() if isinstance(t, torch.Tensor) else t, np.float32))
        if t.dim() == 1 and t.numel() == 3:
            t = t.reshape(1, 3)
        if t.dim() != 2 or t.shape[1] != 3 or t.shape[0] not in (1, B):
            raise ValueError(f"{what} must have shape [1,3] or [{B},3], not {tuple(t.shape)}")
        return t.expand(B, 3).contiguous()

    # ---- construction ------------------------------------------------------------------------------
    def _run_forward(self):
        with torch.cuda.device(self.device), tf.use_store(self.store):
            self.outputs = list(self._forward())
        return self.outputs

    def _finish_init(self):
        from ._lib import lib
        with torch.cuda.device(self.device):
            self._run_forward()                      # warm-up: packs weights, sets kernel attributes, sizes the allocator
            torch.cuda.synchronize()
            if self.store.strict and self.store.unused():
                import warnings
                warnings.warn(f"{len(self.store.unused())} loaded weights were never used by the model, e.g. "
                              f"{self.store.unused()[:4]} (other network's variables, or a wrong prefix / spelling?)")
            n0 = lib.rn_launch_count()
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                self._run_forward()
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            self.launches_per_step = int(lib.rn_launch_count() - n0)   # kernels of one steady-state step
            if self._use_graph:
                self.graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(self.graph):
                    self._run_forward()
                torch.cuda.synchronize()
            self.inputs_host = [torch.zeros(t.shape, dtype=t.dtype).pin_memory() for t in self.inputs]
            self.outputs_host = [torch.zeros(tuple(t.shape), dtype=t.dtype).pin_memory() for t in self.outputs]

    # ---- synchronous path --------------------------------------------------------------------------
    def step_device(self):
        """One pass over the inputs already resident in the device input buffers."""
        if self.graph is not None:
            self.graph.replay()
        else:
            self._run_forward()
        return self.outputs

    def _upload(self, host_tensors: Sequence[torch.Tensor]):
        if self._h2d_done is not None:
            self._h2d_done.synchronize()             # the previous H2D has finished reading the pinned staging buffers
        for h, t in zip(self.inputs_host, host_tensors):
            h.copy_(t.reshape(h.shape))
        with torch.cuda.device(self.device):
            for d, h in zip(self.inputs, self.inputs_host):
                d.copy_(h, non_blocking=True)
            self._h2d_done = torch.cuda.Event()
            self._h2d_done.record(torch.cuda.current_stream())

    def _download(self, which: Sequence[int]):
        with torch.cuda.device(self.device):
            for i in which:
                self.outputs_host[i].copy_(self.outputs[i], non_blocking=True)
            torch.cuda.current_stream().synchronize()
        return [self.outputs_host[i] for i in which]

    # ---- pipelined path ----------------------------------------------------------------------------
    def _pipe_outputs(self) -> Sequence[int]:
        """Indices into self.outputs that travel to the host in the pipelined path."""
        return list(range(len(self.outputs)))

    def _init_pipeline(self):
        if self._pipe is not None:
            return
        with torch.cuda.device(self.device):
            P = {"s_in": torch.cuda.Stream(), "s_out": torch.cuda.Stream()}
            P["in_host"] = [[torch.zeros(t.shape, dtype=t.dtype).pin_memory() for t in self.inputs] for _ in range(2)]
            P["in_stage"] = [[torch.zeros_like(t) for t in self.inputs] for _ in range(2)]
            src = [self.outputs[i] for i in self._pipe_outputs()]
            P["out_stage"] = [[torch.zeros_like(t) for t in src] for _ in range(2)]
            P["out_host"] = [[torch.zeros(tuple(t.shape), dtype=t.dtype).pin_memory() for t in src] for _ in range(2)]
            for k in ("h2d_done", "stage_free", "out_ready", "d2h_done"):
                P[k] = [torch.cuda.Event() for _ in range(2)]
                for e in P[k]:
                    e.record(torch.cuda.current_stream())
            P["n"] = 0
            torch.cuda.synchronize()
        self._pipe = P

    def _submit(self, host_tensors: Sequence[torch.Tensor]) -> int:
        self._init_pipeline()
        P = self._pipe
        i = P["n"]
        s = i % 2
        P["n"] = i + 1
        P["h2d_done"][s].synchronize()                       # the pinned input slot is no longer being read
        for h, t in zip(P["in_host"][s], host_tensors):
            h.copy_(t.reshape(h.shape))
        with torch.cuda.device(self.device):
            cur = torch.cuda.current_stream()
            with torch.cuda.stream(P["s_in"]):
                P["s_in"].wait_event(P["stage_free"][s])
                for d, h in zip(P["in_stage"][s], P["in_host"][s]):
                    d.copy_(h, non_blocking=True)
                P["h2d_done"][s].record(P["s_in"])
            cur.wait_event(P["h2d_done"][s])
            for d, st in zip(self.inputs, P["in_stage"][s]):
                d.copy_(st)
            P["stage_free"][s].record(cur)
            self.step_device()
            cur.wait_event(P["d2h_done"][s])                 # the output staging slot has been drained
            for st, i_out in zip(P["out_stage"][s], self._pipe_outputs()):
                st.copy_(self.outputs[i_out])
            P["out_ready"][s].record(cur)
            with torch.cuda.stream(P["s_out"]):
                P["s_out"].wait_event(P["out_ready"][s])
                for h, st in zip(P["out_host"][s], P["out_stage"][s]):
                    h.copy_(st, non_blocking=True)
                P["d2h_done"][s].record(P["s_out"])
        return i

    def _result(self, ticket: int) -> List[torch.Tensor]:
        P = self._pipe
        if P is None or ticket >= P["n"]:
            raise RuntimeError("result() of a step that was never submitted")
        if ticket < P["n"] - 2:
            raise RuntimeError("result() of a step whose host slot has been reused (keep at most 2 steps in flight)")
        s = ticket % 2
        P["d2h_done"][s].synchronize()
        return P["out_host"][s]

    @property
    def submitted(self) -> int:
        return 0 if self._pipe is None else self._pipe["n"]


class RenderEngine(_EngineBase):
    def __init__(self, weights: Optional[Dict[str, np.ndarray]], batch: int, is_greyscale: bool = False,
                 size: int = 64, new_size: int = 128, use_graph: bool = True, phong: Optional[dict] = None,
                 seed: int = 0, device: str = "cuda", precision: str = "fast", strict: bool = True,
                 fuse_phong: bool = True):
        """weights: {tf variable name: array} (None -> the reference's initialisers, seeded).
        phong: None, or dict(light_dir[1|B,3], light_col[1|B,3], ambient, k_diffuse) to apply the demo's
        Phong composite + uint8 quantisation; fuse_phong: inside the output layer's epilogue (default) or as a separate pass.
        The light direction and colour are device inputs like the voxels: `upload`, `submit` and `render` take light_dir= and
        light_col= ([1|B,3]; None keeps the last one given, initially phong's), so relighting needs no re-capture.  ambient and
        k_diffuse are fixed here.  precision: "fast" | "exact" (module docstring)."""
        super().__init__(weights, precision, seed, device, use_graph, strict)
        self.B, self.size, self.new_size = batch, size, new_size
        self.is_greyscale = is_greyscale
        dev = self.device
        self.vox = torch.zeros((batch, size, size, size, 1), device=dev, dtype=torch.float32)
        self.minv = torch.zeros((batch, 3, 4), device=dev, dtype=torch.float32)
        self.inputs = [self.vox, self.minv]
        self.phong = phong
        self.fuse_phong = fuse_phong
        if phong is not None:
            # the graph reads these buffers (the fused epilogue through their pointers): a step's light is uploaded into them
            self._light_host = [self._light_rows(np.asarray(phong["light_dir"], np.float32).reshape(-1, 3), batch, "light_dir"),
                                self._light_rows(np.asarray(phong["light_col"], np.float32).reshape(-1, 3), batch, "light_col")]
            self.light_dir, self.light_col = (t.to(dev) for t in self._light_host)
            self.inputs += [self.light_dir, self.light_col]
        self.out = None
        self.out_u8 = None
        self._finish_init()
        self.vox_host, self.minv_host = self.inputs_host[:2]
        self.out_host = self.outputs_host[0]
        self.out_u8_host = self.outputs_host[1] if phong is not None else None

    # -------------------------------------------------------------------------------------------
    def _forward(self):
        grid = ResampledGrid(self.vox, self.minv, self.new_size, transform=True)   # deferred: fuses into e_conv1
        st = self.store
        if self.phong is not None and self.fuse_phong and not self.is_greyscale:
            # the composite runs in the sigmoid epilogue of the last up-conv: no separate pass, no normal-map round trip
            st.phong = dict(light_dir=self.light_dir, light_col=self.light_col, ambient=self.phong["ambient"],
                            k_diffuse=self.phong["k_diffuse"], background_white=self.phong.get("background_white", False),
                            with_mask=self.phong.get("with_mask", True))
        st.phong_u8 = None
        try:
            img = RenderNet(grid, is_training=False, is_greyscale=self.is_greyscale)
        finally:
            st.phong = None
        if self.phong is not None:
            if st.phong_u8 is not None:
                shaded, u8, st.phong_u8 = img, st.phong_u8, None
            else:
                shaded, u8 = ops.phong_composite(img, self.light_dir, self.light_col, self.phong["ambient"],
                                                 self.phong["k_diffuse"],
                                                 background_white=self.phong.get("background_white", False),
                                                 with_mask=self.phong.get("with_mask", True), want_u8=True)
            self.out, self.out_u8 = shaded, u8
            return [shaded, u8]
        self.out = img
        return [img]

    pose_to_matrix = staticmethod(pose_to_matrix)

    def _host_inputs(self, voxels, view_params, light_dir=None, light_col=None):
        v = voxels if isinstance(voxels, torch.Tensor) else torch.as_tensor(np.asarray(voxels, np.float32))
        got = [v, torch.from_numpy(pose_to_matrix(view_params, self.size, self.new_size))]
        if self.phong is None:
            if light_dir is not None or light_col is not None:
                raise ValueError("light_dir / light_col need an engine built with phong=")
            return got
        for i, (t, what) in enumerate(((light_dir, "light_dir"), (light_col, "light_col"))):
            if t is not None:
                self._light_host[i] = self._light_rows(t, self.B, what)
        return got + list(self._light_host)

    def _pipe_outputs(self):
        return [0] if self.phong is None else [1]            # the float image, or the uint8 Phong image

    def step_device(self):
        super().step_device()
        return self.out

    def upload(self, voxels, view_params, non_blocking=True, light_dir=None, light_col=None):
        self._upload(self._host_inputs(voxels, view_params, light_dir, light_col))

    def submit(self, voxels, view_params, light_dir=None, light_col=None) -> int:
        """Asynchronously enqueue one step: pinned-host staging -> H2D (copy stream) -> graph replay (compute
        stream) -> D2H (copy stream).  Uploads of step i+1 and downloads of step i-1 overlap the compute of step i.
        light_dir / light_col (phong engines): this step's light, [1|B,3] (None: the last one given).
        Returns a ticket for `result()`."""
        return self._submit(self._host_inputs(voxels, view_params, light_dir, light_col))

    def result(self, ticket: int) -> torch.Tensor:
        """Block until the step `ticket` (one of the last two submitted) has landed in pinned host memory."""
        return self._result(ticket)[0]

    def render(self, voxels, view_params, to_host: bool = True, light_dir=None, light_col=None):
        """voxels [B,64,64,64,1] float32 (host), view_params [B,3] -> image [B,512,512,3|1] float32
        (and uint8 Phong image when configured; light_dir / light_col as in `submit`).  Includes H2D and D2H."""
        self.upload(voxels, view_params, light_dir=light_dir, light_col=light_col)
        self.step_device()
        if not to_host:
            return self.out if self.phong is None else (self.out, self.out_u8)
        got = self._download([0] if self.phong is None else [0, 1])
        return got[0] if self.phong is None else (got[0], got[1])


TEXTURE_PHONG_DEFAULTS = dict(light_col=(1.0, 1.0, 1.0), ambient=0.0, k_diffuse=1.0, composite="tf", background_white=True,
                              with_mask=True)     # the reconstruction's shading (Reconstruct_RenderNet_Face.py:326-328, :377)


class TextureRenderEngine(_EngineBase):
    """BASELINE config 4: voxels + 199-d texture vector + pose -> (albedo image, normal map), as one CUDA graph
    (texture decoder -> two resamplings (C=1, C=4) -> concat -> Texture/Normal RenderNet;
    RenderNet_Texture_Face_Normal.py:155-179).

    model="texture": RenderNet_Texture_Face_Normal's decoder_texture + RenderNet on `weights` {tf variable name: array} (None:
    the seeded initialisers).  model="pretrained": Reconstruct_RenderNet_Face's texture_decoder_pretrained + RenderNet_pretrained
    on the npz-keyed dictionary FaceReconstruction holds (ReLU residual blocks), as backward.TextureInputGradients does.

    phong=dict(light_dir [1|B,3], light_col=(1,1,1), ambient=0., k_diffuse=1., composite="tf", background_white=True,
    with_mask=True) adds the shaded image to the step: compos = albedo * Phong(normal, light) (composite "tf": the reconstruction's
    tf_phong_composite, "numpy": the demo's np_phong_composite) and its uint8 form, in one more kernel inside the same graph.
    The outputs are then (albedo, normal, compos, compos_u8).  The light direction is a device input like the voxels: `upload`,
    `submit` and `render` take light_dir=[1|B,3] (None: the light given here), so relighting needs no re-capture."""

    def __init__(self, weights: Optional[Dict[str, np.ndarray]], batch: int, size: int = 64, new_size: int = 128,
                 use_graph: bool = True, seed: int = 0, device: str = "cuda", precision: str = "fast", strict: bool = True,
                 fuse_input: bool = True, model: str = "texture", phong: Optional[dict] = None):
        if model not in ("texture", "pretrained"):
            raise ValueError(f"model must be 'texture' or 'pretrained', not {model!r}")
        if model == "pretrained" and weights is None:
            raise ValueError("model='pretrained' builds its variables from the npz-keyed weight dictionary: pass one")
        if phong is not None:
            unknown = set(phong) - set(TEXTURE_PHONG_DEFAULTS) - {"light_dir"}
            if unknown or "light_dir" not in phong:
                raise ValueError(f"phong needs light_dir and takes {sorted(TEXTURE_PHONG_DEFAULTS)}; got {sorted(phong)}")
            phong = {**TEXTURE_PHONG_DEFAULTS, **phong}
            if phong["composite"] not in ops.PHONG_COMPOSITES:
                raise ValueError(f"phong composite must be one of {sorted(ops.PHONG_COMPOSITES)}, not {phong['composite']!r}")
            self._light_default = self._light_rows(phong["light_dir"], batch, "light_dir")
            light_col = self._light_rows(phong["light_col"], batch, "light_col")
        super().__init__(weights if model == "texture" else None, precision, seed, device, use_graph, strict)
        self.B, self.size, self.new_size = batch, size, new_size
        self.model = model
        self.weight_dict = weights if model == "pretrained" else None
        self.phong = phong
        self.fuse_input = fuse_input      # False: two stand-alone resamplings + concat + CUDA-core e_conv1 (the r01 path; A/B, tests)
        dev = self.device
        self.vox = torch.zeros((batch, size, size, size, 1), device=dev, dtype=torch.float32)
        self.tex = torch.zeros((batch, 199), device=dev, dtype=torch.float32)
        self.minv = torch.zeros((batch, 3, 4), device=dev, dtype=torch.float32)
        self.inputs = [self.vox, self.tex, self.minv]
        if phong is not None:
            self.light_dir = self._light_default.to(dev)          # the graph reads this buffer: a step's light is uploaded into it
            self.light_col = light_col.to(dev)
            self.inputs.append(self.light_dir)
        self.out = None
        self._finish_init()
        self.vox_host, self.tex_host, self.minv_host = self.inputs_host[:3]
        self.out_host = tuple(self.outputs_host)

    def _forward(self):
        from .RenderNet_Texture_Face_Normal import RenderNet as RenderNetTexture, decoder_texture
        from .Reconstruct_RenderNet_Face import RenderNet_pretrained, texture_decoder_pretrained
        # both resamplings stay deferred: resample x2 + axis transform + concat + e_conv1 run as one kernel
        if self.model == "texture":
            tex3d = tf.realize(decoder_texture(self.tex))
        else:
            tex3d = tf.realize(texture_decoder_pretrained(self.tex, self.weight_dict))
        if not self.fuse_input:
            x5 = ops.concat_channels(ops.resample(self.vox, self.minv, self.new_size, True),
                                     ops.resample(tex3d, self.minv, self.new_size, True))
        else:
            x5 = ConcatResampledGrid(ResampledGrid(self.vox, self.minv, self.new_size, transform=True),
                                     ResampledGrid(tex3d, self.minv, self.new_size, transform=True))
        if self.model == "texture":
            self.out = RenderNetTexture(x5, is_training=False)
        else:
            self.out = RenderNet_pretrained(x5, self.weight_dict)
        if self.phong is not None:
            albedo, normal = self.out
            p = self.phong
            _, compos, u8 = ops.phong_shade(normal, self.light_dir, self.light_col, p["ambient"], p["k_diffuse"], albedo=albedo,
                                            composite=p["composite"], background_white=p["background_white"],
                                            with_mask=p["with_mask"], want_shade=False)
            self.out = (albedo, normal, compos, u8)
        return list(self.out)

    def _host_inputs(self, voxels, texture, view_params, light_dir=None):
        got = [torch.as_tensor(np.asarray(voxels, np.float32)), torch.as_tensor(np.asarray(texture, np.float32)),
               torch.from_numpy(pose_to_matrix(view_params, self.size, self.new_size))]
        if self.phong is not None:
            got.append(self._light_default if light_dir is None else self._light_rows(light_dir, self.B, "light_dir"))
        elif light_dir is not None:
            raise ValueError("light_dir needs an engine built with phong=")
        return got

    def _pipe_outputs(self):
        return [0, 1] if self.phong is None else [3]          # (albedo, normal), or the uint8 shaded image

    def step_device(self):
        super().step_device()
        return self.out

    def upload(self, voxels, texture, view_params, light_dir=None):
        self._upload(self._host_inputs(voxels, texture, view_params, light_dir))

    def submit(self, voxels, texture, view_params, light_dir=None) -> int:
        """Pipelined step (see RenderEngine.submit); `result(ticket)` -> (albedo image, normal map) in pinned host memory, or
        with phong the uint8 shaded image alone (what RenderEngine ships).  light_dir: this step's light (None: the engine's)."""
        return self._submit(self._host_inputs(voxels, texture, view_params, light_dir))

    def result(self, ticket: int):
        got = self._result(ticket)
        return tuple(got) if self.phong is None else got[0]

    def render(self, voxels, texture, view_params, light_dir=None):
        """-> (albedo, normal) fp32 [B,512,512,3] on the host, or with phong (albedo, normal, compos fp32, compos uint8)."""
        self.upload(voxels, texture, view_params, light_dir)
        self.step_device()
        return tuple(self._download(range(len(self.outputs))))
