"""The renderer as PyTorch autograd layers: `loss.backward()` through RenderNet like through any other layer.

    from rendernet_b200.nn import ShaderRenderer, TextureRenderer, ShapeDecoder, phong_shade

    r = ShaderRenderer(weights, precision="exact", trainable=False)   # weights: {tf name: array} or None (seeded initialisers)
    img = r(voxels, view_params)                 # [B,64,64,64(,1)] CUDA fp32, [B,3] -> [B,512,512,3|1]; any B
    shaded = phong_shade(img, light_dir, composite="numpy", ambient=0.1, k_diffuse=0.9, background_white=False)
    loss = torch.nn.functional.l1_loss(shaded, target)
    loss.backward()                              # voxels.grad, view_params.grad, light_dir.grad (and parameter .grad if trainable)

No new arithmetic here: a module's forward records the tape of the existing gradient objects (backward.ShaderInputGradients,
TextureInputGradients, ShapeDecoderGradients; one per batch size, all sharing the module's variable store, so weights are
packed once per module) and its backward is their reverse walk, asked only for what `ctx.needs_input_grad` says.  The
Phong composite's gradient for an arbitrary upstream gradient is rn_phong_shade_backward.

Semantics:
  * trainable=True: every variable of the store is an nn.Parameter in `params` (an nn.ParameterDict keyed by the TF name, so
    state_dict keys are "params.<tf name>"); the Parameters ARE the store's fp32 device masters.  Before each forward the
    parameters' versions are compared with those the packed (kernel-layout) filters were made from; any change (an optimiser
    step, an in-place edit) drops the packed copies.  An in-place edit between a forward and its backward raises RuntimeError.
  * A forward records as ShaderTrainer does (pre-activations kept) when a parameter needs a gradient -- one walk then gives
    the parameter and the input gradients -- as the input-gradient objects do when only inputs do, and records nothing under
    torch.no_grad() or when nothing needs a gradient.  The two recordings evaluate the PReLU pre-activations with different
    kernels, so at the few elements whose pre-activation is within a few ulps of 0 they may take opposite branches of the kink
    (DESIGN §8b).
  * Each autograd node owns its recording: several forwards may be outstanding.  The recording (every activation of the
    forward) is dropped as soon as the node's backward has run, as autograd frees saved tensors; to walk a node twice, set
    `retain_recording = True` on the module and pass retain_graph=True.  A node returns aliases of the recorded outputs, so
    the tape never refers back to the node.  Double backward is not supported.
  * The loss scale of the 16-bit walk is chosen per call as in the gradient objects; an overflow that survives the retries
    raises FloatingPointError out of backward().
  * Dropout is never applied (train() does not turn it on); the pretrained Texture+Normal model is a constant.
  * ShapeDecoder(weight_dict_decoder, trainable=True) fine-tunes the face-reconstruction shape decoder: its 12 variables
    (g_zP/g_gc1/weights ... g_conv5/biases) are Parameters under the same rules, their gradients come from
    ShapeDecoderGradients' walk (rn_conv3d_f32_weight_grad, rn_fully_connected_param_grad), and decoder_weight_dict() returns
    them under their npz keys, the dictionary ShapeDecoderGradients and FaceReconstruction take.
"""
from __future__ import annotations

from types import SimpleNamespace
from typing import Dict, Optional

import numpy as np
import torch
from torch import nn
from torch.autograd.function import once_differentiable

from . import ops
from . import tfcompat as tf
from .RenderNet_Shader import RenderNet
from .backward import ShaderInputGradients, ShapeDecoderGradients, TextureInputGradients
from .engine import pose_to_matrix
from .resampling_voxel_grid import ResampledGrid

SIZE = 64
PARAMS_PREFIX = "params."


def param_key(tf_name: str) -> str:
    """state_dict key of the Parameter of a TF variable."""
    return PARAMS_PREFIX + tf_name


def tf_name_of(key: str) -> str:
    """TF variable name of a state_dict key (param_key's inverse)."""
    if not key.startswith(PARAMS_PREFIX):
        raise KeyError(f"{key!r} is not a parameter key")
    return key[len(PARAMS_PREFIX):]


# ----------------------------------------------------------------------------------------------- argument checks (no launch)
def _check_voxels(voxels) -> int:
    if not isinstance(voxels, torch.Tensor):
        raise TypeError(f"voxels must be a CUDA tensor, not {type(voxels).__name__}")
    shp = tuple(voxels.shape)
    if len(shp) not in (4, 5) or shp[1:4] != (SIZE,) * 3 or (len(shp) == 5 and shp[4] != 1) or shp[0] < 1:
        raise ValueError(f"voxels must be [B,{SIZE},{SIZE},{SIZE}] or [B,{SIZE},{SIZE},{SIZE},1], not {shp}")
    if voxels.dtype != torch.float32:
        raise TypeError(f"voxels must be float32, not {voxels.dtype}")
    if not voxels.is_cuda:
        raise TypeError("voxels must be a CUDA tensor (there is no CPU path)")
    return shp[0]


def _rows(x, B: int, n: int, what: str) -> None:
    shp = tuple(x.shape) if isinstance(x, torch.Tensor) else np.shape(x)
    if tuple(shp) != (B, n):
        raise ValueError(f"{what} must be [{B},{n}], not {tuple(shp)}")


def _host_f32(x) -> np.ndarray:
    if isinstance(x, torch.Tensor):
        return np.ascontiguousarray(x.detach().to(device="cpu", dtype=torch.float32).numpy())
    return np.ascontiguousarray(np.asarray(x, np.float32))


def _like(a, ref):
    """Host/device array `a` as a tensor on the device and with the dtype of the tensor `ref`."""
    return torch.as_tensor(np.asarray(a) if not isinstance(a, torch.Tensor) else a).to(device=ref.device, dtype=ref.dtype)


def _grad_mode(params, *inputs) -> Optional[str]:
    """"train" (a parameter needs a gradient: ShaderTrainer's tape, pre-activations kept; the walk also gives whatever input
    gradients are asked for), "input" (only inputs do: the input-gradient objects' tape) or None (record nothing)."""
    if not torch.is_grad_enabled():
        return None
    if any(p.requires_grad for p in params):
        return "train"
    if any(isinstance(x, torch.Tensor) and x.requires_grad for x in inputs):
        return "input"
    return None


# ----------------------------------------------------------------------------------------------- shared module machinery
class _Renderer(nn.Module):
    """One variable store, one gradient object per batch size, the masters adopted to the device (as Parameters if trainable)
    and the packed-weight invalidation."""

    def _setup(self, base, trainable: bool):
        self.store = base.store
        self._base = base
        self._objects = {base.B: base}
        dev = self.store.device
        adopted, params = {}, {}
        for name, t in list(self.store.vars.items()):
            d = adopted.get(id(t))
            if d is None:
                nm = getattr(t, "_rn_name", name)
                d = t.detach().to(device=dev, dtype=torch.float32).contiguous()
                if trainable:
                    d = nn.Parameter(d)
                    params[nm] = d
                d._rn_name = nm
                adopted[id(t)] = d
            self.store.vars[name] = d
        self.params = nn.ParameterDict(params)
        self.retain_recording = False                      # keep each node's recording after its backward (retain_graph)
        self._masters = list({id(v): v for v in self.store.vars.values()}.values())
        self._packed_versions = tuple(v._version for v in self._masters)

    def _object(self, B: int):
        o = self._objects.get(B)
        if o is None:
            o = self._make(B)
            o._dgrad_cache = self._base._dgrad_cache        # shared: nothing in it depends on B
            self._objects[B] = o
        return o

    def _sync_packed(self):
        """Drop the packed filters (forward: store.packed; backward: the shared _dgrad_cache, alpha<0 flags included) once a
        master changed since they were made from it."""
        v = tuple(t._version for t in self._masters)
        if v != self._packed_versions:
            self.store.packed.clear()
            self._base._dgrad_cache.clear()
            self._packed_versions = v

    def tf_state_dict(self) -> Dict[str, np.ndarray]:
        """{tf variable name: fp32 ndarray}, loadable by every engine of this package."""
        return {name: t.detach().cpu().numpy().copy() for name, t in self.store.vars.items()}


def _check_versions(ctx):
    for p, v in ctx.versions:
        if p._version != v:
            raise RuntimeError(f"parameter {p._rn_name!r} was modified by an inplace operation after the forward pass this "
                               f"backward differentiates (version {p._version}, recorded {v})")


# what a walk leaves on a gradient object besides the recording: dL/dgrid, the input gradients, the weight gradients
_WALK_RESULTS = ("last_dgrid", "_dgrid", "_dvox", "_dminv", "weight_grads")


def _release(o):
    """Drop the object's references to a recording and to the last walk's results: the node owns them."""
    for k in o._RECORDING + _WALK_RESULTS:
        if hasattr(o, k):
            setattr(o, k, None)


def _take_recording(ctx):
    """The node's recording for its backward; dropped from the node afterwards unless the module retains recordings."""
    rec = ctx.rec
    if rec is None:
        raise RuntimeError("this node's recording was freed by its first backward: set retain_recording = True on the module "
                           "(and pass retain_graph=True) to walk it twice")
    if not ctx.module.retain_recording:
        ctx.rec = None
    return rec


def _record(o, mode, run):
    """Run the model function under the object's store: with a fresh tape (mode "input" / "train", pre-activations kept for
    "train") or with none."""
    st = o.store
    o.tape = [] if mode else None
    st.tape, st.keep_preact = o.tape, mode == "train"
    try:
        with torch.cuda.device(o.device), tf.use_store(st):
            return run()
    finally:
        st.tape, st.keep_preact = None, False


# ----------------------------------------------------------------------------------------------- Shader
class _ShaderFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, module, mode, voxels, view_params, *params):
        B = voxels.shape[0]
        ig = module._object(B)
        ig.view_params = _host_f32(view_params)
        ig.vox = voxels.reshape(B, SIZE, SIZE, SIZE, 1).contiguous()
        ig.minv = torch.from_numpy(pose_to_matrix(ig.view_params, ig.size, ig.new_size)).to(ig.store.device)

        def run():
            grid = ResampledGrid(ig.vox, ig.minv, ig.new_size, transform=True)
            return RenderNet(grid, is_training=mode == "train", prob=1.0, is_greyscale=ig.is_greyscale)

        ig.img = _record(ig, mode, run)
        img = ig.img.detach()                              # the output: an alias, so the tape holds no reference to the node
        ctx.rec = ig._snapshot() if mode else None
        _release(ig)
        if mode:
            ctx.module, ctx.B, ctx.vshape = module, B, tuple(voxels.shape)
            ctx.vp = view_params if isinstance(view_params, torch.Tensor) else None
            ctx.versions = [(p, p._version) for p in params]
            ctx.save_for_backward(voxels, img)
        return img

    @staticmethod
    @once_differentiable
    def backward(ctx, dimg):
        _ = ctx.saved_tensors                              # raises if the voxels or the image were modified in place
        _check_versions(ctx)
        need = ctx.needs_input_grad
        want_dvox, want_dpose, want_w = need[2], need[3], any(need[4:])
        ig = ctx.module._object(ctx.B)
        ig._restore(_take_recording(ctx))
        try:
            dvox, dpose = ig.backward(dimg, want_dvox=want_dvox, want_dpose=want_dpose, want_weight_grads=want_w,
                                      dvox_on_device=True)
            wg = ig.weight_grads if want_w else {}
        finally:
            _release(ig)
        gvox = dvox.reshape(ctx.vshape) if want_dvox else None
        gvp = _like(dpose, ctx.vp) if want_dpose else None
        return (None, None, gvox, gvp) + tuple(wg[p._rn_name] if n else None for (p, _), n in zip(ctx.versions, need[4:]))


class ShaderRenderer(_Renderer):
    """RenderNet_Shader as an autograd layer: forward(voxels, view_params) -> image [B,512,512,3|1] fp32 on the device, for any
    B.  Gradients reach the voxels (dL/dvoxels in the shape passed), the pose (on view_params' device, with its dtype; view_params
    may be a CUDA or CPU tensor or NumPy -- M^-1 is engine.pose_to_matrix on the host) and, with trainable=True, the 166
    parameters.  `weights`: {tf variable name: array} or None (the reference's initialisers, seeded by `seed`)."""

    def __init__(self, weights: Optional[Dict[str, np.ndarray]] = None, precision: str = "exact", is_greyscale: bool = False,
                 trainable: bool = False, loss_scale=None, seed: int = 0, device: str = "cuda"):
        super().__init__()
        self.precision, self.is_greyscale, self.trainable = precision, bool(is_greyscale), bool(trainable)
        self._loss_scale, self._device = loss_scale, device
        base = ShaderInputGradients(weights, 1, precision, is_greyscale, loss_scale=loss_scale, seed=seed, device=device)
        with torch.no_grad():                              # creates the variables (weights None: seeded, in the reference's order)
            _ShaderFn.forward(SimpleNamespace(), _Once(base), None, torch.zeros((1, SIZE, SIZE, SIZE, 1), device=base.store.device),
                              np.array([[0.0, 0.0, 1.0]], np.float32))
        self._setup(base, self.trainable)

    def _make(self, B):
        return ShaderInputGradients(None, B, self.precision, self.is_greyscale, loss_scale=self._loss_scale, device=self._device,
                                    store=self.store)

    def forward(self, voxels, view_params):
        B = _check_voxels(voxels)
        _rows(view_params, B, 3, "view_params")
        self._sync_packed()
        params = list(self.params.values())
        return _ShaderFn.apply(self, _grad_mode(params, voxels, view_params), voxels, view_params, *params)


class _Once:
    """Stand-in module for a constructor's first forward: the one gradient object it has."""

    def __init__(self, o):
        self.o = o

    def _object(self, B):
        return self.o


# ----------------------------------------------------------------------------------------------- Texture+Normal
class _TextureFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, module, mode, voxels, texture, view_params, *params):
        B = voxels.shape[0]
        tig = module._object(B)
        dev = tig.store.device
        tig.view_params = _host_f32(view_params)
        tig.vox = voxels.reshape(B, SIZE, SIZE, SIZE, 1).contiguous()
        tex = texture if isinstance(texture, torch.Tensor) else torch.as_tensor(np.asarray(texture, np.float32))
        tig.tex_in = tex.to(device=dev, dtype=torch.float32).reshape(B, -1).contiguous()
        tig.minv = torch.from_numpy(pose_to_matrix(tig.view_params, tig.size, tig.new_size)).to(dev)
        _record(tig, mode, lambda: tig._record_network(is_training=mode == "train", prob=1.0))
        albedo, normal = tig.albedo.detach(), tig.normal.detach()
        ctx.rec = tig._snapshot() if mode else None
        _release(tig)
        if mode:
            ctx.set_materialize_grads(False)
            ctx.module, ctx.B, ctx.vshape = module, B, tuple(voxels.shape)
            ctx.tex = texture if isinstance(texture, torch.Tensor) else None
            ctx.vp = view_params if isinstance(view_params, torch.Tensor) else None
            ctx.versions = [(p, p._version) for p in params]
            ctx.save_for_backward(voxels, albedo, normal, *([] if ctx.tex is None else [texture]))
        return albedo, normal

    @staticmethod
    @once_differentiable
    def backward(ctx, d_albedo, d_normal):
        _ = ctx.saved_tensors
        _check_versions(ctx)
        need = ctx.needs_input_grad
        want_dvox, want_dtex, want_dpose, want_w = need[2], need[3], need[4], any(need[5:])
        tig = ctx.module._object(ctx.B)
        tig._restore(_take_recording(ctx))
        try:
            dvox, dtex, dpose = tig._walk_outputs(d_albedo, d_normal, want_dvox, want_dtex, want_dpose, want_w, True)
            wg = tig.weight_grads if want_w else {}
        finally:
            _release(tig)
        gvox = dvox.reshape(ctx.vshape) if want_dvox else None
        gtex = _like(dtex, ctx.tex).reshape(ctx.tex.shape) if want_dtex else None
        gvp = _like(dpose, ctx.vp) if want_dpose else None
        zero = (lambda p: torch.zeros_like(p))             # a variable no output gradient reached (e.g. one head unused)
        return (None, None, gvox, gtex, gvp) + tuple((wg[p._rn_name] if p._rn_name in wg else zero(p)) if n else None
                                                     for (p, _), n in zip(ctx.versions, need[5:]))


class TextureRenderer(_Renderer):
    """The Texture+Normal network as an autograd layer: forward(voxels, texture, view_params) -> (albedo, normal), fp32
    [B,512,512,3] each.  Gradients reach the voxels, the texture vector [B,199] and the pose, and with trainable=True the 186
    parameters (texture decoder included).  model="texture": RenderNet_Texture_Face_Normal under TF variable names (`weights`
    {tf name: array} or None); model="pretrained": the npz-keyed RenderNet_pretrained of face reconstruction, constant as in the
    reference (trainable=True raises)."""

    def __init__(self, weights: Optional[Dict[str, np.ndarray]] = None, precision: str = "exact", model: str = "texture",
                 trainable: bool = False, loss_scale=None, seed: int = 0, device: str = "cuda"):
        if model not in ("texture", "pretrained"):
            raise ValueError(f"model must be 'texture' or 'pretrained', not {model!r}")
        if model == "pretrained" and trainable:
            raise ValueError("model='pretrained' is a constant network (as in the reference): it has no trainable parameters")
        super().__init__()
        self.precision, self.model, self.trainable = precision, model, bool(trainable)
        self._loss_scale, self._device = loss_scale, device
        base = TextureInputGradients(weights, 1, precision, model=model, loss_scale=loss_scale, seed=seed, device=device)
        with torch.no_grad():
            _TextureFn.forward(SimpleNamespace(), _Once(base), None, torch.zeros((1, SIZE, SIZE, SIZE, 1), device=base.store.device),
                               np.zeros((1, 199), np.float32), np.array([[0.0, 0.0, 1.0]], np.float32))
        self._setup(base, self.trainable)

    def _make(self, B):
        return TextureInputGradients(self._base.weight_dict, B, self.precision, model=self.model, loss_scale=self._loss_scale,
                                     device=self._device, store=self.store)

    def forward(self, voxels, texture, view_params):
        B = _check_voxels(voxels)
        _rows(texture, B, 199, "texture")
        _rows(view_params, B, 3, "view_params")
        self._sync_packed()
        params = list(self.params.values())
        return _TextureFn.apply(self, _grad_mode(params, voxels, texture, view_params), voxels, texture, view_params, *params)


# ----------------------------------------------------------------------------------------------- shape decoder
class _ShapeDecoderFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, module, mode, latent, *params):
        from .Reconstruct_RenderNet_Face import decoder_3d_pretrained
        B = latent.shape[0]
        sdg = module._object(B)
        sdg.latent = latent.to(device=sdg.store.device, dtype=torch.float32).reshape(B, -1).contiguous()
        sdg.vox = _record(sdg, mode, lambda: tf.realize(decoder_3d_pretrained(sdg.latent, sdg.weight_dict)))
        vox = sdg.vox.detach()
        ctx.rec = sdg._snapshot() if mode else None
        _release(sdg)
        if mode:
            ctx.module, ctx.B = module, B
            ctx.versions = [(p, p._version) for p in params]
            ctx.save_for_backward(latent, vox)
        return vox

    @staticmethod
    @once_differentiable
    def backward(ctx, dvox):
        latent, _ = ctx.saved_tensors
        _check_versions(ctx)
        need = ctx.needs_input_grad
        want_dlatent, want_w = need[2], any(need[3:])
        sdg = ctx.module._object(ctx.B)
        sdg._restore(_take_recording(ctx))
        try:
            dz = sdg.backward(dvox, on_device=True, want_weight_grads=want_w, want_dlatent=want_dlatent)
            wg = sdg.weight_grads if want_w else {}
        finally:
            _release(sdg)
        gz = dz.to(device=latent.device, dtype=latent.dtype).reshape(latent.shape) if want_dlatent else None
        return (None, None, gz) + tuple(wg[p._rn_name] if n else None for (p, _), n in zip(ctx.versions, need[3:]))


def _check_decoder_weights(weight_dict_decoder) -> None:
    """The decoder's 12 npz-keyed arrays, with the shapes decoder_3d_pretrained builds from them (checked on the host)."""
    from .Reconstruct_RenderNet_Face import DECODER_VARIABLES
    if not hasattr(weight_dict_decoder, "keys") or not hasattr(weight_dict_decoder, "__getitem__"):
        raise TypeError(f"weight_dict_decoder must be a mapping of npz keys to arrays, not {type(weight_dict_decoder).__name__}")
    missing = [k for _, k, _ in DECODER_VARIABLES if k not in weight_dict_decoder]
    if missing:
        raise KeyError(f"weight_dict_decoder lacks {missing}")
    for _, k, shape in DECODER_VARIABLES:
        got = tuple(np.shape(weight_dict_decoder[k]))
        if shape is not None and got != shape:
            raise ValueError(f"weight_dict_decoder[{k!r}] has shape {got}, not {shape}")


class ShapeDecoder(_Renderer):
    """The face-reconstruction shape decoder (Reconstruct_RenderNet_Face.decoder_3d_pretrained) as an autograd layer:
    forward(latent [B,200]) -> voxels [B,64,64,64,1] fp32 on the device; dL/dlatent from ShapeDecoderGradients on the device.
    `weight_dict_decoder`: the decoder's 12 npz-keyed arrays (g_zP_g_gc1_weights, ..., g_conv5_biases).  trainable=False: they
    are constants, as in the reference's reconstruction.  trainable=True (fine-tuning, decoder_3d_pretrained(trainable=True)):
    they are the 12 Parameters `params.<tf name>`, and the walk that gives dL/dlatent also gives their gradients.
    decoder_weight_dict() returns the current values under their npz keys."""

    def __init__(self, weight_dict_decoder: Dict[str, np.ndarray], trainable: bool = False, device: str = "cuda"):
        if not isinstance(trainable, (bool, np.bool_)):
            raise TypeError(f"trainable must be a bool, not {type(trainable).__name__}")
        _check_decoder_weights(weight_dict_decoder)
        super().__init__()
        self._device, self.trainable = device, bool(trainable)
        base = ShapeDecoderGradients(weight_dict_decoder, 1, device=device)
        with torch.no_grad():
            _ShapeDecoderFn.forward(SimpleNamespace(), _Once(base), None, torch.zeros((1, 200), device=base.store.device))
        self._setup(base, self.trainable)

    def _make(self, B):
        return ShapeDecoderGradients(self._base.weight_dict, B, device=self._device, store=self.store)

    def decoder_weight_dict(self) -> Dict[str, np.ndarray]:
        """{npz key: fp32 ndarray} of the 12 variables (the TF name with '/' -> '_'): the dictionary ShapeDecoder,
        ShapeDecoderGradients and FaceReconstruction take, so fine-tuned weights can be fed back into the reconstruction."""
        from .Reconstruct_RenderNet_Face import DECODER_VARIABLES
        names = dict((t, k) for t, k, _ in DECODER_VARIABLES)
        return {names[n]: t.detach().cpu().numpy().copy() for n, t in self.store.vars.items() if n in names}

    def forward(self, latent):
        if not isinstance(latent, torch.Tensor) or latent.dim() != 2 or latent.shape[0] < 1 or latent.shape[1] != 200:
            raise ValueError(f"latent must be a [B,200] tensor, not {getattr(latent, 'shape', type(latent))}")
        self._sync_packed()
        params = list(self.params.values())
        return _ShapeDecoderFn.apply(self, _grad_mode(params, latent), latent, *params)


# ----------------------------------------------------------------------------------------------- Phong composite
class _PhongFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, normal, light_dir, albedo, light_col, ambient, opts):
        _, compos, _ = ops.phong_shade(normal, light_dir, albedo=albedo, light_col=light_col, ambient=ambient, want_shade=False,
                                       want_compos=True, want_u8=False, **opts)
        ctx.opts = opts
        ctx.consts = (None if isinstance(light_col, torch.Tensor) else light_col,
                      None if isinstance(ambient, torch.Tensor) else ambient)
        ctx.save_for_backward(normal, light_dir, albedo, *(t for t in (light_col, ambient) if isinstance(t, torch.Tensor)))
        return compos

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        normal, light_dir, albedo, *rest = ctx.saved_tensors
        light_col, ambient = ctx.consts
        if light_col is None:
            light_col = rest.pop(0)
        if ambient is None:
            ambient = rest.pop(0)
        need = ctx.needs_input_grad
        shading = need[3] or need[4]
        out = ops.phong_shade_backward(normal, g, light_dir, albedo=albedo, light_col=light_col, ambient=ambient,
                                       want_light_grad=need[1], want_shading_grad=shading, **ctx.opts)
        d_normal, d_albedo, d_light = out[:3]

        def per_input(d, t):          # a [1,...] row (or a 0-d ambient) gets the gradient summed over the batch
            d = d.sum(0, keepdim=True) if t.shape[:1] != d.shape[:1] else d
            return d.reshape(t.shape).to(device=t.device, dtype=t.dtype)
        d_col = per_input(out[3], light_col) if need[3] else None
        d_amb = per_input(out[4], ambient) if need[4] else None
        if need[1]:
            d_light = per_input(d_light, light_dir)
        return (d_normal if need[0] else None), (d_light if need[1] else None), (d_albedo if need[2] else None), d_col, d_amb, None


def phong_shade(normal, light_dir, albedo=None, composite: str = "tf", light_col=(1.0, 1.0, 1.0), ambient: float = 0.0,
                k_diffuse: float = 1.0, background_white: bool = True, with_mask: bool = True):
    """Differentiable Phong composite: compos = albedo * shade (albedo None: shade) of a normal map [B,H,W,3] fp32 CUDA tensor;
    the forward is ops.phong_shade's image bit for bit, the backward rn_phong_shade_backward (rn_phong_shade_backward_params when
    the light colour or the ambient term needs a gradient).  composite "tf" (face reconstruction) or "numpy" (the demo's).
    light_dir: a [1,3] (its gradient summed over the batch) or [B,3] tensor.  light_col: a [1|B,3] floating-point tensor (or a
    constant triple), ambient: a float or a [1|B] (or 0-d) floating-point tensor; either tensor may require grad, and a single
    row gets its gradient summed over the batch.  k_diffuse is a constant: the composites see only k_diffuse * light_col, so its
    gradient would duplicate the colour's.  Gradients reach normal, albedo, light_dir, light_col and ambient."""
    if len(getattr(normal, "shape", ())) != 4 or normal.shape[3] != 3:
        raise ValueError(f"phong_shade: normal map must be [B,H,W,3], not {tuple(getattr(normal, 'shape', ()))}")
    B = int(normal.shape[0])
    if not isinstance(light_dir, torch.Tensor):
        light_dir = torch.as_tensor(np.asarray(light_dir, np.float32))
    if light_dir.dim() != 2 or light_dir.shape[1] != 3 or light_dir.shape[0] not in (1, B):
        raise ValueError(f"phong_shade: light_dir must be [1,3] or [{B},3], not {tuple(light_dir.shape)}")
    if isinstance(light_col, torch.Tensor):
        if light_col.dim() != 2 or light_col.shape[1] != 3 or light_col.shape[0] not in (1, B):
            raise ValueError(f"phong_shade: light_col must be [1,3] or [{B},3], not {tuple(light_col.shape)}")
    if isinstance(ambient, torch.Tensor):
        if ambient.dim() > 1 or ambient.numel() not in (1, B):
            raise ValueError(f"phong_shade: ambient must be a float or [1] or [{B}], not {tuple(ambient.shape)}")
    else:
        ambient = float(ambient)
    for name, t in (("light_col", light_col), ("ambient", ambient)):
        if isinstance(t, torch.Tensor):
            if not t.dtype.is_floating_point:
                raise TypeError(f"phong_shade: {name} must be a floating-point tensor, not {t.dtype}")
            if t.is_cuda and t.device != normal.device:
                raise ValueError(f"phong_shade: {name} is on {t.device}, the normal map on {normal.device}")
    if composite not in ops.PHONG_COMPOSITES:
        raise ValueError(f"composite must be one of {sorted(ops.PHONG_COMPOSITES)}, not {composite!r}")
    for name, t in (("normal", normal), ("albedo", albedo)):
        if t is not None and (not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != torch.float32):
            raise TypeError(f"phong_shade: {name} must be a float32 CUDA tensor")
    if albedo is not None and tuple(albedo.shape) != tuple(normal.shape):
        raise ValueError(f"phong_shade: albedo {tuple(albedo.shape)} and normal map {tuple(normal.shape)} differ in shape")
    opts = dict(k_diffuse=float(k_diffuse), composite=composite, background_white=bool(background_white),
                with_mask=bool(with_mask))
    return _PhongFn.apply(normal, light_dir, albedo, light_col, ambient, opts)
