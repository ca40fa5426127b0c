"""Backward pass of the forward rendering path with respect to its INPUTS (SURVEY §8 f-4, first stage).

This is what the reference's inverse rendering differentiates (Reconstruct_RenderNet_Face.py:383-412: `tf.gradients` of an
image loss w.r.t. the latent shape / texture / pose, through the frozen RenderNet and through the trilinear weights of
tools/resampling_voxel_grid.py:465-485).  With `want_weight_grads` the same walk also produces dL/d(every variable) -- filters,
biases, PReLU slopes -- which rendernet_b200/training.py turns into the training step of RenderNet_Shader.py:154-167.

How it works: the model function (RenderNet_Shader.RenderNet) is run once with a TAPE attached to the variable store; every
realised layer appends (kind, input, filter, activation, residual, output).  `backward()` walks the tape in reverse:

  * activations: PReLU / sigmoid derivatives from the STORED post-activation tensors (rn_prelu_backward_16, rn_sigmoid_backward);
  * data gradient of a stride-1 SAME convolution = a stride-1 convolution of the output gradient with the spatially mirrored,
    channel-transposed filter -> the SAME wgmma implicit-GEMM kernel as the forward pass (rn_conv_igemm) with a mirrored
    tap list; 3^3 convs through the depth-folded (banded) form; the residual adds of the forward graph become the fused
    `residual` input of the gradient convolution (gradient accumulation at a fan-out costs no extra pass);
  * data gradient of a stride-1 transposed conv = a forward SAME conv with the very same filter array;
  * data gradient of a stride-2 transposed conv (k = 4) = space-to-depth of the output gradient ([B,2H,2W,C] -> [B,H,W,4C])
    followed by ONE 3x3 convolution whose filter holds the 16 taps at their (phase, offset) slots (the transpose of the
    forward "merged-phase" trick);
  * e_conv2 / e_conv1 (thin, strided, 1.7 % of the MACs): CUDA-core gather kernels (rn_conv3d_backward_data_direct);
  * resampler: scatter-add to the voxel grid and the 3x4 matrix gradient (rn_resample_backward_f32); the 12 matrix entries
    are mapped to (azimuth, elevation, scale) on the host by differentiating the reference's matrix construction
    (tools/resampling_voxel_grid.py:515-602) -- a 3 -> 12 map, float64.

The Texture+Normal network (TextureInputGradients) walks the same tape the same way.  Its two heads both read enc5_skip, a
fan-out like the residual adds.  Its input chain is two resamplings (geometry C = 1, decoded texture C = 4) concatenated into
e_conv1: rn_resample5_backward_f32 splits dL/d(concat) into dL/dvoxels, dL/d(texture volume) and dL/dM^-1, and dL/d(texture
volume) continues, in fp32, through the texture decoder (rn_prelu_backward_f32, rn_conv3d_small, rn_fully_connected_backward_data)
to dL/d(texture vector).

The face-reconstruction shape decoder (ShapeDecoderGradients, Reconstruct_RenderNet_Face.decoder_3d_pretrained) is walked the same
way, in fp32: ELU / sigmoid derivatives from the stored outputs (rn_act_backward_f32), each conv3d_transpose's data gradient a
conv3d on the same filter array (rn_conv3d_f32), the FC's rn_fully_connected_backward_data, down to dL/dlatent.  The voxel grid is
the seam between it and TextureInputGradients; dL/dvoxels can stay on the device between the two.  With want_weight_grads the same
walk also gives the decoder's 12 parameter gradients (rn_conv3d_f32_weight_grad, rn_fully_connected_param_grad): fine-tuning.

Gradients travel in the activations' 16-bit format (fp16, or fp16 hi/lo pairs in the exact mode) with a loss scale to keep
them inside fp16's range; they are un-scaled when they leave the tensor-core part (fp32 from there on).  By default the scale
is chosen per backward call (choose_loss_scale): the power of two that brings the largest |g * s(1 - s)| at the output heads
to LOSS_SCALE_TARGET.  A power of two keeps every step of the walk exact under the scaling, so the result does not depend on
the magnitude of dL/d(output) as long as nothing leaves fp16's range (DESIGN §4).
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import numpy as np
import torch

from . import ops
from . import tfcompat as tf
from .RenderNet_Shader import RenderNet
from .engine import pose_to_matrix
from .resampling_voxel_grid import ConcatResampledGrid, CroppedGrid, ResampledGrid


def _key(t) -> int:
    """Identity of an activation on the tape: its storage address (reshapes / views share it)."""
    return t.data_ptr()


def pose_matrix_jacobian_vjp(view_params: np.ndarray, dminv: np.ndarray, size: int = 64, new_size: int = 128) -> np.ndarray:
    """dL/d(view_params) [B,3] from dL/d(Minv[:, :3, :]) [B,3,4]: differentiates M = T(+new/2).S.R.T(-size/2), R = RotZ(el).RotY(az-pi/2)
    (tools/resampling_voxel_grid.py:515-602) and the matrix inverse, in float64 on the host (a 3 -> 12 map per item).  Runs
    under torch.enable_grad(), so it also works inside a torch.autograd.Function's backward (rendernet_b200.nn)."""
    with torch.enable_grad():
        return _pose_matrix_jacobian_vjp(view_params, dminv, size, new_size)


def _pose_matrix_jacobian_vjp(view_params, dminv, size, new_size):
    vp = torch.tensor(np.asarray(view_params, np.float64), requires_grad=True)
    B = vp.shape[0]
    az = vp[:, 0] - math.pi * 0.5
    el, sc = vp[:, 1], vp[:, 2]
    ca, sa, ce, se = torch.cos(az), torch.sin(az), torch.cos(el), torch.sin(el)
    z, o = torch.zeros_like(ca), torch.ones_like(ca)
    rot_y = torch.stack([torch.stack([ca, z, -sa, z], 1), torch.stack([z, o, z, z], 1), torch.stack([sa, z, ca, z], 1),
                         torch.stack([z, z, z, o], 1)], 1)
    rot_z = torch.stack([torch.stack([ce, se, z, z], 1), torch.stack([-se, ce, z, z], 1), torch.stack([z, z, o, z], 1),
                         torch.stack([z, z, z, o], 1)], 1)
    R = rot_z @ rot_y
    S = torch.stack([torch.stack([sc, z, z, z], 1), torch.stack([z, sc, z, z], 1), torch.stack([z, z, sc, z], 1),
                     torch.stack([z, z, z, o], 1)], 1)
    T = torch.eye(4, dtype=torch.float64).repeat(B, 1, 1).clone()
    T[:, :3, 3] = -size * 0.5
    Tn = torch.eye(4, dtype=torch.float64).repeat(B, 1, 1).clone()
    Tn[:, :3, 3] = new_size * 0.5
    minv = torch.linalg.inv(Tn @ S @ R @ T)[:, :3, :]
    (minv * torch.as_tensor(np.asarray(dminv, np.float64))).sum().backward()
    return vp.grad.numpy()


# Where the adaptive loss scale puts the largest 16-bit gradient of the output heads.  On its way into the network the largest
# gradient grows by up to 21x (the training walk's e_conv2 / e_conv3, dropout 0.75; 5.4x without dropout; measured with
# scripts/grad_range.py, DESIGN §4): 2^9 keeps the largest interior gradient 6x below fp16's largest value, 65504.
LOSS_SCALE_TARGET = 2.0 ** 9
# An output gradient that still overflows is walked again at a 16x lower scale, at most this many times.
OVERFLOW_RETRIES = 3


def choose_loss_scale(amax: float, target: float = LOSS_SCALE_TARGET) -> float:
    """The loss scale 2^floor(log2(target / amax)) for a backward walk whose largest scaled output-head gradient |g s (1 - s)|
    is `amax`: scale * amax lies in (target / 2, target].  A power of two, within [2^-126, 2^126] (scale and 1 / scale are
    normal fp32 numbers); amax = 0 (nothing to scale) gives 1.  A non-finite amax raises FloatingPointError."""
    amax, target = float(amax), float(target)
    if not (math.isfinite(target) and target > 0.0):
        raise ValueError(f"the loss-scale target must be a positive finite number, not {target}")
    if not math.isfinite(amax):
        raise FloatingPointError(f"the output gradient is not finite (max |g s(1-s)| = {amax})")
    if amax <= 0.0:
        return 1.0
    e = math.floor(math.log2(target) - math.log2(amax))
    while math.ldexp(amax, e) > target:            # log2 is rounded: settle the floor exactly
        e -= 1
    while math.ldexp(amax, e + 1) <= target:
        e += 1
    return math.ldexp(1.0, max(-126, min(126, e)))


def _loss_scale_mode(loss_scale) -> Optional[float]:
    """None or "auto": the scale is chosen per backward call (returns None); a number: that fixed scale."""
    if loss_scale is None or (isinstance(loss_scale, str) and loss_scale == "auto"):
        return None
    v = float(loss_scale)
    if not (math.isfinite(v) and v > 0.0):
        raise ValueError(f"loss_scale must be None, 'auto' or a positive finite number, not {loss_scale!r}")
    return v


def _all_finite(tensors) -> bool:
    ts = [t for t in tensors if t is not None]
    return not ts or bool(torch.stack([torch.isfinite(t).all() for t in ts]).all().item())


class _InputGradients:
    """What the Shader and the Texture+Normal input gradients share: the variable store, the per-layer data-gradient filters
    and the reverse walk over the tape (`_reverse_walk`).  A subclass records the tape in `forward` and differentiates, in
    `_input_chain`, the fused resample + e_conv1 record that starts its network."""

    # the attributes a recording consists of (_snapshot / _restore)
    _RECORDING = ("tape",)

    def __init__(self, weights: Optional[Dict[str, np.ndarray]], batch: int, precision: str, size: int, new_size: int,
                 loss_scale, seed: int, device: str, store: Optional[tf.VariableStore] = None):
        if not torch.cuda.is_available():
            raise RuntimeError(f"{type(self).__name__} needs a CUDA device (no CPU fallback)")
        self.B, self.size, self.new_size = batch, size, new_size
        self.loss_scale = _loss_scale_mode(loss_scale)     # None: chosen per backward call, with headroom target scale_target
        self.scale_target = LOSS_SCALE_TARGET
        self.overflow_retries = OVERFLOW_RETRIES
        self.last_loss_scale = None                        # the scale the last walk used
        self.device = torch.device(device)
        if store is not None:                              # shared with gradient objects of other batch sizes: weights and
            if store.precision != precision:               # packed filters exist once
                raise ValueError(f"the shared store computes in {store.precision!r}, not {precision!r}")
            self.store = store
        else:
            self.store = tf.VariableStore(precision=precision, device=str(self.device) if self.device.index is not None else "cuda",
                                          seed=seed)
        if weights is not None:
            with tf.use_store(self.store):
                tf.load_weight_dict(weights)
        self._dgrad_cache: Dict[object, object] = {}
        self.tape = None
        self.last_dgrid = None
        self._fc_dx = False          # weight-gradient walk: also carry dL/d(texture vector) through the decoder's FC

    def _snapshot(self) -> Dict[str, object]:
        """What `backward` reads from the object: the tape, the inputs and the outputs of the last forward.  Holding it keeps
        that recording alive across later forwards (one recording per torch.autograd node, rendernet_b200.nn)."""
        return {k: getattr(self, k, None) for k in self._RECORDING}

    def _restore(self, rec: Dict[str, object]):
        """Make a recording taken by _snapshot the object's current one again."""
        for k, v in rec.items():
            setattr(self, k, v)

    # ------------------------------------------------------------------------------------------- packed gradient filters
    def _zeros(self, n):
        z = self._dgrad_cache.get(("zeros", n))
        if z is None:
            z = torch.zeros(n, device=self.store.device, dtype=torch.float32)
            self._dgrad_cache[("zeros", n)] = z
        return z

    def _dgrad_layer(self, rec):
        """Kernel-ready filter of the data-gradient convolution of one recorded layer (cached per weight)."""
        w, kind, stride, fmt = rec["w"], rec["kind"], rec["stride"], self.store.fmt
        key = (w._rn_name, kind, stride, fmt)
        L = self._dgrad_cache.get(key)
        if L is not None:
            return L
        dev = self.store.device
        wt = w.to(dev)
        if kind == "conv2d":                       # [kh,kw,Ci,Co] -> mirrored, channel roles swapped: [kh,kw,Co,Ci]
            k = int(w.shape[0])
            wd = torch.flip(wt, dims=(0, 1)).permute(0, 1, 3, 2).contiguous()
            L = ops.pack_conv("conv2d", wd, None, None, device=dev, fmt=fmt, winograd=False, exponent=True)
            pb = (k - 1) // 2
            L.taps = [(kx - (k - 1 - pb), ky - (k - 1 - pb)) for ky in range(k) for kx in range(k)]   # offset of mirrored tap
        elif kind == "conv3d":                     # 3^3, stride 1: depth-folded gradient conv
            wd = torch.flip(wt, dims=(0, 1, 2)).permute(0, 1, 2, 4, 3).contiguous()
            L = ops.BandedConv3d(wd, None, device=dev, sz=1, fmt=fmt, exponent=True)
        elif kind == "conv2d_transpose" and stride == 1:
            # y[o] = sum_k x[o - k + pb] w[k][co][ci]  =>  dx[i] = sum_k g[i + k - pb] w[k][co][ci]: a forward SAME conv whose TF filter
            # [kh,kw,Cin'=Co,Cout'=Ci] IS the transposed-conv filter array; Co is zero padded to a multiple of 16 (e_conv11: 3)
            co = int(w.shape[2])
            cp = ops.round_up(co, 16)
            wd = torch.zeros((w.shape[0], w.shape[1], cp, w.shape[3]), device=dev, dtype=torch.float32)
            wd[:, :, :co] = wt
            L = ops.pack_conv("conv2d", wd, None, None, device=dev, fmt=fmt, winograd=False, exponent=True)
            L.taps = None
        elif kind == "conv2d_transpose" and stride == 2:
            # o = 2i + k - 1.  With g2[i,j,(ay,ax,co)] = g[2i+ay, 2j+ax, co]:  dx[i] = sum_{dy,dx in -1..1} g2[i+dy, j+dx] . Wd[dy+1][dx+1]
            # where Wd[dy+1][dx+1][(ay,ax,co)][ci] = w[2dy+ay+1][2dx+ax+1][co][ci] when both indices lie in [0,4), else 0
            assert tuple(w.shape[:2]) == (4, 4)
            co, ci = int(w.shape[2]), int(w.shape[3])
            wd = torch.zeros((3, 3, 2, 2, co, ci), device=dev, dtype=torch.float32)
            for dy in (-1, 0, 1):
                for ay in (0, 1):
                    ky = 2 * dy + ay + 1
                    if not 0 <= ky < 4:
                        continue
                    for dx in (-1, 0, 1):
                        for ax in (0, 1):
                            kx = 2 * dx + ax + 1
                            if 0 <= kx < 4:
                                wd[dy + 1, dx + 1, ay, ax] = wt[ky, kx]
            L = ops.pack_conv("conv2d", wd.reshape(3, 3, 4 * co, ci), None, None, device=dev, fmt=fmt, winograd=False, exponent=True)
            L.taps = None
        else:
            raise NotImplementedError(f"no data-gradient path for {kind} stride {stride}")
        self._dgrad_cache[key] = L
        return L

    @staticmethod
    def _space_to_depth(g):
        """[B,2H,2W,C] -> [B,H,W,(ay,ax,C)] (pure data movement; hi/lo planes alike)."""
        t = g.planes if isinstance(g, ops.Split16) else g
        lead = t.shape[:-3]
        H2, W2, Cc = t.shape[-3:]
        t = t.reshape(*lead, H2 // 2, 2, W2 // 2, 2, Cc).permute(*range(len(lead)), len(lead), len(lead) + 2, len(lead) + 1,
                                                                  len(lead) + 3, len(lead) + 4)
        t = t.reshape(*lead, H2 // 2, W2 // 2, 4 * Cc).contiguous()
        return ops.Split16(t) if isinstance(g, ops.Split16) else t

    def _has_negative_slope(self, alpha, a_dev) -> bool:
        key = ("alpha<0", alpha._rn_name)
        v = self._dgrad_cache.get(key)
        if v is None:
            v = bool((a_dev < 0).any().item())
            self._dgrad_cache[key] = v
        return v

    def _alpha(self, alpha, n):
        if isinstance(alpha, str):                 # tf.nn.relu branch
            return self._zeros(n)
        key = ("alpha", alpha._rn_name)
        a = self._dgrad_cache.get(key)
        if a is None:
            a = alpha.to(device=self.store.device, dtype=torch.float32).reshape(-1).contiguous()
            self._dgrad_cache[key] = a
        return a

    def _w32(self, w):
        """fp32 device copy of a recorded filter (cached per variable)."""
        key = ("w32", w._rn_name)
        d = self._dgrad_cache.get(key)
        if d is None:
            d = w.to(device=self.store.device, dtype=torch.float32).contiguous()
            self._dgrad_cache[key] = d
        return d

    # ------------------------------------------------------------------------------------------- reverse walk
    def _choose_scale(self, grads) -> float:
        """The fixed loss scale, or choose_loss_scale of max |g s (1 - s)| over the sigmoid heads that `grads` reaches."""
        if self.loss_scale is not None:
            return self.loss_scale
        amax = None
        for rec in self.tape:
            y = rec["y"]
            if rec["op"] in ("conv_small", "conv_f32", "fc") or rec.get("act") != "sigmoid" or _key(y) not in grads:
                continue
            g = grads[_key(y)].reshape(tuple(y.shape))
            a = torch.amax(torch.abs(g * y * (1.0 - y)))
            amax = a if amax is None else torch.maximum(amax, a)
        return 1.0 if amax is None else choose_loss_scale(amax.item(), self.scale_target)

    def _walk_checked(self, walk):
        """Run walk(shrink) -> the tensors it returns; shrink multiplies the chosen loss scale.  A non-finite result (an fp16
        overflow inside the walk) raises FloatingPointError with a fixed scale; an adaptive scale is retried 16x lower, at
        most `overflow_retries` times."""
        shrink = 1.0
        for _ in range(self.overflow_retries + 1):
            if _all_finite(walk(shrink)):
                return
            if self.loss_scale is not None:
                break
            shrink /= 16.0
        raise FloatingPointError(f"gradient overflow in the 16-bit backward pass at loss scale {self.last_loss_scale:g}")

    def _reverse_walk(self, grads, want_weight_grads: bool, tensor_core_wgrad: bool, shrink: float = 1.0):
        """Walk the tape backwards from `grads` {_key(output): dL/doutput}.  16-bit layers take and give gradients carrying the
        loss scale (`_choose_scale` times `shrink`, kept in last_loss_scale); the fused input record goes to `_input_chain`; the
        texture decoder's fp32 layers (records "conv_small", "fc"), which come after it in the walk, take and give unscaled fp32
        gradients."""
        fmt = self.store.fmt
        self.last_loss_scale = scale = self._choose_scale(grads) * shrink
        inv = 1.0 / scale
        for rec in reversed(self.tape):
            y = rec["y"]
            g = grads.pop(_key(y), None)
            if g is None:
                continue                                   # no gradient reaches this layer
            if tuple(g.shape) != tuple(y.shape):           # the consumer saw a reshaped view (projection unit: [..,D,C] -> [..,D*C])
                g = g.reshape(tuple(y.shape))
            op = rec["op"]
            if op == "copy":                               # a device copy made on the way into the resampler (_to_cuda_f32)
                k = _key(rec["x"])
                grads[k] = grads[k] + g if k in grads else g
                continue
            if op == "dropout":                            # d(x * mask / keep) = g * mask / keep: the same stateless kernel
                grads[_key(rec["x"])] = ops.dropout(g, rec["keep"], rec["seed"], rec["salt"])
                continue
            if op in ("conv_small", "conv_f32", "fc"):
                self._decoder_step(rec, g, grads, want_weight_grads)
                continue
            act = rec["act"]
            if act == "sigmoid":
                co = int(y.shape[-1])
                g = ops.sigmoid_backward(g, y, ops.round_up(co, 16), scale, fmt)
            elif act == "prelu":
                alpha = rec["alpha"]
                a_dev = self._alpha(alpha, int(y.shape[-1]))
                sign_src = y                    # the stored output tells the side of the kink as long as every slope is >= 0
                if not isinstance(alpha, str) and (want_weight_grads or self._has_negative_slope(alpha, a_dev)):
                    # Re-run the layer without its PReLU to get the pre-activation z: dL/dalpha = sum_{z<0} g*z needs it (alpha
                    # starts at 0), and so does the derivative itself once a slope is negative (y = alpha*z > 0 for z < 0;
                    # Adam's first step already makes half of the slopes negative).
                    sign_src = rec["rerun"]()
                    if want_weight_grads:
                        self.weight_grads[alpha._rn_name] = ops.prelu_alpha_grad(g, sign_src, inv)
                g = ops.prelu_backward(g, sign_src, a_dev)
            if want_weight_grads:
                self._weight_grads_of(rec, g, inv, tensor_core_wgrad)
            if op in ("resample_conv1", "resample5_conv1"):   # e_conv1 fused with the resampler(s) in the forward pass
                self._input_chain(rec, g, grads)
                continue
            res = rec.get("residual")
            if res is not None:                            # y = act(conv(x) + res): the gradient flows to res unchanged
                k = _key(res)
                grads[k] = ops.bias_act(g, None, None, None, residual=grads[k]) if k in grads else g
            x = rec["x"]
            acc = grads.pop(_key(x), None)                 # gradient already collected for x (fan-out): fused as `residual`
            grads[_key(x)] = self._data_grad_of(rec, g, acc)

    def _input_chain(self, rec, g, grads):
        raise NotImplementedError

    def _decoder_step(self, rec, g, grads, want_weight_grads: bool = False):
        """One layer of the texture decoder or the shape decoder (fp32, unscaled).  PReLU: once a layer has a negative slope the
        side of the kink comes from the pre-activation (re-run without the activation): pretrained decoder slopes may be negative.
        ELU and sigmoid (shape decoder): TF-1's EluGrad / SigmoidGrad from the stored output (rn_act_backward_f32).  The data
        gradients need no kernel of their own: TF defines conv3d_transpose as the input gradient of conv3d with the same filter
        array and padding, so the gradient of a conv3d is the transposed conv on that array, the gradient of a conv3d_transpose
        is the forward conv on it (same stride) -- rn_conv3d_small for the thin layers, rn_conv3d_f32 for the wide ones -- and
        the gradient of fully_connected is rn_fully_connected_backward_data.

        want_weight_grads (Texture+Normal training, PReLU layers): the pre-activation (kept on the tape, or re-run) gives
        dL/dz, db and dalpha in one pass (rn_prelu_grad_f32; the FC's rn_fully_connected_param_grad, which also gives dW), the
        filter gradient comes from the thin correlation kernel (fp32 operands).  The gradients reaching the decoder are unscaled
        fp32, so no 1/scale is applied.  The FC's data gradient -- dL/d(texture vector), an input of the network -- is skipped
        unless `_fc_dx` asks for it.  Shape decoder (fine-tuning): a conv_f32 layer's dL/dz from the stored output as above, dW and
        db from rn_conv3d_f32_weight_grad, the data gradient as without weight gradients; the FC without activation gives dW and db
        from rn_fully_connected_param_grad with gz = gy."""
        act = rec["act"]
        if want_weight_grads:
            self._decoder_weight_step(rec, g, grads, want_dx=self._fc_dx)
            return
        if act == "prelu":
            alpha = rec["alpha"]
            a_dev = self._alpha(alpha, int(rec["y"].shape[-1]))
            # with every slope >= 0 the output's sign is the pre-activation's (z <= 0 -> y = alpha z <= 0), as in the trunk
            neg = not isinstance(alpha, str) and self._has_negative_slope(alpha, a_dev)
            g = ops.prelu_backward_f32(g, rec["rerun"]() if neg else rec["y"], a_dev)
        elif act in ("elu", "sigmoid"):
            g = ops.act_backward_f32(g, rec["y"], act)
        elif act is not None:
            raise NotImplementedError(f"no backward for a fused {act} on a decoder layer")
        w32 = self._w32(rec["w"])
        if rec["op"] == "fc":
            dx = ops.fully_connected_backward_data(g, w32)
        elif rec["op"] == "conv_f32":
            dx = ops.conv3d_f32(g, w32, None, int(rec["stride"]), not rec["transposed"])
        else:
            dx = ops.conv3d_small(g, w32, None, None, int(rec["stride"]), not rec["transposed"], want32=True)
        k = _key(rec["x"])
        grads[k] = grads[k] + dx if k in grads else dx

    def _decoder_weight_step(self, rec, g, grads, want_dx: bool = False):
        alpha, w, b, x = rec["alpha"], rec["w"], rec["b"], rec["x"]
        if rec["op"] == "conv_f32" and rec["act"] in ("elu", "sigmoid", None):
            self._f32_conv_weight_step(rec, g, grads)
            return
        if rec["op"] == "fc" and rec["act"] is None:
            self._fc_weight_step(rec, g, grads, want_dx)
            return
        if rec["act"] != "prelu" or isinstance(alpha, str) or b is None or rec["op"] not in ("fc", "conv_small"):
            raise NotImplementedError(f"no weight gradients for a decoder {rec['op']} record with act {rec['act']!r}")
        wg = self.weight_grads
        z = rec["rerun"]()
        a_dev = self._alpha(alpha, int(rec["y"].shape[-1]))
        if rec["op"] == "fc":
            gz, wg[w._rn_name], wg[b._rn_name], wg[alpha._rn_name] = ops.fully_connected_param_grad(x, g, z, a_dev,
                                                                                                     want_gz=want_dx)
            if want_dx:                        # dL/d(texture vector) as well (input and weight gradients in one walk)
                dx = ops.fully_connected_backward_data(gz, self._w32(w))
                k = _key(x)
                grads[k] = grads[k] + dx if k in grads else dx
            return
        g, wg[b._rn_name], wg[alpha._rn_name] = ops.prelu_grad_f32(g, z, a_dev)
        s = int(rec["stride"])
        ks = tuple(int(v) for v in w.shape[:3])
        if rec["transposed"]:                  # filter [k,k,k,co,ci]; o = i*s + k - pb: P = the layer's input, Q = dL/dz
            co, ci = int(w.shape[3]), int(w.shape[4])
            pad = tuple(ops.same_pad_before(int(x.shape[1 + i]) * s, ks[i], s) for i in range(3))
            d = ops.conv_weight_grad_direct(x, g, ks, (s, s, s), pad, Ca=ci, Cb=co)                  # [k,k,k,ci,co]
        else:                                  # filter [k,k,k,ci,co]: P = dL/dz, Q = the layer's input
            ci, co = int(w.shape[3]), int(w.shape[4])
            pad = tuple(ops.same_pad_before(int(x.shape[1 + i]), ks[i], s) for i in range(3))
            d = ops.conv_weight_grad_direct(g, x, ks, (s, s, s), pad, Ca=co, Cb=ci)                  # [k,k,k,co,ci]
        wg[w._rn_name] = d.permute(0, 1, 2, 4, 3).contiguous()
        dx = ops.conv3d_small(g, self._w32(w), None, None, s, not rec["transposed"], want32=True)
        k = _key(x)
        grads[k] = grads[k] + dx if k in grads else dx

    def _f32_conv_weight_step(self, rec, g, grads):
        """A shape-decoder conv (rn_conv3d_f32, + bias, ELU / sigmoid / none): dL/dz from the stored output, dW and db in one
        launch pair, then the data gradient exactly as the walk without weight gradients computes it."""
        w, b, x, s = rec["w"], rec["b"], rec["x"], int(rec["stride"])
        gz = ops.act_backward_f32(g, rec["y"], rec["act"]) if rec["act"] is not None else g
        dw, db = ops.conv3d_f32_weight_grad(x, gz, s, rec["transposed"])
        self.weight_grads[w._rn_name] = dw
        if b is not None:
            self.weight_grads[b._rn_name] = db
        dx = ops.conv3d_f32(gz, self._w32(w), None, s, not rec["transposed"])
        k = _key(x)
        grads[k] = grads[k] + dx if k in grads else dx

    def _fc_weight_step(self, rec, g, grads, want_dx: bool):
        """An FC without activation (the shape decoder's g_gc1): dW = x^T g and db = sum_b g, and dL/dx = g W^T only if
        want_dx."""
        w, b, x = rec["w"], rec["b"], rec["x"]
        _, dw, db, _ = ops.fully_connected_param_grad(x, g, None, None)
        self.weight_grads[w._rn_name] = dw
        if b is not None:
            self.weight_grads[b._rn_name] = db
        if want_dx:
            dx = ops.fully_connected_backward_data(g, self._w32(w))
            k = _key(x)
            grads[k] = grads[k] + dx if k in grads else dx

    def _data_grad_of(self, rec, g, acc=None):
        """dL/dx of one recorded convolution layer from g = dL/d(its pre-activation) (16-bit, carrying the loss scale); `acc`, a
        gradient already collected for x at a fan-out, is added to the result (fused as the kernels' `residual` input)."""
        x, kind, stride = rec["x"], rec["kind"], rec["stride"]
        if kind == "conv3d" and stride == 2:           # e_conv2: thin, z-strided -> CUDA cores
            w32 = rec["w"].to(self.store.device).float().contiguous()
            gx = ops.conv3d_backward_data_direct(g, w32, tuple(x.shape), (1, 1, 2))
            return gx if acc is None else ops.bias_act(gx, None, None, None, residual=acc)
        L = self._dgrad_layer(rec)
        if kind == "conv3d":
            return ops.conv3d_banded(g, L, residual=acc)
        if kind == "conv2d":
            k = int(rec["w"].shape[0])
            if k % 2 == 1:
                return ops.conv2d(g, L, residual=acc)
            return ops.conv2d_taps(g, L.w, L.bias, L.taps, L.cout, L.cout_pad, self.store.fmt, residual=acc,
                                   ny=k if L.cin % 64 == 0 else 0, w_unscale=L.w_unscale)
        if stride == 1:                                # transposed conv, stride 1
            return ops.conv2d(g, L, residual=acc)
        return ops.conv2d(self._space_to_depth(g), L, residual=acc)      # transposed conv, stride 2

    # ------------------------------------------------------------------------------------------- weight gradients
    def _weight_grads_of(self, rec, g, inv: float, tensor_core: bool):
        """dL/dW and dL/db of one recorded layer from g = dL/d(pre-activation) (16-bit, carrying the loss scale)."""
        w, b = rec["w"], rec["b"]
        wg = self.weight_grads
        cout = int(w.shape[2]) if rec.get("kind") == "conv2d_transpose" else int(w.shape[-1])
        if b is not None:
            wg[b._rn_name] = ops.bias_grad(g)[:cout] * inv          # g may carry zero-padded channels (e_conv11: 3 of 16)
        if rec["op"] in ("resample_conv1", "resample5_conv1"):
            # e_conv1 read the resampled grid straight out of the fused kernel: materialise it once for the correlation (the
            # standalone resampler is bit-identical to the fused one); Texture+Normal: geometry and decoded texture, concatenated
            # (a patch record: the same grid's window alone, SAME-padded at the patch's borders)
            grid = rec["grid"]
            win = {} if rec.get("window") is None else dict(window=rec["window"])
            if rec["op"] == "resample_conv1":
                q = ops.resample(grid.voxel, grid.minv, self.new_size, True, **win)
            else:
                q = ops.concat_channels(ops.resample(grid.geom.voxel, grid.minv, self.new_size, True, **win),
                                        ops.resample(grid.tex.voxel, grid.minv, self.new_size, True, **win))
            st = tuple(int(v) for v in rec["stride"])
            ks = tuple(int(v) for v in w.shape[:3])
            pad = tuple(ops.same_pad_before(int(q.shape[1 + i]), ks[i], st[i]) for i in range(3))
            d = ops.conv_weight_grad_direct(g, q, ks, st, pad, Ca=cout, Cb=int(w.shape[3]), scale=inv)      # [k,k,k,co,ci]
            wg[w._rn_name] = d.permute(0, 1, 2, 4, 3).contiguous()
            return
        x, kind, stride = rec["x"], rec["kind"], rec["stride"]
        if kind == "conv2d":
            kh, kw, ci, co = (int(v) for v in w.shape)
            if tensor_core and ci % 128 == 0 and co % 128 == 0 and kh * kw <= 16:
                wg[w._rn_name] = ops.conv2d_weight_grad(x, g, kh, kw) * inv
            else:
                pad = (ops.same_pad_before(int(x.shape[1]), kh, 1), ops.same_pad_before(int(x.shape[2]), kw, 1))
                d = ops.conv_weight_grad_direct(g, x, (kh, kw), (1, 1), pad, Ca=co, Cb=ci, scale=inv)           # [kh,kw,co,ci]
                wg[w._rn_name] = d.permute(0, 1, 3, 2).contiguous()
        elif kind == "conv3d":
            k1, k2, k3, ci, co = (int(v) for v in w.shape)
            st = (1, 1, int(stride))                                   # stride 2 = the z-strided e_conv2 ([1,1,2])
            D = int(x.shape[3])
            if (tensor_core and st == (1, 1, 1) and (k1, k2, k3) == (3, 3, 3) and (D * ci) % 128 == 0 and (D * co) % 128 == 0):
                # depth-folded: a 3x3 conv2d over [B,H,W,D*ci] -> [B,H,W,D*co] whose filter is block-banded; its tensor-core
                # weight gradient holds dW[k1][k2][k3] on the (k3-1)-th block diagonal, summed over the D depth slices
                B_, H, Wd = (int(v) for v in x.shape[:3])
                full = ops.conv2d_weight_grad(x.reshape(B_, H, Wd, D * ci), g.reshape(B_, H, Wd, D * co), 3, 3)
                full = full.view(3, 3, D, ci, D, co)
                d = torch.stack([torch.diagonal(full, offset=-(k - 1), dim1=2, dim2=4).sum(-1) for k in range(3)], dim=2)
                wg[w._rn_name] = (d * inv).contiguous()                # [3,3,3,ci,co]
            else:
                pad = tuple(ops.same_pad_before(int(x.shape[1 + i]), (k1, k2, k3)[i], st[i]) for i in range(3))
                d = ops.conv_weight_grad_direct(g, x, (k1, k2, k3), st, pad, Ca=co, Cb=ci, scale=inv)           # [k,k,k,co,ci]
                wg[w._rn_name] = d.permute(0, 1, 2, 4, 3).contiguous()
        elif kind == "conv2d_transpose":
            kh, kw, co, ci = (int(v) for v in w.shape)                 # TF transposed-conv filter [kh,kw,Cout,Cin]
            s = int(stride)
            pad = (ops.same_pad_before(int(x.shape[1]) * s, kh, s), ops.same_pad_before(int(x.shape[2]) * s, kw, s))
            d = ops.conv_weight_grad_direct(x, g, (kh, kw), (s, s), pad, Ca=ci, Cb=co, scale=inv)               # [kh,kw,ci,co]
            wg[w._rn_name] = d.permute(0, 1, 3, 2).contiguous()
        else:
            raise NotImplementedError(f"no weight-gradient path for {kind}")


class ShaderInputGradients(_InputGradients):
    """Forward + input-gradient backward of the Shader network for a fixed batch size.

        ig = ShaderInputGradients(weights, batch=1, precision="exact")
        img = ig.forward(voxels, view_params)                 # [B,512,512,3] fp32 on the device (tape recorded)
        dvox, dpose = ig.backward(dL_dimg)                    # [B,64,64,64,1], [B,3] fp32 (NumPy)

    `weights`: {tf variable name: array} or None (seeded reference initialisers).  `loss_scale`: None / "auto" chooses it per
    call (choose_loss_scale; an overflow is retried at a lower scale); a number fixes it (an overflow raises
    FloatingPointError)."""

    _RECORDING = ("tape", "vox", "minv", "view_params", "img")

    def __init__(self, weights: Optional[Dict[str, np.ndarray]], batch: int, precision: str = "exact", is_greyscale: bool = False,
                 size: int = 64, new_size: int = 128, loss_scale=None, seed: int = 0, device: str = "cuda",
                 store: Optional[tf.VariableStore] = None):
        super().__init__(weights, batch, precision, size, new_size, loss_scale, seed, device, store)
        self.is_greyscale = is_greyscale
        self.img = None

    # ------------------------------------------------------------------------------------------- forward
    def forward(self, voxels, view_params) -> torch.Tensor:
        """voxels [B,64,64,64,1], view_params [B,3] -> image [B,512,512,3|1] fp32 on the device.  voxels may be a CUDA tensor
        (e.g. a shape fit's occupancy, expanded over the views): it is used in place, without a host round trip."""
        dev = self.store.device
        self.view_params = np.asarray(view_params, np.float32)
        if isinstance(voxels, torch.Tensor) and voxels.is_cuda:
            self.vox = voxels.to(device=dev, dtype=torch.float32).reshape(self.B, self.size, self.size, self.size, 1).contiguous()
        else:
            self.vox = torch.as_tensor(np.asarray(voxels, np.float32)).reshape(self.B, self.size, self.size, self.size, 1).to(dev)
        self.minv = torch.from_numpy(pose_to_matrix(self.view_params, self.size, self.new_size)).to(dev)
        self.tape = []
        self.store.tape = self.tape
        try:
            with tf.use_store(self.store):
                grid = ResampledGrid(self.vox, self.minv, self.new_size, transform=True)
                self.img = RenderNet(grid, is_training=False, is_greyscale=self.is_greyscale)
        finally:
            self.store.tape = None
        return self.img

    # ------------------------------------------------------------------------------------------- backward
    def backward(self, dimg, want_dvox: bool = True, want_dpose: bool = True, want_weight_grads: bool = False,
                 tensor_core_wgrad: bool = True, dvox_on_device: bool = False):
        """dimg: dL/dimg [B,512,512,3|1] (NumPy or tensor).  Returns (dL/dvoxels [B,S,S,S,1] or None, dL/dview_params [B,3] or None).
        dvox_on_device: dL/dvoxels stays a CUDA tensor (for the shape fit's rn_voxel_fit_grad).
        want_weight_grads: also fills `self.weight_grads` {variable name: fp32 device tensor in the variable's TF layout} for EVERY
        variable the forward pass used -- filters (wgmma weight-gradient kernel for the wide stride-1 2-D layers and, depth-folded,
        the 3^3 layers; the strided-correlation kernel rn_conv_weight_grad_direct for the thin / strided / transposed ones), biases
        and PReLU slopes (pre-activation recomputed: alpha starts at 0, tools/layer_util.py:38).  tensor_core_wgrad=False sends
        every filter through the direct kernel (cross-check)."""
        if self.tape is None:
            raise RuntimeError("call forward() first")
        dev = self.store.device
        dimg = torch.as_tensor(np.asarray(dimg, np.float32) if not isinstance(dimg, torch.Tensor) else dimg).to(dev).float()
        if tuple(dimg.shape) != tuple(self.img.shape):
            raise ValueError(f"dimg shape {tuple(dimg.shape)} != image shape {tuple(self.img.shape)}")
        dimg = dimg.contiguous()
        self._need_inputs = want_dvox or want_dpose
        out = {}

        def walk(shrink):
            self._dgrid = None
            self.weight_grads = {}
            self._reverse_walk({_key(self.img): dimg}, want_weight_grads, tensor_core_wgrad, shrink)
            dgrid = self._dgrid
            dvox = dminv = None
            if self._need_inputs:
                if dgrid is None:
                    raise RuntimeError("the tape holds no fused resample + e_conv1 record (is this the Shader path?)")
                dvox, dminv = ops.resample_backward(self.vox, self.minv, dgrid, True, want_dvox, want_dpose)
            out.update(dgrid=dgrid, dvox=dvox, dminv=dminv)
            # every path of the walk reaches e_conv1's filter gradient: an overflow anywhere makes it non-finite
            first = next((g for n, g in self.weight_grads.items() if n.endswith("e_conv1/e_conv1/weights")), None)
            return dvox, dminv, first

        with torch.cuda.device(self.device), tf.use_store(self.store):
            self._walk_checked(walk)
            torch.cuda.synchronize()
        dgrid, dvox, dminv = out["dgrid"], out["dvox"], out["dminv"]
        self.last_dgrid = dgrid
        dpose = None
        if want_dpose:
            dpose = pose_matrix_jacobian_vjp(self.view_params, dminv.cpu().numpy(), self.size, self.new_size)
        if dvox is not None and not dvox_on_device:
            dvox = dvox.cpu().numpy()
        return dvox, dpose

    def _input_chain(self, rec, g, grads):
        """e_conv1 (5^3 s2, 1 -> 8) fused with the resampler: its data gradient dL/dgrid, fp32 and un-scaled."""
        if rec["op"] != "resample_conv1":
            raise RuntimeError(f"a Shader tape cannot hold a {rec['op']} record")
        if self._need_inputs:
            if rec.get("window") is not None:
                raise NotImplementedError("input gradients (dL/dvoxels, dL/dpose) of a patch forward: render whole frames")
            N = self.new_size
            w32 = rec["w"].to(self.store.device).float().contiguous()
            self._dgrid = ops.conv3d_backward_data_direct(g, w32, (self.B, N, N, N, 1), rec["stride"], want32=True,
                                                          out_scale=1.0 / self.last_loss_scale)


class TextureInputGradients(_InputGradients):
    """Forward + input-gradient backward of the Texture+Normal network (texture decoder -> two resamplings -> concat ->
    RenderNet; RenderNet_Texture_Face_Normal.py:155-179) for a fixed batch size: the gradients face reconstruction descends
    (Reconstruct_RenderNet_Face.py:383-412).

        tig = TextureInputGradients(weights, batch=5, precision="exact")
        albedo, normal = tig.forward(voxels, texture, view_params)        # [B,512,512,3] fp32 each, on the device
        dvox, dtex, dpose = tig.backward(dL_dalbedo, dL_dnormal)          # [B,64,64,64,1], [B,199], [B,3] fp32 (NumPy)

    model="texture": RenderNet_Texture_Face_Normal's decoder_texture + RenderNet, `weights` {tf variable name: array} or None
    (seeded initialisers).  model="pretrained": Reconstruct_RenderNet_Face's texture_decoder_pretrained + RenderNet_pretrained
    (ReLU residual blocks), `weights` the npz-keyed dictionary those functions read.  `loss_scale` as in ShaderInputGradients."""

    _RECORDING = ("tape", "vox", "minv", "view_params", "albedo", "normal", "tex_in", "tex3d")

    def __init__(self, weights: Optional[Dict[str, np.ndarray]], batch: int, precision: str = "exact", model: str = "texture",
                 size: int = 64, new_size: int = 128, loss_scale=None, seed: int = 0, device: str = "cuda",
                 store: Optional[tf.VariableStore] = None):
        if model not in ("texture", "pretrained"):
            raise ValueError(f"model must be 'texture' or 'pretrained', not {model!r}")
        if model == "pretrained" and weights is None:
            raise ValueError("model='pretrained' builds its variables from the npz-keyed weight dictionary: pass one")
        super().__init__(weights if model == "texture" else None, batch, precision, size, new_size, loss_scale, seed, device,
                         store)
        self.model = model
        self.weight_dict = weights if model == "pretrained" else None
        self.albedo = self.normal = None

    def forward(self, voxels, texture, view_params):
        """voxels [B,64,64,64,1], texture [B,199], view_params [B,3] -> (albedo, normal), fp32 [B,512,512,3] on the device.
        voxels may be a CUDA tensor (e.g. the shape decoder's output): it is used in place, without a host round trip."""
        self._set_inputs(voxels, texture, view_params)
        self.tape = []
        self.store.tape = self.tape
        try:
            with tf.use_store(self.store):
                self._record_network(is_training=False, prob=1.0)
        finally:
            self.store.tape = None
        return self.albedo, self.normal

    def _set_inputs(self, voxels, texture, view_params):
        dev = self.store.device
        self.view_params = np.asarray(view_params, np.float32)
        if isinstance(voxels, torch.Tensor) and voxels.is_cuda:
            self.vox = voxels.to(device=dev, dtype=torch.float32).reshape(self.B, self.size, self.size, self.size, 1).contiguous()
        else:
            self.vox = torch.as_tensor(np.asarray(voxels, np.float32)).reshape(self.B, self.size, self.size, self.size, 1).to(dev)
        self.tex_in = torch.as_tensor(np.asarray(texture, np.float32)).reshape(self.B, -1).to(dev).contiguous()
        self.minv = torch.from_numpy(pose_to_matrix(self.view_params, self.size, self.new_size)).to(dev)

    def _record_network(self, is_training: bool, prob: float, window=None):
        """Decoder -> two deferred resamplings -> RenderNet under the current store and tape (is_training / prob: dropout).
        window = (y0, x0, ph, pw): the network runs on that patch of the concatenated grid (CroppedGrid)."""
        from .RenderNet_Texture_Face_Normal import RenderNet as RenderNetTexture, decoder_texture
        from .Reconstruct_RenderNet_Face import RenderNet_pretrained, texture_decoder_pretrained
        if self.model == "texture":
            self.tex3d = tf.realize(decoder_texture(self.tex_in))
        else:
            self.tex3d = tf.realize(texture_decoder_pretrained(self.tex_in, self.weight_dict))
        # both resamplings stay deferred: resample x2 + axis transform + concat + e_conv1 run as one kernel, whose
        # record holds the very tensors (geometry, decoded texture) the backward scatters into
        grid = ConcatResampledGrid(ResampledGrid(self.vox, self.minv, self.new_size, transform=True),
                                   ResampledGrid(self.tex3d, self.minv, self.new_size, transform=True))
        if window is not None:
            grid = CroppedGrid(grid, *window)
        if self.model == "texture":
            self.albedo, self.normal = RenderNetTexture(grid, prob=prob, is_training=is_training)
        else:
            self.albedo, self.normal = RenderNet_pretrained(grid, self.weight_dict)

    def backward(self, d_albedo, d_normal, want_dvox: bool = True, want_dtex: bool = True, want_dpose: bool = True,
                 want_weight_grads: bool = False, dvox_on_device: bool = False):
        """d_albedo, d_normal: dL/d(albedo), dL/d(normal map) [B,512,512,3] (NumPy or tensor; None = zero).  Returns
        (dL/dvoxels [B,64,64,64,1], dL/dtexture [B,199], dL/dview_params [B,3]) as fp32 NumPy arrays, each None unless asked for.
        dvox_on_device: dL/dvoxels stays a CUDA tensor (for ShapeDecoderGradients.backward)."""
        if want_weight_grads:
            raise NotImplementedError("TextureInputGradients differentiates the inputs only: the weight gradients of the "
                                      "Texture+Normal network come from training.TextureTrainer")
        return self._walk_outputs(d_albedo, d_normal, want_dvox, want_dtex, want_dpose, False, dvox_on_device)

    def _walk_outputs(self, d_albedo, d_normal, want_dvox: bool, want_dtex: bool, want_dpose: bool, want_weight_grads: bool,
                      dvox_on_device: bool):
        """backward's walk.  want_weight_grads (rendernet_b200.nn.TextureRenderer): the walk TextureTrainer.loss_and_gradients
        runs, filling `self.weight_grads` {variable name: fp32 device tensor}, dL/d(texture volume) carried through the decoder
        with its weight gradients -- together with the input gradients asked for (the decoder's FC then also yields dL/d(texture
        vector))."""
        if self.tape is None:
            raise RuntimeError("call forward() first")
        dev = self.store.device
        grads = {}
        for out, d in ((self.albedo, d_albedo), (self.normal, d_normal)):
            if d is None:
                continue
            d = torch.as_tensor(np.asarray(d, np.float32) if not isinstance(d, torch.Tensor) else d).to(dev).float()
            if tuple(d.shape) != tuple(out.shape):
                raise ValueError(f"output gradient shape {tuple(d.shape)} != output shape {tuple(out.shape)}")
            grads[_key(out)] = d.contiguous()
        self._want = (want_dvox, want_dtex or want_weight_grads, want_dpose)
        self._fc_dx = want_weight_grads and want_dtex
        out = {}

        def walk(shrink):
            self._dvox = self._dminv = None
            self._dtex_reached = False
            self.last_dgrid = None
            if want_weight_grads:
                self.weight_grads = {}
            g = dict(grads)
            self._reverse_walk(g, want_weight_grads, True, shrink)
            dtex = None
            if want_dtex:
                dtex = g.pop(_key(self.tex_in), None)
                if dtex is None and self._dtex_reached:
                    raise RuntimeError("dL/d(texture volume) was computed but never reached the texture vector: the tape "
                                       "lost the link between the resampler and the texture decoder")
            out["dtex"] = dtex
            # with weight gradients every path of the walk reaches e_conv1's filter gradient
            first = next((w for n, w in self.weight_grads.items() if n.endswith("e_conv1/e_conv1/weights")), None) \
                if want_weight_grads else None
            return self._dvox, dtex, self._dminv, first

        out["dtex"] = self._dvox = self._dminv = self.last_dgrid = None
        try:
            with torch.cuda.device(self.device), tf.use_store(self.store):
                if grads and (want_dvox or want_dtex or want_dpose or want_weight_grads):
                    self._walk_checked(walk)
                torch.cuda.synchronize()
        finally:
            self._fc_dx = False
        dtex = out["dtex"]
        B, S = self.B, self.size
        dvox = dpose = None
        if want_dvox and dvox_on_device:
            dvox = self._dvox if self._dvox is not None else torch.zeros((B, S, S, S, 1), device=dev, dtype=torch.float32)
        elif want_dvox:
            dvox = self._dvox.cpu().numpy() if self._dvox is not None else np.zeros((B, S, S, S, 1), np.float32)
        if want_dtex:
            dtex = dtex.cpu().numpy() if dtex is not None else np.zeros(tuple(self.tex_in.shape), np.float32)
        if want_dpose:
            dminv = self._dminv.cpu().numpy() if self._dminv is not None else np.zeros((B, 3, 4), np.float32)
            dpose = pose_matrix_jacobian_vjp(self.view_params, dminv, self.size, self.new_size)
        return dvox, dtex, dpose

    def _input_chain(self, rec, g, grads):
        """e_conv1 (5^3 s2, 5 -> 8) fused with both resamplings: dL/d(concat) [B,N,N,N,5] fp32 from the thin data-gradient
        kernel, then rn_resample5_backward_f32 -> dvox, dM^-1 and dL/d(decoded texture), which continues into the decoder."""
        if rec["op"] != "resample5_conv1":
            raise RuntimeError(f"a Texture tape cannot hold a {rec['op']} record")
        want_dvox, want_dtex, want_dpose = self._want
        grid, win = rec["grid"], rec.get("window")
        N = self.new_size
        ph, pw = (N, N) if win is None else win[2:]      # a patch record: dL/d(the concat's window), scattered from it alone
        dgrid = ops.conv3d_backward_data_direct(g, self._w32(rec["w"]), (self.B, ph, pw, N, 5), rec["stride"], want32=True,
                                                out_scale=1.0 / self.last_loss_scale)
        self.last_dgrid = dgrid
        self._dvox, dtex, self._dminv = ops.resample5_backward(grid.geom.voxel, grid.tex.voxel, grid.minv, dgrid, want_dvox,
                                                               want_dtex, want_dpose, window=win)
        if dtex is not None:
            grads[_key(grid.tex.voxel)] = dtex
            self._dtex_reached = True


class ShapeDecoderGradients(_InputGradients):
    """Forward + latent gradient of the face-reconstruction shape decoder (Reconstruct_RenderNet_Face.decoder_3d_pretrained,
    reference :31-75) for a fixed batch size: the first link of `tf.gradients(recon_loss, initial_vector)` (:402).

        sdg = ShapeDecoderGradients(weight_dict_decoder, batch=5)
        vox = sdg.forward(latent)                 # [B,64,64,64,1] fp32 on the device (tape recorded)
        dlatent = sdg.backward(dvox)              # [B,200] fp32 (NumPy); dvox NumPy or a CUDA tensor
        dlatent = sdg.backward(dvox, want_weight_grads=True)   # ... and sdg.weight_grads {tf name: dL/dvariable} (fine-tuning)

    Every layer is fp32 on the CUDA cores (rn_fully_connected, rn_conv3d_f32), whatever the Texture+Normal network's precision,
    so the object has no precision of its own.  `weight_dict`: the decoder's npz-keyed arrays (g_zP_g_gc1_weights, ...)."""

    _RECORDING = ("tape", "latent", "vox")

    def __init__(self, weight_dict: Dict[str, np.ndarray], batch: int, device: str = "cuda",
                 store: Optional[tf.VariableStore] = None):
        super().__init__(None, batch, "exact", 64, 128, 1.0, 0, device, store)    # fp32 walk: the scale is never applied
        self.weight_dict = weight_dict
        self.vox = None

    def forward(self, latent) -> torch.Tensor:
        from .Reconstruct_RenderNet_Face import decoder_3d_pretrained
        dev = self.store.device
        lat = latent if isinstance(latent, torch.Tensor) else torch.as_tensor(np.asarray(latent, np.float32))
        self.latent = lat.to(device=dev, dtype=torch.float32).reshape(self.B, -1).contiguous()
        self.tape = []
        self.store.tape = self.tape
        try:
            with torch.cuda.device(self.device), tf.use_store(self.store):
                self.vox = tf.realize(decoder_3d_pretrained(self.latent, self.weight_dict))
        finally:
            self.store.tape = None
        return self.vox

    def backward(self, dvox, on_device: bool = False, want_weight_grads: bool = False, want_dlatent: bool = True):
        """dvox: dL/dvoxels [B,64,64,64,1] -> dL/dlatent [B,200] fp32 (NumPy; a CUDA tensor if on_device), or None without
        want_dlatent.  want_weight_grads: the same walk also fills `self.weight_grads` {tf name: fp32 device tensor in the
        variable's layout} for the decoder's 12 variables (g_zP/g_gc1/weights, g_zP/g_gc1/biases, g_conv1/g_conv1/weights, ...,
        g_conv5/biases); dL/dlatent is bit for bit the one the walk without weight gradients gives.  Without want_dlatent the FC's
        data gradient is skipped."""
        if self.tape is None:
            raise RuntimeError("call forward() first")
        if not (want_dlatent or want_weight_grads):
            raise ValueError("nothing to compute: want_dlatent and want_weight_grads are both False")
        dev = self.store.device
        d = torch.as_tensor(np.asarray(dvox, np.float32) if not isinstance(dvox, torch.Tensor) else dvox).to(dev).float()
        if tuple(d.shape) != tuple(self.vox.shape):
            raise ValueError(f"dvox shape {tuple(d.shape)} != voxel shape {tuple(self.vox.shape)}")
        grads = {_key(self.vox): d.contiguous()}
        if want_weight_grads:
            self.weight_grads = {}
        self._fc_dx = want_dlatent
        try:
            with torch.cuda.device(self.device), tf.use_store(self.store):
                self._reverse_walk(grads, want_weight_grads, True)
                dz = grads.pop(_key(self.latent), None)
                if not want_dlatent:
                    return None
                if dz is None:
                    raise RuntimeError("the shape decoder's tape lost the link between the voxels and the latent vector")
                out = dz if on_device else dz.cpu().numpy()
        finally:
            self._fc_dx = False
        return out
