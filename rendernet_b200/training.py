"""The training steps of the Shader network (SURVEY §8 f-4, stage 2) -- RenderNet_Shader.py:154-167 on the H100 path -- and of the
Texture+Normal network (TextureTrainer, RenderNet_Texture_Face_Normal.py:155-187).  The Shader step:

    images_pred = RenderNet(rotated voxels, is_training=True, prob=cfg['keep_prob'])          (:156, dropout after ten layers)
    recon_loss  = BCE (greyscale, :159-161)  |  tf.losses.mean_squared_error (:163)
    learning_rate = tf.train.exponential_decay(cfg['e_eta'], global_step, cfg['decay_steps'], 0.96, staircase=True)   (:166)
    tf.train.AdamOptimizer(learning_rate, beta1=0.5).minimize(recon_loss, global_step)       (:167)

One `ShaderTrainer.step(voxels, view_params, target)` = forward with a tape (tensor-core convolutions, stateless hashed dropout)
-> loss + dL/dimage (rn_image_loss_grad) -> backward walk (rendernet_b200/backward.py: data gradients through the wgmma
implicit-GEMM kernel, weight gradients through the wgmma weight-gradient kernel / the strided-correlation kernel, bias and
PReLU-slope reductions) -> rn_adam_step on every variable -> the kernel-ready packed copies of the filters are dropped and
re-packed from the updated fp32 masters at the next forward.

Scope notes.  The variables live on the device as fp32 masters (exactly what TF keeps); arithmetic inside the convolutions is the
store's precision mode ("exact": fp16 hi/lo operand pairs, fp32-equivalent; "fast": fp16 operands, gradients loss-scaled).  The
reference's random patch crop (:152-155, a memory workaround of 2018 GPUs) is not reproduced: a step trains on whole frames.
Data loading, the Supervisor / checkpoint loop and sample dumps (:170-306) stay out of scope (SURVEY §2)."""
from __future__ import annotations

import contextlib
import math
from typing import Dict, Optional

import numpy as np
import torch

from . import ops
from . import tfcompat as tf
from .RenderNet_Shader import RenderNet
from .backward import ShaderInputGradients, TextureInputGradients, _key
from .engine import pose_to_matrix
from .resampling_voxel_grid import ResampledGrid

# every path of a backward walk reaches e_conv1's filter gradient: an fp16 overflow anywhere makes it non-finite
E_CONV1_WEIGHTS = "encoder/e_conv1/e_conv1/weights"


def _as_device_f32(t, like: torch.Tensor) -> torch.Tensor:
    t = torch.as_tensor(np.asarray(t, np.float32) if not isinstance(t, torch.Tensor) else t)
    return t.to(device=like.device, dtype=torch.float32).reshape(tuple(like.shape)).contiguous()


class _Trainer:
    """What ShaderTrainer and TextureTrainer share: the learning-rate schedule, the dropout seed, Adam over the fp32 masters and
    the re-pack of the kernel-ready filters, the dynamic-loss-scale retry loop, data-parallel averaging and state_dict.  A
    subclass also derives from an input-gradient class (the variable store, the tape, the reverse walk) and defines
    `loss_and_gradients(*inputs, training=True) -> (loss, {variable name: gradient})`."""

    def _init_training(self, keep_prob: float, learning_rate: float, decay_steps: int, decay_rate: float, beta1: float,
                       beta2: float, epsilon: float, seed: int, data_parallel: bool):
        # dynamic loss scaling lives in _step(): an overflow halves the headroom target (or a fixed scale) and redoes the step;
        # after growth_interval steps without one the target doubles again, up to where it started
        self.overflow_retries = 0
        self.growth_interval = 1000
        self._target_ceiling = self.scale_target
        self._steps_since_overflow = 0
        self.data_parallel = bool(data_parallel)      # one process per GPU, `batch` items each: gradients averaged over the ranks
        if not 0.0 < keep_prob <= 1.0:
            raise ValueError("keep_prob must be in (0, 1]")
        self.keep_prob = float(keep_prob)
        self.e_eta, self.decay_steps, self.decay_rate = float(learning_rate), int(decay_steps), float(decay_rate)
        self.beta1, self.beta2, self.epsilon = float(beta1), float(beta2), float(epsilon)
        self.global_step = 0
        self.seed = int(seed)
        self.m: Dict[str, torch.Tensor] = {}
        self.v: Dict[str, torch.Tensor] = {}
        self.last_loss: Optional[float] = None

    # ------------------------------------------------------------------------------------------- pieces of a step
    def learning_rate(self, step: Optional[int] = None) -> float:
        """tf.train.exponential_decay(e_eta, global_step, decay_steps, 0.96, staircase=True)."""
        step = self.global_step if step is None else step
        return self.e_eta * self.decay_rate ** (step // self.decay_steps)

    def dropout_seed(self, step: int) -> int:
        """Seed of the dropout masks of optimiser step `step` (mixes the trainer's seed and the step; 32 bits)."""
        rank = 0
        if self.data_parallel and torch.distributed.is_available() and torch.distributed.is_initialized():
            rank = torch.distributed.get_rank()           # data-parallel ranks draw different masks from the same trainer seed
        return (self.seed * 0x9E3779B1 + step * 0x85EBCA6B + rank * 0xC2B2AE35 + 0x1234567) & 0xFFFFFFFF

    @contextlib.contextmanager
    def _training_tape(self, training: bool):
        """Record a fresh tape; PReLU layers keep their pre-activation on it (slope gradient, derivative); with training and
        keep_prob < 1 the dropout masks are drawn from (seed, global_step, call index, element)."""
        self.tape = []
        st = self.store
        st.tape = self.tape
        st.keep_preact = True
        st.dropout_seed = self.dropout_seed(self.global_step) if (training and self.keep_prob < 1.0) else None
        st.dropout_calls = 0
        try:
            with torch.cuda.device(self.device), tf.use_store(st):
                yield
                self._adopt_variables()
        finally:
            st.tape = None
            st.keep_preact = False
            st.dropout_seed = None

    def _adopt_variables(self):
        """Move the fp32 masters of every variable to the device (once): Adam updates them in place, the packers read them there."""
        dev = self.store.device
        for name, t in list(self.store.vars.items()):
            if not t.is_cuda:
                d = t.to(device=dev, dtype=torch.float32).contiguous()
                d._rn_name = name
                self.store.vars[name] = d

    def apply_gradients(self, grads: Dict[str, torch.Tensor]):
        """tf.train.AdamOptimizer.apply_gradients + global_step += 1; then the packed (kernel-layout) filter copies are dropped."""
        t = self.global_step + 1
        lr_t = self.learning_rate(self.global_step) * math.sqrt(1.0 - self.beta2 ** t) / (1.0 - self.beta1 ** t)
        with torch.cuda.device(self.device):
            for name, g in grads.items():
                p = self.store.vars[name]
                if tuple(g.shape) != tuple(p.shape):
                    raise ValueError(f"gradient of {name}: shape {tuple(g.shape)} != variable shape {tuple(p.shape)}")
                if name not in self.m:
                    self.m[name], self.v[name] = torch.zeros_like(p), torch.zeros_like(p)
                ops.adam_step(p, g.contiguous(), self.m[name], self.v[name], lr_t, self.beta1, self.beta2, self.epsilon)
        self.global_step = t
        self.store.packed.clear()            # forward filters, biases, slopes ...
        self._dgrad_cache.clear()            # ... and the mirrored data-gradient filters are re-packed from the new masters

    def _check_all_variables(self):
        missing = sorted(set(self.store.vars) - set(self.weight_grads))
        if missing:
            raise RuntimeError(f"{len(missing)} variables received no gradient, e.g. {missing[:3]}")

    # ------------------------------------------------------------------------------------------- the step
    def _step(self, *inputs) -> float:
        """One optimiser step on `inputs` (loss_and_gradients' arguments); returns the loss BEFORE the update."""
        dp = self.data_parallel and torch.distributed.is_available() and torch.distributed.is_initialized()
        for _ in range(12):
            overflow = False
            try:
                loss, grads = self.loss_and_gradients(*inputs, training=True)
            except FloatingPointError:                 # dynamic loss scaling: halve and redo the step (same dropout masks)
                overflow = True
            if dp:                                     # every rank must take the same branch
                flag = torch.tensor([1.0 if overflow else 0.0], device=self.store.device)
                torch.distributed.all_reduce(flag, op=torch.distributed.ReduceOp.MAX)
                overflow = bool(flag.item() > 0)
            if not overflow:
                break
            self._steps_since_overflow = 0
            if self.loss_scale is None:
                self.scale_target *= 0.5
            else:
                self.loss_scale *= 0.5
        else:
            raise FloatingPointError("the backward pass overflows even at a loss scale of %g" % self.last_loss_scale)
        self._steps_since_overflow += 1
        if (self.loss_scale is None and self._steps_since_overflow >= self.growth_interval
                and self.scale_target < self._target_ceiling):
            self.scale_target *= 2.0
            self._steps_since_overflow = 0
        if dp:
            # data-parallel step: every rank holds the same variables and its own `batch` items; the mean loss over the global
            # batch is the mean of the per-rank means, so the gradients are averaged (NCCL all-reduce, bucketed) before Adam
            from .parallel import all_reduce_gradients
            all_reduce_gradients(grads, average=True)
            lt = torch.tensor([loss], device=self.store.device, dtype=torch.float64)
            torch.distributed.all_reduce(lt)
            loss = float(lt.item()) / torch.distributed.get_world_size()
        self.apply_gradients(grads)
        return loss

    def state_dict(self) -> Dict[str, np.ndarray]:
        """{tf variable name: fp32 ndarray}: what tf.train.Saver would write (loadable by every engine of this package)."""
        return {name: t.detach().cpu().numpy().copy() for name, t in self.store.vars.items()}


class ShaderTrainer(_Trainer, ShaderInputGradients):
    """Adam training of RenderNet_Shader.RenderNet for a fixed batch size.

        tr = ShaderTrainer(None, batch=1, precision="exact", keep_prob=0.75, learning_rate=1e-5)      # reference initialisers
        loss = tr.step(voxels[B,64,64,64,1], view_params[B,3], target[B,512,512,3])                   # one optimiser step
        weights = tr.state_dict()                                                                      # {tf name: ndarray}

    learning_rate / decay_steps / keep_prob default to config_RenderNet.json (e_eta 1e-5, 100000, 1.0); beta1 = 0.5 as in
    RenderNet_Shader.py:167, beta2 / epsilon are TF's defaults.  loss_scale=None (default) chooses the 16-bit gradients' scale
    per step below the headroom target `scale_target`; an fp16 overflow halves that target and redoes the step with the same
    dropout masks, and `growth_interval` overflow-free steps double it again, up to its initial value.  A fixed loss_scale is
    halved on overflow instead.  data_parallel=True (one process per GPU under torchrun, same
    initial weights / seed on every rank; the rank is mixed into the dropout-mask seed): gradients are averaged over the
    ranks before Adam (rendernet_b200.parallel.all_reduce_gradients; its bucketing is tested on a 2-process gloo group, the
    multi-GPU step itself has not been run on GPUs in round 2)."""

    def __init__(self, weights: Optional[Dict[str, np.ndarray]], batch: int, precision: str = "exact", is_greyscale: bool = False,
                 keep_prob: float = 1.0, learning_rate: float = 1e-5, decay_steps: int = 100000, decay_rate: float = 0.96,
                 beta1: float = 0.5, beta2: float = 0.999, epsilon: float = 1e-8, loss: Optional[str] = None,
                 size: int = 64, new_size: int = 128, loss_scale=None, seed: int = 0, device: str = "cuda",
                 data_parallel: bool = False):
        super().__init__(weights, batch, precision=precision, is_greyscale=is_greyscale, size=size, new_size=new_size,
                         loss_scale=loss_scale, seed=seed, device=device)
        self._init_training(keep_prob, learning_rate, decay_steps, decay_rate, beta1, beta2, epsilon, seed, data_parallel)
        self.loss_kind = loss or ("bce" if is_greyscale else "mse")        # RenderNet_Shader.py:158-163

    def forward(self, voxels, view_params, training: bool = True) -> torch.Tensor:
        """The training-mode forward pass (dropout masks drawn from (seed, global_step, call index, element)); tape recorded."""
        dev = self.store.device
        self.view_params = np.asarray(view_params, np.float32)
        self.vox = torch.as_tensor(np.asarray(voxels, np.float32)).reshape(self.B, self.size, self.size, self.size, 1).to(dev)
        self.minv = torch.from_numpy(pose_to_matrix(self.view_params, self.size, self.new_size)).to(dev)
        with self._training_tape(training):
            grid = ResampledGrid(self.vox, self.minv, self.new_size, transform=True)
            self.img = RenderNet(grid, is_training=training, prob=self.keep_prob, is_greyscale=self.is_greyscale)
        return self.img

    def loss_and_gradients(self, voxels, view_params, target, training: bool = True):
        """-> (loss (Python float), {variable name: dL/dvariable fp32 device tensor}); no update."""
        img = self.forward(voxels, view_params, training=training)
        tgt = _as_device_f32(target, img)
        with torch.cuda.device(self.device):
            loss, dimg = ops.image_loss_grad(img.contiguous(), tgt, self.loss_kind)
        # an fp16 overflow in the walk raises FloatingPointError (overflow_retries = 0: step() chooses the next scale)
        self.backward(dimg, want_dvox=False, want_dpose=False, want_weight_grads=True)
        self._check_all_variables()
        self.last_loss = float(loss.item())
        return self.last_loss, self.weight_grads

    def step(self, voxels, view_params, target) -> float:
        """One optimiser step (RenderNet_Shader.py:156-167); returns the loss BEFORE the update."""
        return self._step(voxels, view_params, target)


class TextureTrainer(_Trainer, TextureInputGradients):
    """Adam training of the Texture+Normal network (RenderNet_Texture_Face_Normal.py:155-187: texture decoder -> two resamplings
    -> concat -> RenderNet with an image and a normal head) for a fixed batch size; all 186 variables, decoder included.

        tr = TextureTrainer(None, batch=1, precision="exact")                  # seeded reference initialisers
        loss = tr.step(voxels[B,64,64,64,1], texture[B,199], view_params[B,3], image_target[B,512,512,3],
                       normal_target[B,512,512,3])                              # one optimiser step
        weights = tr.state_dict()                                               # loadable by engine.TextureRenderEngine

    Loss (:182-183): mean((image - image_target)^2) + mean((normal - normal_target)^2).  Dropout at the twelve sites of the
    mirror (e_conv1, 2, 3, 5, then e_conv6..9 of the Image head, then of the Normal head).  learning_rate / decay_steps /
    keep_prob default to config_RenderNet_texture.json (1e-5, 100000, 1.0); loss scaling, Adam and data_parallel as in
    ShaderTrainer.  The backward walk asks resample5_backward for dL/d(texture volume) only (the geometry and the pose are
    inputs, not variables) and carries it through the fp32 decoder with its weight gradients."""

    def __init__(self, weights: Optional[Dict[str, np.ndarray]], batch: int, precision: str = "exact", keep_prob: float = 1.0,
                 learning_rate: float = 1e-5, decay_steps: int = 100000, decay_rate: float = 0.96, beta1: float = 0.5,
                 beta2: float = 0.999, epsilon: float = 1e-8, size: int = 64, new_size: int = 128, loss_scale=None,
                 seed: int = 0, device: str = "cuda", data_parallel: bool = False):
        super().__init__(weights, batch, precision=precision, model="texture", size=size, new_size=new_size,
                         loss_scale=loss_scale, seed=seed, device=device)
        self._init_training(keep_prob, learning_rate, decay_steps, decay_rate, beta1, beta2, epsilon, seed, data_parallel)

    def forward(self, voxels, texture, view_params, training: bool = True):
        """The training-mode forward pass -> (image, normal map), fp32 [B,512,512,3] each on the device; tape recorded."""
        self._set_inputs(voxels, texture, view_params)
        with self._training_tape(training):
            self._record_network(is_training=training, prob=self.keep_prob)
        return self.albedo, self.normal

    def loss_and_gradients(self, voxels, texture, view_params, image_target, normal_target, training: bool = True):
        """-> (loss (Python float), {variable name: dL/dvariable fp32 device tensor}); no update."""
        img, nrm = self.forward(voxels, texture, view_params, training=training)
        with torch.cuda.device(self.device):
            l_img, d_img = ops.image_loss_grad(img.contiguous(), _as_device_f32(image_target, img), "mse")
            l_nrm, d_nrm = ops.image_loss_grad(nrm.contiguous(), _as_device_f32(normal_target, nrm), "mse")
        grads = {_key(img): d_img, _key(nrm): d_nrm}
        self._want = (False, True, False)              # resample5_backward: dL/d(texture volume) only

        def walk(shrink):
            self.weight_grads = {}
            self._dvox = self._dminv = self.last_dgrid = None
            self._dtex_reached = False
            self._reverse_walk(dict(grads), True, True, shrink)
            return [self.weight_grads.get(E_CONV1_WEIGHTS)]

        # an fp16 overflow in the walk raises FloatingPointError (overflow_retries = 0: step() chooses the next scale)
        with torch.cuda.device(self.device), tf.use_store(self.store):
            self._walk_checked(walk)
            torch.cuda.synchronize()
        self._check_all_variables()
        self.last_loss = float((l_img + l_nrm).item())
        return self.last_loss, self.weight_grads

    def step(self, voxels, texture, view_params, image_target, normal_target) -> float:
        """One optimiser step (RenderNet_Texture_Face_Normal.py:176-187); returns the loss BEFORE the update."""
        return self._step(voxels, texture, view_params, image_target, normal_target)
