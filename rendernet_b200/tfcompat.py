"""GPU-backed stand-in for the handful of TensorFlow-1 idioms the reference's *model functions* use
(RenderNet_Shader.py:32-131, tools/layer_util.py): variable scopes, `tf.get_variable`, `tf.add`,
`tf.cast`, `tf.nn.dropout/sigmoid/relu/elu`, `tf.cond`, `slim.conv2d(_transpose)`.

Design: the reference builds a TF graph node by node; TF then runs each node as its own kernel.  Here
each convolution call returns a *deferred* tensor (`Deferred`) whose epilogue is still open, so that the
`prelu(...)`, `tf.add(conv, shortcut)` or `tf.nn.sigmoid(...)` that the reference applies next is folded
into the convolution kernel's fused epilogue instead of becoming a separate pass over HBM.  A deferred
tensor is realised (its kernel launched) the moment anything else consumes it.

Variables live in a `VariableStore` keyed by the reference's scoped names ("encoder/res2_3/con1_3X3/weights", ...);
kernel-ready packed copies are cached per variable.  There is a default store (what `tf.reset_default_graph()` and the
bare model functions use) and every engine owns its own, made current with `use_store` around its forward pass.
"""
from __future__ import annotations

import contextlib
import math
from typing import Callable, Dict, List, Optional

import numpy as np
import torch

from . import ops

float32 = torch.float32
float16 = torch.float16
bfloat16 = torch.bfloat16
int32 = torch.int32

COMPUTE_DTYPE = torch.float16   # element type of every 16-bit plane of the tensor-core path
PRECISIONS = ("fast", "exact")


# ------------------------------------------------------------------------------------------ variables
class VariableStore:
    """Variables (reference names -> fp32 host tensors) + their kernel-ready packed copies for ONE model replica.
    `precision`: "fast" = fp16 operands / stored activations (RN_FMT_F16); "exact" = fp16 hi/lo pairs with three
    tensor-core products per tap (RN_FMT_F16X2), matching the reference's fp32 convolutions to ~1e-6."""

    def __init__(self, precision: str = "fast", device: str = "cuda", seed: int = 0):
        if precision not in PRECISIONS:
            raise ValueError(f"precision must be one of {PRECISIONS}, got {precision!r}")
        self.vars: Dict[str, torch.Tensor] = {}
        self.packed: Dict[str, object] = {}
        self.scope: List[str] = []
        self.rng = np.random.default_rng(seed)
        self.device = device
        self.precision = precision
        self.strict = False            # True: get_variable raises for a name that is not among the loaded weights
        self.loaded: set = set()       # names installed by load_weight_dict
        self.consumed: set = set()     # loaded names a model function has asked for
        self.tape = None               # list -> every realised layer appends a record (rendernet_b200/backward.py)
        self.keep_preact = False       # with a tape: PReLU layers keep their pre-activation (training step) instead of fusing it away
        self.dropout_seed = None       # int -> tf.nn.dropout(keep < 1) draws its masks from (seed, call index, element)
        self.dropout_calls = 0
        self.phong = None              # dict (ops.conv2d_transpose_xfold) -> the output layer applies the Phong composite itself
        self.phong_u8 = None           # ... and leaves the uint8 image here

    @property
    def fmt(self) -> int:
        return 2 if self.precision == "exact" else 0

    def reset(self, seed: int = 0):
        self.vars.clear()
        self.packed.clear()
        self.scope = []
        self.rng = np.random.default_rng(seed)
        self.strict = False
        self.loaded = set()
        self.consumed = set()
        self.tape = None
        self.keep_preact = False
        self.dropout_seed, self.dropout_calls = None, 0
        self.phong, self.phong_u8 = None, None

    def full_name(self, name: str) -> str:
        return "/".join(self.scope + [name])

    def unused(self) -> List[str]:
        """Loaded weights that no model function has consumed (a wrong prefix / spelling shows up here)."""
        return sorted(self.loaded - self.consumed)


_DEFAULT_STORE = VariableStore()
_STORE = _DEFAULT_STORE              # the CURRENT store (module functions below act on it)


def get_store() -> VariableStore:
    return _STORE


@contextlib.contextmanager
def use_store(store: VariableStore):
    """Make `store` the current variable store for the duration of the block (every engine owns one, so engines with
    different weights / precisions can coexist in a process)."""
    global _STORE
    prev = _STORE
    _STORE = store
    try:
        yield store
    finally:
        _STORE = prev


def compute_fmt() -> int:
    """RN_FMT_* of the current store's 16-bit tensors (0 fp16, 2 fp16 hi/lo pairs)."""
    return _STORE.fmt


def set_precision(precision: str):
    """Precision of the current store; packed weights are re-derived on the next use."""
    if precision not in PRECISIONS:
        raise ValueError(f"precision must be one of {PRECISIONS}, got {precision!r}")
    if precision != _STORE.precision:
        _STORE.precision = precision
        _STORE.packed.clear()


def reset_default_graph(seed: int = 0):
    _STORE.reset(seed)


def _npz_key(name: str) -> str:
    """npz-dir spelling of a variable (tools/model_util.py:32-38, Reconstruct_RenderNet_Face.py:128):
    path with '/' -> '_' minus the leading 'encoder/'."""
    n = name[len("encoder/"):] if name.startswith("encoder/") else name
    return n.replace("/", "_")


def load_weight_dict(weights: Dict[str, np.ndarray], strict: bool = True):
    """Install pretrained/seeded weights.  Keys may be TF variable names
    ('encoder/e_conv1/e_conv1/weights[:0]') or the npz-dir spelling ('e_conv1_e_conv1_weights').
    strict (default): a model function that asks for a variable which is NOT among the loaded ones raises KeyError
    instead of silently falling back to a random initialiser, and `get_store().unused()` lists loaded entries nothing
    consumed."""
    _STORE.packed.clear()
    for k, v in weights.items():
        k = k[:-2] if k.endswith(":0") else k
        _STORE.vars[k] = torch.as_tensor(np.asarray(v), dtype=torch.float32)
        _STORE.loaded.add(k)
    _STORE.strict = bool(strict)


def _lookup(full: str) -> Optional[torch.Tensor]:
    v = _STORE.vars.get(full)
    if v is not None:
        if full in _STORE.loaded:
            _STORE.consumed.add(full)
        return v
    alt = _npz_key(full)
    v = _STORE.vars.get(alt)
    if v is not None:
        _STORE.vars[full] = v
        if alt in _STORE.loaded:
            _STORE.consumed.add(alt)
    return v


@contextlib.contextmanager
def variable_scope(name, reuse=None, **_):
    _STORE.scope.append(name)
    try:
        yield
    finally:
        _STORE.scope.pop()


class constant_initializer:
    def __init__(self, value=0.0):
        self.value = value

    def __call__(self, shape):
        return np.full(shape, self.value, np.float32)


class random_normal_initializer:
    def __init__(self, mean=0.0, stddev=1.0):
        self.mean, self.stddev = mean, stddev

    def __call__(self, shape):
        return (_STORE.rng.standard_normal(shape) * self.stddev + self.mean).astype(np.float32)


class xavier_initializer:
    """tf.contrib.layers.xavier_initializer (uniform): limit = sqrt(6/(fan_in+fan_out))."""

    def __call__(self, shape):
        rf = int(np.prod(shape[:-2])) if len(shape) > 2 else 1
        lim = math.sqrt(6.0 / (rf * shape[-2] + rf * shape[-1]))
        return _STORE.rng.uniform(-lim, lim, size=shape).astype(np.float32)


def get_variable(name, shape=None, dtype=None, initializer=None, trainable=True, **_) -> torch.Tensor:
    """tf.get_variable under the current scope; existing (loaded) values win, like a restored checkpoint."""
    full = _STORE.full_name(name)
    v = _lookup(full)
    if v is None:
        if _STORE.strict and not isinstance(initializer, (np.ndarray, torch.Tensor, list, tuple)):
            raise KeyError(f"variable {full!r} (npz spelling {_npz_key(full)!r}) is not among the loaded weights; "
                           f"refusing to fall back to a random initialiser (load_weight_dict(..., strict=False) allows it)")
        if callable(initializer):
            shp = tuple(int(s) for s in (shape if isinstance(shape, (list, tuple)) else [shape]))
            v = torch.from_numpy(initializer(shp))
        elif initializer is not None:
            v = torch.as_tensor(np.asarray(initializer), dtype=torch.float32)
        else:
            shp = tuple(int(s) for s in shape)
            v = torch.from_numpy(xavier_initializer()(shp))
        _STORE.vars[full] = v
    elif shape is not None:
        shp = tuple(int(s) for s in (shape if isinstance(shape, (list, tuple)) else [shape]))
        if tuple(v.shape) != shp:
            raise ValueError(f"variable {full}: stored shape {tuple(v.shape)} != requested {shp}")
    v._rn_name = full
    return v


def global_variables() -> Dict[str, torch.Tensor]:
    return dict(_STORE.vars)


# ------------------------------------------------------------------------------------------ deferred tensors
class Deferred:
    """A convolution whose fused epilogue (activation, residual) is still open."""

    def __init__(self, run: Callable, shape, dtype):
        self._run = run                    # run(act, alpha, residual, want32) -> tensor
        self.shape = tuple(shape)
        self.dtype = dtype
        self.act: Optional[str] = None
        self.alpha: Optional[torch.Tensor] = None
        self.residual: Optional[torch.Tensor] = None
        self._value: Optional[torch.Tensor] = None
        self.want32 = False

    @property
    def open(self) -> bool:
        return self._value is None

    def realize(self) -> torch.Tensor:
        if self._value is None:
            self._value = self._run(self.act, self.alpha, self.residual, self.want32)
            self._run = None
            self.residual = None
        return self._value

    def get_shape(self):
        return list(self.shape)


def realize(x):
    """Materialise a (possibly deferred) tensor (Deferred conv output or a deferred ResampledGrid)."""
    return x.realize() if hasattr(x, "realize") else x


Split16 = ops.Split16      # "exact" precision activation: fp16 hi/lo planes [2, *shape]


def to_float(x) -> torch.Tensor:
    """fp32 copy of any activation (16-bit tensor, fp16 hi/lo pair, deferred tensor) -- for tests / stage dumps."""
    x = realize(x)
    return x.float() if isinstance(x, (Split16, torch.Tensor)) else torch.as_tensor(x).float()


def shape(x):
    return list(x.shape)


def cast(x, dtype):
    """tf.cast.  The reference casts to float32 around residual adds (layer_util.py:73,105); deferred
    tensors pass through untouched because the add happens in fp32 inside the epilogue anyway."""
    if isinstance(x, Deferred):
        return x
    return x                # 16-bit (or hi/lo pair) storage is kept; arithmetic on it is fp32 in-kernel


def add(a, b):
    """tf.add(conv_out, shortcut) -> residual fused into the conv epilogue when possible."""
    if isinstance(a, Deferred) and a.open and a.residual is None:
        a.residual = realize(b)
        return a
    if isinstance(b, Deferred) and b.open and b.residual is None:
        b.residual = realize(a)
        return b
    a, b = realize(a), realize(b)
    return ops.bias_act(a, None, None, None, residual=b)


def cond(pred, true_fn, false_fn):
    return true_fn() if bool(pred) else false_fn()


def constant(v, dtype=None):
    return v


class _NN:
    @staticmethod
    def dropout(x, keep_prob):
        kp = float(keep_prob)
        if kp == 1.0:
            return x
        st = _STORE
        if st.dropout_seed is None:
            raise NotImplementedError("dropout with keep_prob < 1 is the training path: it needs a store with a dropout seed "
                                      "(rendernet_b200.training.ShaderTrainer); inference uses keep_prob(prob, is_training=False)")
        y = realize(x)                         # 16-bit activation of the producing layer (its PReLU already applied)
        if not isinstance(y, ops.Split16) and y.dtype == torch.float32:
            raise NotImplementedError("dropout on an fp32 tensor is not on the Shader path")
        salt = st.dropout_calls                # index of this dropout call within the step: part of the mask's counter
        st.dropout_calls += 1
        yd = ops.dropout(y, kp, st.dropout_seed, salt)
        if st.tape is not None:
            st.tape.append(dict(op="dropout", x=y, y=yd, keep=kp, seed=st.dropout_seed, salt=salt))
        return yd

    @staticmethod
    def sigmoid(x, name=None):
        if isinstance(x, Deferred) and x.open and x.act is None and x.residual is None:
            x.act = "sigmoid"
            x.want32 = True            # the network output is float32 like the reference's
            return x
        return ops.bias_act(realize(x), None, None, "sigmoid", want32=True)

    @staticmethod
    def elu(x, name=None):
        """tf.nn.elu (Reconstruct_RenderNet_Face.py:48-69), fused into the epilogue of the fp32 convolution that produces x."""
        if isinstance(x, Deferred) and x.open and x.act is None and x.residual is None:
            x.act = "elu"
            return x
        raise NotImplementedError("tf.nn.elu runs in the epilogue of the shape decoder's fp32 convolutions: apply it to an "
                                  "unrealised conv3d / conv3d_transpose output")

    @staticmethod
    def relu(x):
        """tf.nn.relu == PReLU with slope 0 (the reference's weight_dict branches, layer_util.py:76,109)."""
        if isinstance(x, Deferred) and x.open and x.act is None and x.residual is None:
            x.act, x.alpha = "prelu", "zeros"
            return x
        x = realize(x)
        zero = torch.zeros(x.shape[-1], device=x.device, dtype=torch.float32)
        return ops.bias_act(x, None, zero, "prelu")


nn = _NN()
