"""A tiny eager NumPy stand-in for the TensorFlow-1 primitives the reference's hot path
calls.  TEST INFRASTRUCTURE ONLY (used by tests/golden/make_golden.py to execute the
reference's *own* Python source from the reference source tree and freeze its outputs).

TensorFlow 1.x cannot be installed in this environment (no network, Python 3.12).
The reference's hot path is ordinary Python that composes ~50 TF primitives
(tools/resampling_voxel_grid.py:370-632, tools/layer_util.py:8-343,
tools/model_util.py:41-49, RenderNet_Shader.py:32-131).  Each primitive below is
implemented from TF-1's documented semantics in float32 NumPy.  The convolutions use
a *direct per-tap* formulation (pad / scatter + one matmul per filter tap) that is
deliberately independent from the torch-based formulation in rendernet_oracle.py, so
that agreement between the two is informative.

install() registers the fake modules `tensorflow`, `tensorflow.contrib`,
`tensorflow.contrib.slim`, `tensorflow.contrib.layers` in sys.modules.
"""
from __future__ import annotations

import contextlib
import math
import sys
import types
from typing import Dict, List, Optional

import numpy as np

float32 = np.float32
int32 = np.int32
bool_ = np.bool_


class Dimension:
    def __init__(self, v):
        self.value = None if v is None else int(v)

    def __int__(self):
        return self.value

    __index__ = __int__

    def __mul__(self, o):
        return Dimension(self.value * int(o))

    __rmul__ = __mul__

    def __eq__(self, o):
        return self.value == (o.value if isinstance(o, Dimension) else o)

    def __hash__(self):
        return hash(self.value)

    def __repr__(self):
        return f"Dimension({self.value})"


class TensorShape(list):
    def as_list(self):
        return [d.value for d in self]


class Tensor(np.ndarray):
    """ndarray with the few TF-1 Tensor methods the reference touches."""

    def get_shape(self):
        return TensorShape(Dimension(s) for s in self.shape)

    def __array_finalize__(self, obj):
        pass


def _T(x, dtype=None):
    a = np.asarray(x, dtype=dtype)
    return a.view(Tensor)


def _ints(shape):
    if isinstance(shape, (Dimension, int, np.integer)):
        return (int(shape),)
    return tuple(int(s) for s in shape)


def _dt(d):
    if d is None:
        return None
    if isinstance(d, str):
        return np.dtype(d)
    return np.dtype(d)


# ---------------------------------------------------------------- variables / scopes
class _State:
    def __init__(self):
        self.scope: List[str] = []
        self.provided: Dict[str, np.ndarray] = {}
        self.created: Dict[str, np.ndarray] = {}
        self.rng = np.random.default_rng(0)


_S = _State()


def reset(provided: Optional[Dict[str, np.ndarray]] = None, seed: int = 0):
    _S.scope = []
    _S.provided = dict(provided or {})
    _S.created = {}
    _S.rng = np.random.default_rng(seed)


def created_variables() -> Dict[str, np.ndarray]:
    return dict(_S.created)


@contextlib.contextmanager
def variable_scope(name, reuse=None, **_):
    _S.scope.append(name)
    try:
        yield
    finally:
        _S.scope.pop()


class _Init:
    def __call__(self, shape, fans=None):
        raise NotImplementedError


class constant_initializer(_Init):
    def __init__(self, value=0.0):
        self.value = value

    def __call__(self, shape, fans=None):
        return np.full(shape, self.value, np.float32)


class random_normal_initializer(_Init):
    def __init__(self, mean=0.0, stddev=1.0):
        self.mean, self.stddev = mean, stddev

    def __call__(self, shape, fans=None):
        return (_S.rng.standard_normal(shape) * self.stddev + self.mean).astype(np.float32)


class xavier_initializer(_Init):
    def __call__(self, shape, fans=None):
        rf = int(np.prod(shape[:-2])) if len(shape) > 2 else 1
        fi, fo = rf * shape[-2], rf * shape[-1]
        lim = math.sqrt(6.0 / (fi + fo))
        return _S.rng.uniform(-lim, lim, size=shape).astype(np.float32)


class zeros_initializer(constant_initializer):
    def __init__(self):
        super().__init__(0.0)


def get_variable(name, shape=None, dtype=None, initializer=None, trainable=True, **_):
    full = "/".join(_S.scope + [name])
    if full in _S.provided:
        v = np.asarray(_S.provided[full], np.float32)
        if shape is not None and tuple(v.shape) != _ints(shape):
            raise ValueError(f"shape mismatch for {full}: provided {v.shape} wanted {_ints(shape)}")
    elif isinstance(initializer, _Init):
        v = initializer(_ints(shape))
    elif initializer is not None:
        v = np.asarray(initializer, np.float32)
    else:
        v = xavier_initializer()(_ints(shape))
    _S.created[full] = v
    return _T(v)


# ---------------------------------------------------------------- basic ops
def shape(x):
    return np.asarray(np.shape(x), np.int32)


def reshape(x, shp):
    return _T(np.reshape(np.asarray(x), _ints(shp)))


def cast(x, dtype):
    return _T(np.asarray(x).astype(_dt(dtype)))


def to_int32(x):
    if isinstance(x, Dimension):
        return int(x)
    return _T(np.asarray(x).astype(np.int32))


def constant(value, dtype=None, shape=None):
    a = np.asarray(value)
    if dtype is not None:
        a = a.astype(_dt(dtype))
    elif a.dtype.kind == "f":
        a = a.astype(np.float32)          # TF default float type
    elif a.dtype.kind == "i":
        a = a.astype(np.int32)
    if shape is not None:
        a = np.broadcast_to(a, _ints(shape)).copy()
    return _T(a)


def zeros(shp, dtype="float32"):
    return _T(np.zeros(_ints(shp), _dt(dtype)))


def ones(shape=None, dtype="float32"):
    return _T(np.ones(_ints(shape), _dt(dtype)))


def ones_like(x):
    return _T(np.ones_like(np.asarray(x)))


def zeros_like(x):
    return _T(np.zeros_like(np.asarray(x)))


def range_(*args, dtype=None):
    a = np.arange(*[int(v) if not isinstance(v, float) else v for v in args])
    a = a.astype(_dt(dtype) if dtype is not None else np.int32)
    return _T(a)


def floor(x):
    return _T(np.floor(np.asarray(x)))


def clip_by_value(x, lo, hi):
    return _T(np.clip(np.asarray(x), lo, hi))


def matmul(a, b):
    return _T(np.matmul(np.asarray(a), np.asarray(b)))


def matrix_inverse(a):
    a = np.asarray(a)
    return _T(np.linalg.inv(a).astype(a.dtype))


def gather(params, idx):
    return _T(np.asarray(params)[np.asarray(idx)])


def expand_dims(x, axis):
    return _T(np.expand_dims(np.asarray(x), axis))


def add_n(xs):
    out = np.asarray(xs[0])
    for t in xs[1:]:
        out = out + np.asarray(t)
    return _T(out)


def add(a, b):
    return _T(np.asarray(a) + np.asarray(b))


def meshgrid(*xs, indexing="xy"):
    return [_T(g) for g in np.meshgrid(*[np.asarray(x) for x in xs], indexing=indexing)]


def concat(xs, axis=0):
    return _T(np.concatenate([np.asarray(x) for x in xs], axis=axis))


def tile(x, multiples):
    return _T(np.tile(np.asarray(x), _ints(multiples)))


def transpose(x, perm=None):
    return _T(np.transpose(np.asarray(x), perm))


def cos(x):
    return _T(np.cos(np.asarray(x)))


def sin(x):
    return _T(np.sin(np.asarray(x)))


def maximum(a, b):
    return _T(np.maximum(np.asarray(a, np.float32) if np.isscalar(a) else a, b))


def minimum(a, b):
    return _T(np.minimum(np.asarray(a, np.float32) if np.isscalar(a) else a, b))


def cond(pred, true_fn, false_fn):
    return true_fn() if bool(pred) else false_fn()


def identity(x):
    return x


class InvalidArgumentError(Exception):
    pass


# ---------------------------------------------------------------- nn ops (direct per-tap forms)
def _same_pad(n_in, k, s):
    out = -(-n_in // s)
    total = max((out - 1) * s + k - n_in, 0)
    return out, total // 2, total - total // 2


def _conv_nd(x, w, strides, padding):
    """Forward cross-correlation, channel-last.  y[o] = sum_tap x[o*s + tap - pb] . w[tap]."""
    assert padding == "SAME"
    x = np.asarray(x, np.float32); w = np.asarray(w, np.float32)
    nd = x.ndim - 2
    s = list(strides[1:1 + nd])
    ks = w.shape[:nd]
    outs, pads = [], []
    for d in range(nd):
        o, pb, pa = _same_pad(x.shape[1 + d], ks[d], s[d])
        outs.append(o); pads.append((pb, pa))
    xp = np.pad(x, [(0, 0)] + pads + [(0, 0)])
    y = np.zeros((x.shape[0], *outs, w.shape[-1]), np.float32)
    for tap in np.ndindex(*ks):
        sl = tuple(slice(tap[d], tap[d] + (outs[d] - 1) * s[d] + 1, s[d]) for d in range(nd))
        y += np.matmul(xp[(slice(None),) + sl], w[tap])
    return _T(y)


def _conv_nd_transpose(x, w, output_shape, strides, padding):
    """Gradient of the forward SAME conv: full[i*s + tap] += x[i] . w[tap]^T, cropped at pb."""
    assert padding == "SAME"
    x = np.asarray(x, np.float32); w = np.asarray(w, np.float32)
    nd = x.ndim - 2
    s = list(strides[1:1 + nd])
    ks = w.shape[:nd]
    ins = x.shape[1:1 + nd]
    full_sz = [(ins[d] - 1) * s[d] + ks[d] for d in range(nd)]
    full = np.zeros((x.shape[0], *full_sz, w.shape[-2]), np.float32)
    for tap in np.ndindex(*ks):
        sl = tuple(slice(tap[d], tap[d] + (ins[d] - 1) * s[d] + 1, s[d]) for d in range(nd))
        full[(slice(None),) + sl] += np.matmul(x, w[tap].T)
    crop = []
    for d in range(nd):
        o = int(output_shape[1 + d])
        _, pb, _ = _same_pad(o, ks[d], s[d])
        crop.append(slice(pb, pb + o))
    return _T(np.ascontiguousarray(full[(slice(None),) + tuple(crop)]))


def _sigmoid(x, name=None):
    x = np.asarray(x, np.float32)
    return _T((1.0 / (1.0 + np.exp(-x))).astype(np.float32))


def _dropout(x, keep_prob):
    kp = float(np.asarray(keep_prob))
    if kp != 1.0:
        raise NotImplementedError("shim only supports inference (keep_prob == 1)")
    return x


def _relu(x):
    return _T(np.maximum(np.asarray(x), 0))


# ---------------------------------------------------------------- slim
def _slim_conv2d(inputs, num_outputs, kernel_size, stride=1, padding="SAME", activation_fn=None,
                 scope=None, **_):
    ks = [kernel_size] * 2 if isinstance(kernel_size, int) else list(kernel_size)
    st = [stride] * 2 if isinstance(stride, int) else list(stride)
    cin = inputs.shape[-1]
    with variable_scope(scope or "Conv"):
        w = get_variable("weights", ks + [cin, int(num_outputs)], initializer=xavier_initializer())
        b = get_variable("biases", [int(num_outputs)], initializer=zeros_initializer())
    y = _conv_nd(inputs, w, [1] + st + [1], padding) + np.asarray(b)
    assert activation_fn is None
    return _T(y)


def _slim_conv2d_transpose(inputs, num_outputs, kernel_size, stride=1, padding="SAME",
                           activation_fn=None, scope=None, **_):
    ks = [kernel_size] * 2 if isinstance(kernel_size, int) else list(kernel_size)
    st = [stride] * 2 if isinstance(stride, int) else list(stride)
    cin = inputs.shape[-1]
    with variable_scope(scope or "Conv2d_transpose"):
        w = get_variable("weights", ks + [int(num_outputs), cin], initializer=xavier_initializer())
        b = get_variable("biases", [int(num_outputs)], initializer=zeros_initializer())
    oshape = [inputs.shape[0], inputs.shape[1] * st[0], inputs.shape[2] * st[1], int(num_outputs)]
    y = _conv_nd_transpose(inputs, w, oshape, [1] + st + [1], padding) + np.asarray(b)
    assert activation_fn is None
    return _T(y)


def install():
    """Register fake `tensorflow` modules; returns the top-level module."""
    tf = types.ModuleType("tensorflow")
    for k, v in dict(
        float32=float32, int32=int32, bool=bool_, Tensor=Tensor,
        variable_scope=variable_scope, get_variable=get_variable,
        constant_initializer=constant_initializer, random_normal_initializer=random_normal_initializer,
        shape=shape, reshape=reshape, cast=cast, to_int32=to_int32, constant=constant, zeros=zeros,
        ones=ones, ones_like=ones_like, zeros_like=zeros_like, range=range_, floor=floor,
        clip_by_value=clip_by_value, matmul=matmul, matrix_inverse=matrix_inverse, gather=gather,
        expand_dims=expand_dims, add_n=add_n, add=add, meshgrid=meshgrid, concat=concat, tile=tile,
        transpose=transpose, cos=cos, sin=sin, maximum=maximum, minimum=minimum, cond=cond,
        identity=identity, InvalidArgumentError=InvalidArgumentError,
    ).items():
        setattr(tf, k, v)
    nn = types.ModuleType("tensorflow.nn")
    nn.conv3d = lambda x, w, padding, strides: _conv_nd(x, w, strides, padding)
    nn.conv2d = lambda x, w, padding, strides: _conv_nd(x, w, strides, padding)
    nn.conv2d_transpose = lambda x, w, output_shape, strides, padding: _conv_nd_transpose(x, w, output_shape, strides, padding)
    nn.conv3d_transpose = lambda x, w, output_shape, strides, padding: _conv_nd_transpose(x, w, output_shape, strides, padding)
    nn.sigmoid = _sigmoid
    nn.dropout = _dropout
    nn.relu = _relu
    tf.nn = nn
    contrib = types.ModuleType("tensorflow.contrib")
    slim = types.ModuleType("tensorflow.contrib.slim")
    slim.conv2d = _slim_conv2d
    slim.conv2d_transpose = _slim_conv2d_transpose
    layers = types.ModuleType("tensorflow.contrib.layers")
    layers.xavier_initializer = xavier_initializer
    contrib.slim = slim
    contrib.layers = layers
    tf.contrib = contrib
    sys.modules["tensorflow"] = tf
    sys.modules["tensorflow.nn"] = nn
    sys.modules["tensorflow.contrib"] = contrib
    sys.modules["tensorflow.contrib.slim"] = slim
    sys.modules["tensorflow.contrib.layers"] = layers
    return tf
