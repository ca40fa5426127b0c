"""Drop-in mirror of the reference's tools/layer_util.py (same function names, argument order, defaults and
variable-scope naming), executing on the sm_90a kernels.  Citations are into the reference RenderNet source tree.

Differences that are deliberate and documented:
  * tensors are torch CUDA tensors (16-bit activations, fp32 accumulation) instead of tf.Tensor;
  * state lives in `tfcompat`'s variable store (names identical to the TF graph's variables);
  * conv ops return deferred tensors so the following prelu / tf.add / sigmoid fuse into the conv epilogue;
  * the per-layer `print(...)` calls of the reference (layer_util.py:157-181) are dropped.
"""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch

from . import ops
from . import tfcompat as tf
from .resampling_voxel_grid import ConcatResampledGrid, CroppedGrid, ResampledGrid
from .tfcompat import Deferred, realize

USE_MERGED_TCONV = True    # one launch (N = 4*Cout, 9 taps) instead of 4 phase launches for k=4 stride-2 transposed convs
USE_XFOLD = True           # fold x-pixels into channels for thin stride-1 transposed convs (e_conv10/11)
USE_FUSED_RESAMPLE_CONV1 = True   # resampler + axis transform + e_conv1 in one kernel with empty-tile skipping
USE_BANDED_CONV3D = True   # depth-folded tensor-core path for 3^3 convs (falls back to the 5-D TMA path)

_XAVIER = tf.xavier_initializer
_RANDN002 = lambda: tf.random_normal_initializer(stddev=0.02)  # noqa: E731  (layer_util.py:149 default)


# ------------------------------------------------------------------------------------------ helpers
def _store():
    return tf.get_store()


def _packed(wvar: torch.Tensor, bvar: Optional[torch.Tensor], kind: str, stride: int = 1):
    st = _store()
    key = (getattr(wvar, "_rn_name", id(wvar)), kind, stride, tf.COMPUTE_DTYPE, st.fmt)
    L = st.packed.get(key)
    if L is None:
        L = ops.pack_conv(kind, wvar, bvar, None, stride=stride, dtype=tf.COMPUTE_DTYPE, device=st.device, fmt=st.fmt)
        st.packed[key] = L
    return L


def _dev_vec(v, n_pad: Optional[int] = None) -> torch.Tensor:
    """fp32 device copy (zero padded to n_pad) of a small per-channel variable, cached."""
    st = _store()
    key = ("vec", getattr(v, "_rn_name", id(v)), n_pad)
    d = st.packed.get(key)
    if d is None:
        t = torch.as_tensor(np.asarray(v) if not isinstance(v, torch.Tensor) else v, dtype=torch.float32).reshape(-1)
        n = t.numel()
        d = torch.zeros(n_pad or n, device=st.device, dtype=torch.float32)
        d[:n] = t.to(st.device)
        st.packed[key] = d
    return d


def _as16(x):
    """Activation in the current store's 16-bit format (fp16 tensor, or a Split16 hi/lo pair in the exact mode)."""
    x = realize(x)
    if isinstance(x, ops.Split16):
        if _store().fmt != 2:
            raise TypeError("fp16 hi/lo activation fed to a fast-precision store")
        return x
    if not isinstance(x, torch.Tensor):
        x = torch.as_tensor(np.asarray(x))
    if not x.is_cuda:
        x = x.to(_store().device)
    if x.dtype == torch.float32:
        return ops.cast_to_16(x.contiguous(), tf.COMPUTE_DTYPE, fmt=_store().fmt)
    if _store().fmt == 2:
        return ops.cast_to_16(x.float().contiguous(), fmt=2)
    return x


def _alpha_arg(alpha, cout_pad):
    if alpha is None:
        return None
    if isinstance(alpha, str) and alpha == "zeros":
        return torch.zeros(cout_pad, device=_store().device, dtype=torch.float32)
    return _dev_vec(alpha, cout_pad)


def _keeps_preact(act, alpha) -> bool:
    """Training step: a PReLU layer keeps its pre-activation on the tape (slope gradient, derivative) instead of fusing it away."""
    st = _store()
    return act == "prelu" and st.tape is not None and st.keep_preact and not isinstance(alpha, str)


def _prelu_f32(z, alpha):
    """PReLU of an fp32 pre-activation: z * (z > 0 ? 1 : alpha) is rn_prelu_backward_f32 with g = z; the same value as the fused
    epilogue max(z, 0) + alpha * min(z, 0) of the decoder kernels."""
    return ops.prelu_backward_f32(z, z, _dev_vec(alpha))


def _record(**rec):
    """Append a layer record to the store's tape (backward.py differentiates the recorded forward pass)."""
    tape = _store().tape
    if tape is not None:
        tape.append(rec)


# ------------------------------------------------------------------------------------------ reference API
def projection_unit(input, n_features=18, scope='projection_unit'):
    """layer_util.py:8-22.  [B,H,W,D,C] -> reshape [B,H,W,D*C] (free in channel-last) -> 1x1 conv -> PReLU.
    `n_features` is overwritten exactly like the reference does (:19)."""
    x = realize(input)
    B, H, W, D, Cc = x.shape
    with tf.variable_scope(scope):
        n_features = D * Cc
        x = x.reshape(B, H, W, n_features)
        conv = prelu(slim_conv2d(inputs=x, num_outputs=n_features, kernel_size=1, activation_fn=None))
        return conv


def lrelu(x, leak=0.2, name="lrelu"):
    """layer_util.py:24-25 (dead code in the reference; kept for API completeness)."""
    x = realize(x)
    a = torch.full((x.shape[-1],), float(leak), dtype=torch.float32)
    return ops.bias_act(_as16(x), None, a.to(_store().device), "prelu")


def prelu(x, trainable=True, alpha=None):
    """layer_util.py:27-45: max(0,x) + alpha*min(0,x); `alpha` variable of shape [channels], init 0."""
    nch = int(x.shape[-1])
    if alpha is None:
        alpha = tf.get_variable(name='alpha', shape=[nch], dtype=tf.float32,
                                initializer=tf.constant_initializer(0.0), trainable=trainable)
    else:
        alpha = tf.get_variable(name='alpha', initializer=alpha, dtype=tf.float32, trainable=trainable)
    if isinstance(x, Deferred) and x.open and x.act is None and x.residual is None:
        x.act, x.alpha = "prelu", alpha
        return x
    return ops.bias_act(_as16(x), None, _dev_vec(alpha), "prelu")


def get_weight(weight_name, weight_dict):
    """layer_util.py:47-58."""
    if weight_dict is None:
        return None
    return weight_dict.get(weight_name)


def res_block_3d(input, out_channels=64, scope='res_block', kernel=[3, 3, 3], stride=[1, 1, 1], weight_dict=None,
                 trainable=True):
    """layer_util.py:60-88: x + conv2(prelu(conv1(x))) (ReLU instead of PReLU when weight_dict is given, :76)."""
    if weight_dict is None:
        with tf.variable_scope(scope):
            net = prelu(conv3d(input, out_channels, kernel_size=kernel, stride=stride, pad="SAME", scope="con1_3X3",
                               weight_initializer_type=_XAVIER()))
            net = conv3d(net, out_channels, kernel_size=kernel, stride=stride, pad="SAME", scope="conv2_3x3",
                         weight_initializer_type=_XAVIER())
        return tf.add(tf.cast(net, tf.float32), tf.cast(input, tf.float32))
    with tf.variable_scope(scope):
        net = tf.nn.relu(conv3d(input, out_channels, kernel_size=kernel, stride=stride, pad="SAME", scope="con1_3X3",
                                trainable=trainable,
                                weight_initializer=get_weight(scope + '_con1_3X3_weights', weight_dict),
                                bias_initializer=get_weight(scope + '_con1_3X3_biases', weight_dict),
                                weight_initializer_type=_XAVIER()))
        net = conv3d(net, out_channels, kernel_size=kernel, stride=stride, pad="SAME", scope="conv2_3x3",
                     trainable=trainable,
                     weight_initializer=get_weight(scope + '_conv2_3x3_weights', weight_dict),
                     bias_initializer=get_weight(scope + '_conv2_3x3_biases', weight_dict),
                     weight_initializer_type=_XAVIER())
    return tf.add(tf.cast(net, tf.float32), tf.cast(input, tf.float32))


def res_block_2d(input, out_channels=64, scope='res_block', kernel=[3, 3], stride=[1, 1], weight_dict=None,
                 trainable=True):
    """layer_util.py:91-121."""
    if weight_dict is None:
        with tf.variable_scope(scope):
            net = prelu(slim_conv2d(input, out_channels, kernel_size=kernel, stride=stride, activation_fn=None,
                                    scope="con1_3X3"))
            net = slim_conv2d(net, num_outputs=out_channels, kernel_size=kernel, stride=stride, activation_fn=None,
                              scope="conv2_3x3")
        return tf.add(tf.cast(net, tf.float32), tf.cast(input, tf.float32))
    with tf.variable_scope(scope):
        net = tf.nn.relu(conv2d(input, out_channels, kernel_size=kernel, stride=stride, pad="SAME", scope="con1_3X3",
                                trainable=trainable,
                                weight_initializer=get_weight(scope + '_con1_3X3_weights', weight_dict),
                                bias_initializer=get_weight(scope + '_con1_3X3_biases', weight_dict),
                                weight_initializer_type=_XAVIER()))
        net = conv2d(net, out_channels, kernel_size=kernel, stride=stride, pad="SAME", scope="conv2_3x3",
                     trainable=trainable,
                     weight_initializer=get_weight(scope + '_conv2_3x3_weights', weight_dict),
                     bias_initializer=get_weight(scope + '_conv2_3x3_biases', weight_dict),
                     weight_initializer_type=_XAVIER())
    return tf.add(tf.cast(net, tf.float32), tf.cast(input, tf.float32))


def keep_prob(dropout, train):
    """layer_util.py:124-131: dropout keep-probability, 1.0 at inference."""
    return tf.cond(train, lambda: float(dropout), lambda: 1.0)


def bias_variable(shape, bias_initializer=None, trainable=True):
    """layer_util.py:133-144: `biases`, constant 0.001 unless an initial value is given."""
    if bias_initializer is None:
        return tf.get_variable(name='biases', shape=shape, initializer=tf.constant_initializer(0.001),
                               trainable=trainable)
    return tf.get_variable(name='biases', initializer=bias_initializer, trainable=trainable)


def _weights_var(shape, weight_initializer, weight_initializer_type, trainable):
    if weight_initializer is None:
        return tf.get_variable(name='weights', shape=shape, initializer=weight_initializer_type or _RANDN002(),
                               dtype=tf.float32, trainable=trainable)
    return tf.get_variable(name='weights', initializer=weight_initializer, dtype=tf.float32, trainable=trainable)


def _check_same(pad):
    if pad != 'SAME':
        raise NotImplementedError("rendernet_b200 implements TF 'SAME' padding (all the reference ever uses)")


def conv2d(input_, num_outputs, kernel_size=[4, 4], stride=[1, 1], pad='SAME', if_bias=True, trainable=True,
           reuse=False, scope='conv2d', weight_initializer=None, bias_initializer=None,
           weight_initializer_type=None):
    """layer_util.py:147-184: tf.nn.conv2d SAME + `biases`.  Returns a deferred tensor."""
    _check_same(pad)
    if list(stride) != [1, 1]:
        raise NotImplementedError("conv2d stride != 1 is not on the hot path")
    cin = int(input_.shape[-1])
    with tf.variable_scope(scope, reuse=reuse):
        w = _weights_var(list(kernel_size) + [cin, int(num_outputs)], weight_initializer, weight_initializer_type,
                         trainable)
        b = None
        if if_bias:
            b = bias_variable([int(num_outputs)], trainable=trainable, bias_initializer=bias_initializer)
    return _deferred_conv("conv2d", input_, w, b, 1)


def conv2d_transpose(x, num_outputs, kernel_size=(4, 4), stride=(1, 1), pad='SAME', if_bias=True, reuse=False,
                     scope="conv2d_transpose", trainable=True, weight_initializer=None, bias_initializer=None,
                     weight_initializer_type=None):
    """layer_util.py:186-226: tf.nn.conv2d_transpose SAME, output = input*stride, filter [kh,kw,Cout,Cin]."""
    _check_same(pad)
    if stride[0] != stride[1]:
        raise NotImplementedError("anisotropic transposed-conv strides are not on the hot path")
    cin = int(x.shape[-1])
    with tf.variable_scope(scope, reuse=reuse):
        w = _weights_var(list(kernel_size) + [int(num_outputs), cin], weight_initializer, weight_initializer_type,
                         trainable)
        b = None
        if if_bias:
            b = bias_variable([int(num_outputs)], trainable=trainable, bias_initializer=bias_initializer)
    return _deferred_conv("conv2d_transpose", x, w, b, int(stride[0]))


def conv3d(input_, num_outputs, pad="SAME", reuse=False, kernel_size=[4, 4, 4], stride=[2, 2, 2], if_bias=True,
           trainable=True, scope="conv3d", weight_initializer=None, bias_initializer=None,
           weight_initializer_type=None):
    """layer_util.py:228-265: tf.nn.conv3d SAME + `biases`.
    Cin % 16 == 0 and stride 1 -> tensor-core implicit GEMM; the thin strided first layers (e_conv1: Cin 1,
    5^3 s2; e_conv2: Cin 8, 3^3 s(1,1,2)) -> CUDA-core direct kernel."""
    _check_same(pad)
    cin = int(input_.shape[-1])
    with tf.variable_scope(scope, reuse=reuse):
        w = _weights_var(list(kernel_size) + [cin, int(num_outputs)], weight_initializer, weight_initializer_type,
                         trainable)
        b = None
        if if_bias:
            b = bias_variable([int(num_outputs)], trainable=trainable, bias_initializer=bias_initializer)
    if list(stride) == [1, 1, 1] and cin % 16 == 0:
        return _deferred_conv("conv3d", input_, w, b, 1)
    if (USE_BANDED_CONV3D and list(kernel_size) == [3, 3, 3] and list(stride[:2]) == [1, 1] and stride[2] == 2
            and ops.BandedConv3d.eligible(cin, int(num_outputs), int(input_.shape[3]), 2)):
        return _deferred_conv("conv3d", input_, w, b, 2)        # e_conv2: z-strided, depth-folded onto the tensor pipe
    return _deferred_direct3d(input_, w, b, list(stride))


def conv3d_transpose(x, num_output, kernel_size=(4, 4), stride=(1, 1), pad='SAME', if_bias=True, reuse=False,
                     scope="conv3d_transpose", trainable=True, weight_initializer=None, bias_initializer=None,
                     weight_initializer_type=None):
    """layer_util.py:269-309: tf.nn.conv3d_transpose SAME, out = in*stride, filter [k,k,k,Cout,Cin] (texture
    decoder, BASELINE config 4; shape decoder).  Thin channels (<= 8) -> rn_conv3d_small; wider -> rn_conv3d_f32; fp32 storage."""
    _check_same(pad)
    if len(set(stride)) != 1 or len(set(kernel_size)) != 1:
        raise NotImplementedError("conv3d_transpose: cubic kernels / isotropic strides only")
    cin = int(x.shape[-1])
    with tf.variable_scope(scope, reuse=reuse):
        w = _weights_var(list(kernel_size) + [int(num_output), cin], weight_initializer, weight_initializer_type,
                         trainable)
        b = None
        if if_bias:
            b = bias_variable([int(num_output)], trainable=trainable, bias_initializer=bias_initializer)
    if max(cin, int(num_output)) > 8:
        return _deferred_f32_3d(x, w, b, int(stride[0]), True)
    return _deferred_small3d(x, w, b, int(stride[0]), True)


def fully_connected(input_, output_size, reuse=False, scope='fully_connected', if_bias=True, weight_initializer=None,
                    bias_initializer=None, trainable=True, weight_initializer_type=None):
    """layer_util.py:311-343: input_ @ weights[in,out] + biases (texture decoder, BASELINE config 4)."""
    xin = realize(input_)
    if not isinstance(xin, torch.Tensor):
        xin = torch.as_tensor(np.asarray(xin, np.float32))
    k_in = int(xin.shape[1])
    with tf.variable_scope(scope, reuse=reuse):
        if weight_initializer is None:
            matrix = tf.get_variable("weights", [k_in, int(output_size)],
                                     initializer=weight_initializer_type or _RANDN002(), dtype=tf.float32,
                                     trainable=trainable)
        else:
            matrix = tf.get_variable("weights", initializer=weight_initializer, dtype=tf.float32, trainable=trainable)
        b = None
        if if_bias:
            b = bias_variable([int(output_size)], bias_initializer, trainable=trainable)

    def run(act, alpha, residual, want32):
        xt = xin.to(device=_store().device, dtype=torch.float32).contiguous()
        wd = _dev_f32(matrix)
        if act not in (None, "prelu") or residual is not None:
            raise NotImplementedError("fully_connected: only a fused PReLU epilogue is supported")
        if _keeps_preact(act, alpha):
            z = ops.fully_connected(xt, wd, _dev_vec(b) if b is not None else None, None, want32=True)
            y = _prelu_f32(z, alpha)
            _record(op="fc", x=xt, w=matrix, b=b, act=act, alpha=alpha, y=y, rerun=lambda: z)
            return y
        y = ops.fully_connected(xt, wd, _dev_vec(b) if b is not None else None,
                                _alpha_arg(alpha, None) if act == "prelu" else None, want32=True)
        _record(op="fc", x=xt, w=matrix, b=b, act=act, alpha=alpha, y=y,
                rerun=lambda: ops.fully_connected(xt, wd, _dev_vec(b) if b is not None else None, None, want32=True))
        return y

    return Deferred(run, (xin.shape[0], int(matrix.shape[1])), torch.float32)   # an initializer's width wins (:337)


# ------------------------------------------------------------------------------------------ slim look-alikes
def slim_conv2d(inputs, num_outputs, kernel_size, stride=1, padding='SAME', activation_fn=None, scope=None, **_):
    """slim.conv2d as the reference calls it (activation_fn=None, SAME, xavier weights, zero `biases`;
    default scope 'Conv', layer_util.py:21,101-104; RenderNet_Shader.py:83,87,98,102)."""
    _check_same(padding)
    if activation_fn is not None:
        raise NotImplementedError("the reference always passes activation_fn=None")
    ks = [kernel_size] * 2 if isinstance(kernel_size, int) else list(kernel_size)
    st = [stride] * 2 if isinstance(stride, int) else list(stride)
    if st != [1, 1]:
        raise NotImplementedError("slim.conv2d stride != 1 is not on the hot path")
    cin = int(inputs.shape[-1])
    with tf.variable_scope(scope or 'Conv'):
        w = tf.get_variable('weights', ks + [cin, int(num_outputs)], initializer=_XAVIER())
        b = tf.get_variable('biases', [int(num_outputs)], initializer=tf.constant_initializer(0.0))
    return _deferred_conv("conv2d", inputs, w, b, 1)


def slim_conv2d_transpose(inputs, num_outputs, kernel_size, stride=1, padding='SAME', activation_fn=None,
                          scope=None, **_):
    """slim.conv2d_transpose (RenderNet_Shader.py:106-129); default scope 'Conv2d_transpose'."""
    _check_same(padding)
    if activation_fn is not None:
        raise NotImplementedError("the reference always passes activation_fn=None")
    ks = [kernel_size] * 2 if isinstance(kernel_size, int) else list(kernel_size)
    st = [stride] * 2 if isinstance(stride, int) else list(stride)
    cin = int(inputs.shape[-1])
    with tf.variable_scope(scope or 'Conv2d_transpose'):
        w = tf.get_variable('weights', ks + [int(num_outputs), cin], initializer=_XAVIER())
        b = tf.get_variable('biases', [int(num_outputs)], initializer=tf.constant_initializer(0.0))
    return _deferred_conv("conv2d_transpose", inputs, w, b, int(st[0]))


class _Slim:
    conv2d = staticmethod(slim_conv2d)
    conv2d_transpose = staticmethod(slim_conv2d_transpose)


slim = _Slim()


# ------------------------------------------------------------------------------------------ deferred execution
def _deferred_conv(kind, x, w, b, stride):
    xin = x
    if kind == "conv2d_transpose":
        oshape = (x.shape[0], x.shape[1] * stride, x.shape[2] * stride, w.shape[-2])
    elif kind == "conv3d":          # `stride` = stride along D (1 or 2); x,y strides are 1
        oshape = tuple(x.shape[:3]) + (-(-x.shape[3] // stride), w.shape[-1])
    else:
        oshape = tuple(x.shape[:-1]) + (w.shape[-1],)

    def run(act, alpha, residual, want32):
        xt = _as16(xin)
        st = _store()
        if act == "prelu" and st.tape is not None and st.keep_preact and not isinstance(alpha, str) and not want32:
            # training step: the PReLU-slope gradient needs the pre-activation, so the layer is run without its fused PReLU, z is
            # kept on the tape and the activation becomes its own (cheap) pass -- instead of re-running the convolution later
            z = _run(xt, None, None, residual, False)
            y = ops.bias_act(z, None, _dev_vec(alpha), "prelu")
            _record(op="conv", kind=kind, stride=stride, x=xt, w=w, b=b, act=act, alpha=alpha, residual=residual, y=y,
                    rerun=lambda: z)
            return y
        y = _run(xt, act, alpha, residual, want32)
        _record(op="conv", kind=kind, stride=stride, x=xt, w=w, b=b, act=act, alpha=alpha, residual=residual, y=y,
                rerun=lambda: _run(xt, None, None, residual, False))      # the pre-activation z (PReLU slope gradient)
        return y

    def _run(xt, act, alpha, residual, want32):
        banded = (kind == "conv3d" and USE_BANDED_CONV3D and tuple(w.shape[:3]) == (3, 3, 3)
                  and ops.BandedConv3d.eligible(int(w.shape[3]), int(w.shape[4]), int(xt.shape[3]), stride))
        if kind == "conv3d" and stride != 1 and not banded:
            raise NotImplementedError("z-strided conv3d needs the depth-folded path")
        xfold = 1
        if (kind == "conv2d_transpose" and USE_XFOLD and stride == 1 and residual is None
                and tuple(w.shape[:2]) == (4, 4)):
            xfold = ops.XFoldConvT.factor(int(w.shape[3]), int(xt.shape[2]))
        merged = (kind == "conv2d_transpose" and USE_MERGED_TCONV and stride == 2 and residual is None
                  and tuple(w.shape[:2]) == (4, 4) and ops.MergedConvT2.eligible(int(w.shape[3]), int(w.shape[2])))
        L = None if (banded or xfold > 1 or merged) else _packed(w, b, kind, stride)
        a = None if (xfold > 1 or merged) else _alpha_arg(alpha, ops.round_up(int(w.shape[-1]), 16) if banded else L.cout_pad)
        want16 = not want32
        if kind == "conv2d":
            return ops.conv2d(xt, L, act=act, residual=residual, want16=want16, want32=want32, alpha=a)
        if kind == "conv3d":
            if banded:
                Lb = _store().packed.get(("banded", w._rn_name, stride, _store().fmt))
                if Lb is None:
                    Lb = ops.BandedConv3d(w, b, dtype=tf.COMPUTE_DTYPE, device=_store().device, sz=stride, fmt=_store().fmt)
                    _store().packed[("banded", w._rn_name, stride, _store().fmt)] = Lb
                return ops.conv3d_banded(xt, Lb, act=act, residual=residual, alpha=a,
                                         alpha_tag=getattr(alpha, "_rn_name", None), want16=want16, want32=want32)
            return ops.conv3d(xt, L, act=act, residual=residual, want16=want16, want32=want32, alpha=a)
        if merged:
            Lm = _store().packed.get(("merged", w._rn_name, _store().fmt))
            if Lm is None:
                Lm = ops.MergedConvT2(w, b, dtype=tf.COMPUTE_DTYPE, device=_store().device, fmt=_store().fmt)
                _store().packed[("merged", w._rn_name, _store().fmt)] = Lm
            al = None
            if act == "prelu":
                al = _dev_vec(alpha) if not isinstance(alpha, str) else torch.zeros(int(w.shape[2]), device=xt.device)
            return ops.conv2d_transpose_s2_merged(xt, Lm, act=act, alpha=al, alpha_tag=getattr(alpha, "_rn_name", None),
                                                  want16=want16, want32=want32)
        if xfold > 1:
            F = xfold
            Lx = _store().packed.get(("xfold", w._rn_name, F, _store().fmt))
            if Lx is None:
                Lx = ops.XFoldConvT(w, b, F, dtype=tf.COMPUTE_DTYPE, device=_store().device, fmt=_store().fmt)
                _store().packed[("xfold", w._rn_name, F, _store().fmt)] = Lx
            al = None
            if act == "prelu":
                al = _dev_vec(alpha) if not isinstance(alpha, str) else torch.zeros(int(w.shape[2]), device=xt.device)
            ph = _store().phong
            if ph is not None and act == "sigmoid" and want32 and Lx.cout == 3:
                # "encoder/output" with the demo's Phong composite + uint8 quantisation applied in the same epilogue
                shaded, _store().phong_u8 = ops.conv2d_transpose_xfold(xt, Lx, act=act, want16=False, want32=True, phong=ph)
                return shaded
            return ops.conv2d_transpose_xfold(xt, Lx, act=act, alpha=al, alpha_tag=getattr(alpha, "_rn_name", None),
                                              want16=want16, want32=want32)
        if residual is not None:
            y = ops.conv2d_transpose(xt, L, act=act, alpha=a)
            return ops.bias_act(y, None, None, None, residual=residual, want32=want32)
        return ops.conv2d_transpose(xt, L, act=act, want16=want16, want32=want32, alpha=a)

    return Deferred(run, oshape, tf.COMPUTE_DTYPE)


def _dev_f32(v: torch.Tensor) -> torch.Tensor:
    st = _store()
    key = ("w32", getattr(v, "_rn_name", id(v)))
    d = st.packed.get(key)
    if d is None:
        d = v.to(device=st.device, dtype=torch.float32).contiguous()
        st.packed[key] = d
    return d


def _deferred_small3d(x, w, b, stride, transposed):
    """Thin-channel conv3d / conv3d_transpose (rn_conv3d_small), fp32 storage."""
    xin = x
    cout = int(w.shape[3] if transposed else w.shape[4])
    if transposed:
        oshape = (x.shape[0], x.shape[1] * stride, x.shape[2] * stride, x.shape[3] * stride, cout)
    else:
        oshape = (x.shape[0], -(-x.shape[1] // stride), -(-x.shape[2] // stride), -(-x.shape[3] // stride), cout)

    def run(act, alpha, residual, want32):
        xt = realize(xin)
        if not xt.is_cuda:
            xt = xt.to(_store().device)
        xt = xt.contiguous()
        if act not in (None, "prelu") or residual is not None:
            raise NotImplementedError("thin conv3d: only a fused PReLU epilogue is supported")
        if _keeps_preact(act, alpha):
            z = ops.conv3d_small(xt, _dev_f32(w), _dev_vec(b) if b is not None else None, None, stride, transposed, want32=True)
            y = _prelu_f32(z, alpha)
            _record(op="conv_small", transposed=transposed, stride=stride, x=xt, w=w, b=b, act=act, alpha=alpha, y=y,
                    rerun=lambda: z)
            return y
        y = ops.conv3d_small(xt, _dev_f32(w), _dev_vec(b) if b is not None else None,
                             _alpha_arg(alpha, cout) if act == "prelu" else None, stride, transposed, want32=True)
        _record(op="conv_small", transposed=transposed, stride=stride, x=xt, w=w, b=b, act=act, alpha=alpha, y=y,
                rerun=lambda: ops.conv3d_small(xt, _dev_f32(w), _dev_vec(b) if b is not None else None, None, stride,
                                               transposed, want32=True))     # the pre-activation z
        return y

    return Deferred(run, oshape, torch.float32)


def _deferred_f32_3d(x, w, b, stride, transposed):
    """conv3d / conv3d_transpose with more than 8 channels and a 4^3 kernel (the shape decoder, Reconstruct_RenderNet_Face.py:31-75):
    rn_conv3d_f32, fp32 storage, + bias + a fused tf.nn.elu / tf.nn.sigmoid."""
    xin = x
    cout = int(w.shape[3] if transposed else w.shape[4])
    if tuple(int(v) for v in w.shape[:3]) != (4, 4, 4):
        raise NotImplementedError(f"conv3d with {tuple(w.shape)} filters has no kernel (k = 4 only above 8 channels)")
    if transposed:
        oshape = (x.shape[0], x.shape[1] * stride, x.shape[2] * stride, x.shape[3] * stride, cout)
    else:
        oshape = (x.shape[0], -(-x.shape[1] // stride), -(-x.shape[2] // stride), -(-x.shape[3] // stride), cout)

    def run(act, alpha, residual, want32):
        if act not in (None, "elu", "sigmoid") or residual is not None:
            raise NotImplementedError("fp32 conv3d: only a fused tf.nn.elu / tf.nn.sigmoid epilogue is supported")
        xt = realize(xin)
        if not isinstance(xt, torch.Tensor):
            xt = torch.as_tensor(np.asarray(xt, np.float32))
        xt = xt.to(device=_store().device, dtype=torch.float32).contiguous()
        y = ops.conv3d_f32(xt, _dev_f32(w), _dev_vec(b) if b is not None else None, stride, transposed, act)
        _record(op="conv_f32", transposed=transposed, stride=stride, x=xt, w=w, b=b, act=act, alpha=None, y=y)
        return y

    return Deferred(run, oshape, torch.float32)


_DIRECT3D = {(1, 8, 5): True, (5, 8, 5): True, (2, 8, 3): True, (8, 16, 3): False, (8, 8, 3): False}  # needs fp32 input?


def _deferred_direct3d(x, w, b, stride):
    key = (int(w.shape[3]), int(w.shape[4]), int(w.shape[0]))
    if key not in _DIRECT3D:
        if len(set(stride)) != 1:
            raise NotImplementedError(f"conv3d {key} with stride {stride} has no kernel")
        if max(key[0], key[1]) > 8:
            return _deferred_f32_3d(x, w, b, int(stride[0]), False)
        return _deferred_small3d(x, w, b, int(stride[0]), False)
    xin = x
    oshape = (x.shape[0], -(-x.shape[1] // stride[0]), -(-x.shape[2] // stride[1]), -(-x.shape[3] // stride[2]),
              w.shape[-1])

    def run(act, alpha, residual, want32):
        cout = w.shape[-1]
        wd = _store().packed.get(("w32", w._rn_name))
        if wd is None:
            wd = w.to(_store().device).contiguous()
            _store().packed[("w32", w._rn_name)] = wd
        # a CroppedGrid (training on patches) runs the same fused kernels on its window; the record keeps the whole grid and
        # the window, so one tape format serves both
        grid, window = (xin.grid, xin.window) if isinstance(xin, CroppedGrid) else (xin, None)
        if (USE_FUSED_RESAMPLE_CONV1 and isinstance(grid, ResampledGrid) and grid.transform and xin._value is None
                and key == (1, 8, 5) and list(stride) == [2, 2, 2] and grid.new_size % 16 == 0
                and act in (None, "prelu") and residual is None and not want32):
            # resample + axis transform + e_conv1 + bias + PReLU in one kernel; the 128^3 grid is never written
            bd = _dev_vec(b) if b is not None else torch.zeros(cout, device=wd.device, dtype=torch.float32)
            ad = _alpha_arg(alpha, cout) if act == "prelu" else None
            if act == "prelu" and _store().tape is not None and _store().keep_preact and not isinstance(alpha, str):
                z = ops.resample_conv1(grid.voxel, grid.minv, grid.new_size, wd, bd, None, tf.COMPUTE_DTYPE, fmt=_store().fmt,
                                       window=window)
                y = ops.bias_act(z, None, _dev_vec(alpha), "prelu")         # training step: keep z (see _deferred_conv.run)
                _record(op="resample_conv1", grid=grid, window=window, w=w, b=b, act=act, alpha=alpha, stride=list(stride), y=y,
                        rerun=lambda: z)
                return y
            y = ops.resample_conv1(grid.voxel, grid.minv, grid.new_size, wd, bd, ad, tf.COMPUTE_DTYPE, fmt=_store().fmt,
                                   window=window)
            _record(op="resample_conv1", grid=grid, window=window, w=w, b=b, act=act, alpha=alpha, stride=list(stride), y=y,
                    rerun=lambda: ops.resample_conv1(grid.voxel, grid.minv, grid.new_size, wd, bd, None, tf.COMPUTE_DTYPE,
                                                     fmt=_store().fmt, window=window))
            return y
        if (USE_FUSED_RESAMPLE_CONV1 and isinstance(grid, ConcatResampledGrid) and grid.transform and xin._value is None
                and key == (5, 8, 5) and list(stride) == [2, 2, 2] and grid.new_size % 16 == 0
                and act in (None, "prelu") and residual is None and not want32):
            # Texture net: resample (C=1) + resample (C=4) + concat + e_conv1 + bias + PReLU in one kernel
            bd = _dev_vec(b) if b is not None else torch.zeros(cout, device=wd.device, dtype=torch.float32)
            ad = _alpha_arg(alpha, cout) if act == "prelu" else None

            def z5():
                return ops.resample5_conv1(grid.geom.voxel, grid.tex.voxel, grid.minv, grid.new_size, wd, bd, None,
                                           tf.COMPUTE_DTYPE, fmt=_store().fmt, window=window)
            if act == "prelu" and _store().tape is not None and _store().keep_preact and not isinstance(alpha, str):
                z = z5()
                y = ops.bias_act(z, None, _dev_vec(alpha), "prelu")         # training step: keep z (see _deferred_conv.run)
                _record(op="resample5_conv1", grid=grid, window=window, w=w, b=b, act=act, alpha=alpha, stride=list(stride),
                        y=y, rerun=lambda: z)
                return y
            y = ops.resample5_conv1(grid.geom.voxel, grid.tex.voxel, grid.minv, grid.new_size, wd, bd, ad, tf.COMPUTE_DTYPE,
                                    fmt=_store().fmt, window=window)
            _record(op="resample5_conv1", grid=grid, window=window, w=w, b=b, act=act, alpha=alpha, stride=list(stride), y=y,
                    rerun=z5)
            return y
        xt = realize(xin)
        if not xt.is_cuda:
            xt = xt.to(_store().device)
        bd = _dev_vec(b) if b is not None else torch.zeros(cout, device=xt.device, dtype=torch.float32)
        if _store().tape is not None:
            raise NotImplementedError("backward tape: the thin direct conv3d is only differentiated in its fused "
                                      "resample + e_conv1 form (Shader path)")
        if act == "prelu":
            ad = _alpha_arg(alpha, cout)
            y = ops.conv3d_direct(xt if isinstance(xt, ops.Split16) else xt.contiguous(), wd, bd, ad, stride, tf.COMPUTE_DTYPE, fmt=_store().fmt)
            act = None
        else:
            y = ops.conv3d_direct(xt if isinstance(xt, ops.Split16) else xt.contiguous(), wd, bd, None, stride, tf.COMPUTE_DTYPE, fmt=_store().fmt)
        if act is not None or residual is not None or want32:
            return ops.bias_act(y, None, None, act, residual=residual, want32=want32)
        return y

    return Deferred(run, oshape, tf.COMPUTE_DTYPE)
