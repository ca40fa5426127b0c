"""Mirror of the forward model functions of the reference's Reconstruct_RenderNet_Face.py that the drop-in boundary lists
(SURVEY §8b): `texture_decoder_pretrained(z_in, weight_dict)` (:77-111) and `RenderNet_pretrained(models_in, weight_dict,
prob=1.0, trainable=False)` (:113-302) -- the texture decoder and the Texture/Normal RenderNet built from a dictionary of
pretrained arrays in the npz-directory key convention of tools/model_util.py:26-39 ("e_conv1_e_conv1_weights",
"res2_4_con1_3X3_biases", "Image_e_conv6_1_alpha", "e_tex_dc1_g_gc1_weights", ...).

It differs from RenderNet_Texture_Face_Normal.RenderNet in exactly the ways the reference's does:
  * the projection unit is written out as reshape + 1x1 `conv2d` under scope `e_conv4` (:168-179);
  * the residual blocks take the `weight_dict` branch of layer_util.res_block_2d/3d, i.e. ReLU instead of PReLU
    (tools/layer_util.py:76,109);
  * head scopes are regular (`Image/e_conv7_1/e_conv7_1`, ...), the last up-convs are `e_conv11_1` and `e_conv11/e_conv11_2`.
`decoder_3d_pretrained(z_in, weight_dict)` (:31-75) mirrors the pretrained shape decoder (200-d latent -> 64^3 voxels, fp32
kernels rn_fully_connected + rn_conv3d_f32 in both precision modes).

`rendernet_b200.backward.TextureInputGradients(model="pretrained")` differentiates the rendering path with respect to the voxels,
the texture vector and the pose, `backward.ShapeDecoderGradients` the shape decoder with respect to its latent, and
`reconstruction_gradients` adds the reconstruction objective (Phong-shaded albedo vs the target, :358-383) and its light-azimuth
gradient.  `FaceReconstruction` puts them together into the reference's optimisation (:335-537): `step` is one inner step
(:402-412, plain gradient descent on the latent, pose, texture and light azimuth), `run` the outer loop over pose hypotheses
(`reconstruction_loop`, :455-537, with `create_param_center`, :304-318).  Deliberate differences: the first epoch's texture
vectors come from a seeded generator (the reference calls the unseeded np.random.randn), and the reference's PNG / binvox / npz
dumps (:497-519, :535) are replaced by a callback that receives the state after every step; `FaceReconstruction.render(state)`
produces the images those dumps show (shading, normal map, shaded prediction, voxels), also from other views and lights.
"""
from __future__ import annotations

import math
from typing import Callable, Dict, Optional

import numpy as np
import torch

from . import ops
from . import tfcompat as tf
from .layer_util import (conv2d, conv2d_transpose, conv3d, conv3d_transpose, fully_connected, prelu, res_block_2d,
                         res_block_3d)
from .tfcompat import realize


# The shape decoder's 12 variables: (TF name, npz key = the TF name with '/' -> '_', shape or None where the array decides it --
# the FC's width, as in the reference).  nn.ShapeDecoder's parameters are keyed by the TF name, its decoder_weight_dict() by the
# npz key.
DECODER_VARIABLES = (
    ("g_zP/g_gc1/weights", "g_zP_g_gc1_weights", None), ("g_zP/g_gc1/biases", "g_zP_g_gc1_biases", None),
    ("g_conv1/g_conv1/weights", "g_conv1_g_conv1_weights", (4, 4, 4, 128, 256)),
    ("g_conv1/g_conv1/biases", "g_conv1_g_conv1_biases", (128,)),
    ("g_conv2/g_conv2/weights", "g_conv2_g_conv2_weights", (4, 4, 4, 64, 128)),
    ("g_conv2/g_conv2/biases", "g_conv2_g_conv2_biases", (64,)),
    ("g_conv3/g_conv3/weights", "g_conv3_g_conv3_weights", (4, 4, 4, 32, 64)),
    ("g_conv3/g_conv3/biases", "g_conv3_g_conv3_biases", (32,)),
    ("g_conv4/g_conv4/weights", "g_conv4_g_conv4_weights", (4, 4, 4, 16, 32)),
    ("g_conv4/g_conv4/biases", "g_conv4_g_conv4_biases", (16,)),
    ("g_conv5/weights", "g_conv5_weights", (4, 4, 4, 1, 16)), ("g_conv5/biases", "g_conv5_biases", (1,)),
)


def decoder_3d_pretrained(z_in, weight_dict, trainable=False):
    """:31-75: latent [B,200] -> voxels [B,64,64,64,1] fp32 on the device: FC 200 -> 4^3 x 256, then conv3d_transpose k4 s2 + ELU
    down to 64^3 x 16 and conv3d_transpose k4 s1 + sigmoid.  Variable scopes and npz keys are the reference's ("g_zP_g_gc1_weights",
    "g_conv1_g_conv1_biases", ..., "g_conv5_weights"; DECODER_VARIABLES); a missing key raises KeyError.  As in
    texture_decoder_pretrained, the FC's width comes from its array.

    `trainable` (the reference's flag "used in fine-tuning") is accepted and changes nothing here: the variables are always the
    current store's fp32 masters (an existing variable wins over the array, like a restored checkpoint), and their gradients come
    from the reverse walk over the recorded layers -- backward.ShapeDecoderGradients.backward(want_weight_grads=True), or
    nn.ShapeDecoder(trainable=True) under torch autograd."""
    wd = weight_dict
    batch_size = z_in.shape[0]
    with tf.variable_scope('g_zP'):
        zP = fully_connected(z_in, 4 * 4 * 4 * 256, scope='g_gc1', trainable=trainable,
                             weight_initializer=wd["g_zP_g_gc1_weights"], bias_initializer=wd["g_zP_g_gc1_biases"])
        zP = realize(zP)
        zCon = zP.reshape(batch_size, 4, 4, 4, int(zP.shape[1]) // 64)
    net = zCon
    for i, ch in ((1, 128), (2, 64), (3, 32), (4, 16)):
        name = f"g_conv{i}"
        with tf.variable_scope(name):
            net = tf.nn.elu(conv3d_transpose(net, ch, kernel_size=[4, 4, 4], stride=[2, 2, 2], pad="SAME", scope=name,
                                             trainable=trainable, weight_initializer=wd[f"{name}_{name}_weights"],
                                             bias_initializer=wd[f"{name}_{name}_biases"]))
    gen5 = tf.nn.sigmoid(conv3d_transpose(net, 1, kernel_size=[4, 4, 4], stride=[1, 1, 1], pad="SAME", scope='g_conv5',
                                          trainable=trainable, weight_initializer=wd["g_conv5_weights"],
                                          bias_initializer=wd["g_conv5_biases"]), name="output")
    return realize(gen5)


def texture_decoder_pretrained(z_in, weight_dict, trainable=False):
    """:77-111: texture vector [B,199] -> 3-D texture volume [B,64,64,64,4] from npz-keyed arrays.  As in the reference, the
    FC's `4*4*4*512` width argument is ignored: with an initializer the variable (and the output) takes the array's width."""
    wd = weight_dict
    with tf.variable_scope("texture_encoder"):
        batch_size = z_in.shape[0]
        with tf.variable_scope('e_tex_dc1'):
            zP = prelu(fully_connected(z_in, 4 * 4 * 4 * 512, scope='g_gc1', trainable=trainable,
                                       weight_initializer=wd["e_tex_dc1_g_gc1_weights"],
                                       bias_initializer=wd["e_tex_dc1_g_gc1_biases"]), alpha=wd["e_tex_dc1_alpha"], trainable=trainable)
            z_resize = realize(zP).reshape(batch_size, 32, 32, 32, 4)
        layers = (("e_tex_conv0", "conv2d_transpose", 4, 1, True), ("e_tex_conv1", "conv2d_transpose", 8, 2, True),
                  ("e_tex_conv2", "conv3d", 4, 1, False))
        net = z_resize
        for name, key, ch, s, transposed in layers:
            with tf.variable_scope(name):
                kw = dict(kernel_size=[4, 4, 4], stride=[s, s, s], trainable=trainable,
                          weight_initializer=wd[f"{name}_{key}_weights"], bias_initializer=wd[f"{name}_{key}_biases"])
                net = prelu((conv3d_transpose if transposed else conv3d)(net, ch, **kw), alpha=wd[name + "_alpha"],
                            trainable=trainable)
        return net


def RenderNet_pretrained(models_in, weight_dict, prob=1.0, trainable=False):
    """models_in: rotated + axis-transformed 5-channel grid [B,H,W,128,5] (geometry + 4 texture channels; the reference's
    docstring says 64^3 x 6, its graph feeds the 128^3 x 5 concat of :360-378).  Returns (albedo, normal), float32 [B,4H,4W,3]."""
    if float(prob) != 1.0:
        raise NotImplementedError("inference path: dropout keep probability must be 1.0")
    wd = weight_dict

    def conv_args(key):
        return dict(trainable=trainable, weight_initializer=wd[key + "_weights"], bias_initializer=wd[key + "_biases"])

    with tf.variable_scope("encoder"):
        net = models_in
        for name, ch, k, stride in (("e_conv1", 8, 5, [2, 2, 2]), ("e_conv2", 16, 3, [1, 1, 2]), ("e_conv3", 16, 3, [1, 1, 1])):
            with tf.variable_scope(name):
                net = prelu(conv3d(net, ch, kernel_size=[k, k, k], stride=stride, pad="SAME", scope=name,
                                   **conv_args(f"{name}_{name}")), alpha=wd[name + "_alpha"], trainable=trainable)
        shortcut = net
        for i in range(1, 11):
            net = res_block_3d(net, 16, scope='res1_%d' % i, weight_dict=wd, trainable=trainable)
        with tf.variable_scope('res1_skip'):
            skip = conv3d(net, 16, kernel_size=[3, 3, 3], stride=[1, 1, 1], pad="SAME", scope="con1_3X3",
                          **conv_args("res1_skip_con1_3X3"))
            enc3_skip = realize(tf.add(tf.cast(skip, tf.float32), tf.cast(shortcut, tf.float32)))

        # collapse the depth axis (free in channel-last) and mix it with a 1x1 convolution (:168-179)
        B, H, W, D, C = enc3_skip.shape
        enc3_2d = enc3_skip.reshape(B, H, W, D * C)
        with tf.variable_scope('e_conv4'):
            net = prelu(conv2d(enc3_2d, num_outputs=D * C, kernel_size=[1, 1], scope='e_conv4', **conv_args("e_conv4_e_conv4")),
                        alpha=wd["e_conv4_alpha"], trainable=trainable)

        for stage, width, nblocks, nxt, nxt_ch in (("res2", 32 * 16, 10, "e_conv5", 32 * 8), ("res3", 32 * 8, 5, None, 0)):
            shortcut = net
            for i in range(1, nblocks + 1):
                net = res_block_2d(net, width, scope='%s_%d' % (stage, i), weight_dict=wd, trainable=trainable)
            with tf.variable_scope(stage + '_skip'):
                skip = conv2d(net, width, kernel_size=[3, 3], scope="con1_3X3", **conv_args(stage + "_skip_con1_3X3"))
                net = tf.add(tf.cast(skip, tf.float32), tf.cast(shortcut, tf.float32))
            if nxt is not None:
                with tf.variable_scope(nxt):
                    net = prelu(conv2d(net, nxt_ch, kernel_size=[4, 4], scope=nxt, **conv_args(f"{nxt}_{nxt}")),
                                alpha=wd[nxt + "_alpha"], trainable=trainable)
        enc5_skip = realize(net)                           # consumed by both heads

        outs = []
        for head, sfx, last_outer in (("Image", "1", "e_conv11_1"), ("Normal", "2", "e_conv11")):
            with tf.variable_scope(head):
                name = "e_conv6_" + sfx
                with tf.variable_scope(name):
                    net = prelu(conv2d(enc5_skip, 32 * 4, kernel_size=[4, 4], scope=name, **conv_args(f"{head}_{name}_{name}")),
                                alpha=wd[f"{head}_{name}_alpha"], trainable=trainable)
                for blk, ch in (("7", 32 * 2), ("8", 32), ("9", 16)):
                    name = "e_conv%s_%s" % (blk, sfx)
                    with tf.variable_scope(name):
                        net = prelu(conv2d_transpose(net, ch, [4, 4], stride=[2, 2], scope=name,
                                                     **conv_args(f"{head}_{name}_{name}")),
                                    alpha=wd[f"{head}_{name}_alpha"], trainable=trainable)
                name = "e_conv11_" + sfx
                with tf.variable_scope(last_outer):
                    net = tf.nn.sigmoid(conv2d_transpose(net, 3, [4, 4], stride=[1, 1], scope=name,
                                                         **conv_args(f"{head}_{name}_{name}")), name="encoder_output")
            outs.append(realize(net))
    return outs[0], outs[1]


def pretrained_dict_from_texture_weights(W):
    """Re-key a Texture/Normal weight dict in TF variable naming (RenderNet_Texture_Face_Normal scopes, e.g. the oracle's
    `init_texture_weights`) into the npz-directory keys `RenderNet_pretrained` and `texture_decoder_pretrained` read.  Both functions then compute the same
    network provided the residual-block alphas are zero (the weight_dict branch uses ReLU).  Test / migration helper."""
    out = {}
    te = "texture_encoder/"
    for src, dst in (("e_tex_fc1/fully_connected", "e_tex_dc1_g_gc1"), ("e_tex_fc1/alpha", "e_tex_dc1_alpha"),
                     ("e_tex_conv0/conv3d_transpose", "e_tex_conv0_conv2d_transpose"), ("e_tex_conv0/alpha", "e_tex_conv0_alpha"),
                     ("e_tex_conv1/conv3d_transpose", "e_tex_conv1_conv2d_transpose"), ("e_tex_conv1/alpha", "e_tex_conv1_alpha"),
                     ("e_tex_conv2/conv3d", "e_tex_conv2_conv3d"), ("e_tex_conv2/alpha", "e_tex_conv2_alpha")):
        if src.endswith("/alpha"):
            if te + src in W:
                out[dst] = W[te + src]
            continue
        for part in ("weights", "biases"):
            if f"{te}{src}/{part}" in W:
                out[f"{dst}_{part}"] = W[f"{te}{src}/{part}"]
    ren = {"projection_unit/Conv": "e_conv4/e_conv4", "projection_unit/alpha": "e_conv4/alpha",
           "Image/e_conv7_1/e_conv7_2": "Image/e_conv7_1/e_conv7_1", "Image/e_conv8_1/conv2d_transpose": "Image/e_conv8_1/e_conv8_1",
           "Image/e_conv9_1/conv2d_transpose": "Image/e_conv9_1/e_conv9_1",
           "Image/e_conv10_1/conv2d_transpose": "Image/e_conv11_1/e_conv11_1", "Normal/e_conv10_2/e_conv10_2": "Normal/e_conv11_2/e_conv11_2"}
    for k, v in W.items():
        if not k.startswith("encoder/"):
            continue
        name = k[len("encoder/"):]
        for a, b in ren.items():
            if name.startswith(a):
                name = b + name[len(a):]
                break
        out[name.replace("/", "_")] = v
    return out


def light_pos(light_azimuth, light_elevation) -> np.ndarray:
    """tools/Phong_shading.py:115-130 (tf_generate_light_pos) in float32: [B,1] azimuths (rad), one elevation (rad) -> [B,3]."""
    az = np.asarray(light_azimuth, np.float32).reshape(-1, 1)
    el = np.full_like(az, np.float32(light_elevation))
    return np.concatenate([np.sin(el) * np.cos(az), np.sin(el) * np.sin(az), np.cos(el)], 1).astype(np.float32)


def reconstruction_gradients(tig, voxels, texture, view_params, light_azimuth, target, light_elevation, ambient=0.,
                             k_diffuse=1., light_col=(1.0, 1.0, 1.0), dvox_on_device=False, want_shading_grad=False):
    """Loss and gradients of one reconstruction step (:358-412): compos = albedo * tf_phong_composite(normal, light(azimuth,
    elevation), light_col, ambient, k_diffuse, with_mask=True) (white background), loss[b] = mean (target - compos)^2.
    tig: a backward.TextureInputGradients of the batch size (model "pretrained" for the reference's network).  Returns
    (loss [B] float64, dL/dvoxels [B,64,64,64,1], dL/dtexture [B,199], dL/dview_params [B,3], dL/dlight_azimuth [B,1]); the
    objective and its image gradients run in rn_phong_recon_loss_grad, the azimuth map is differentiated on the host in float64.
    dvox_on_device: dL/dvoxels is returned as a CUDA tensor (what ShapeDecoderGradients.backward takes).  light_col: 1 or B rows
    of 3; ambient: a float or a [1|B] tensor.  want_shading_grad: two more results, dL/dlight_col [B,3] and dL/dambient [B]
    (float64, rn_phong_recon_loss_grad_params)."""
    albedo, normal = tig.forward(voxels, texture, view_params)
    dev = albedo.device
    B = albedo.shape[0]
    az = np.asarray(light_azimuth, np.float64).reshape(B, 1)
    ldir = torch.from_numpy(light_pos(az, light_elevation)).to(dev)
    lcol = torch.as_tensor(np.asarray(light_col, np.float32).reshape(-1, 3)).to(dev).expand(B, 3).contiguous()
    tgt = torch.as_tensor(np.asarray(target, np.float32) if not isinstance(target, torch.Tensor) else target)
    tgt = tgt.to(device=dev, dtype=torch.float32).reshape(tuple(albedo.shape)).contiguous()
    with torch.cuda.device(dev):
        out = ops.phong_recon_loss_grad(albedo, normal, tgt, ldir, lcol, ambient, k_diffuse, black_background=False,
                                        with_mask=True, **(dict(want_shading_grad=True) if want_shading_grad else {}))
        loss, d_albedo, d_normal, d_light = out[:4]
    dvox, dtex, dpose = tig.backward(d_albedo, d_normal, dvox_on_device=dvox_on_device)
    dl = d_light.double().cpu().numpy()
    el = float(np.float32(light_elevation))
    # d light / d azimuth = (-sin(el) sin(az), sin(el) cos(az), 0)
    dlaz = (dl[:, 0:1] * -np.sin(el) * np.sin(az) + dl[:, 1:2] * np.sin(el) * np.cos(az))
    if want_shading_grad:
        return loss.cpu().numpy(), dvox, dtex, dpose, dlaz, out[4].double().cpu().numpy(), out[5].double().cpu().numpy()
    return loss.cpu().numpy(), dvox, dtex, dpose, dlaz


# ------------------------------------------------------------------------------------------ the reconstruction (:304-537)
# step size of the light colour and the ambient term (FaceReconstruction(fit_shading=True)): not in the reference, not tuned
SHADING_ETA = 0.5
RECON_DEFAULTS = dict(shape_eta=0.8, pose_eta=0.01, tex_eta=0.8, light_eta=0.4, inner_step=200, max_epochs=10, z_dim=200,
                      target_azimuth_light=294.0, target_elevation_light=105.0)     # config_reconstruction_RenderNet.json


def create_param_center(phi_mid=90, phi_range=240, theta_mid=90, theta_range=120, batch_size=5):
    """:304-318: five pose hypotheses [azimuth, elevation, scale] (radians) at the corners and centre of a (phi, theta) window in
    degrees; theta is measured from the horizon (elevation = 90 - theta).  The reference fills exactly five rows and resets the
    scale to 1.0, so any other batch size is rejected."""
    if batch_size != 5:
        raise ValueError(f"create_param_center fills exactly 5 pose hypotheses; batch_size is {batch_size}")
    phi_min = ((phi_mid - phi_range * 0.5) % 360) * math.pi / 180.0
    phi_max = ((phi_mid + phi_range * 0.5) % 360) * math.pi / 180.0
    theta_min = (90 - (theta_mid - theta_range * 0.5)) * math.pi / 180.0
    theta_max = (90 - (theta_mid + theta_range * 0.5)) * math.pi / 180.0
    phi_mid = phi_mid * math.pi / 180.0
    theta_mid = (90 - theta_mid) * math.pi / 180.0
    params = np.zeros(shape=[batch_size, 3], dtype=np.float32)
    params[0] = np.array([phi_min, theta_min, 1.0], dtype=np.float32)
    params[1] = np.array([phi_min, theta_max, 1.0], dtype=np.float32)
    params[2] = np.array([phi_mid, theta_mid, 1.0], dtype=np.float32)
    params[3] = np.array([phi_max, theta_min, 1.0], dtype=np.float32)
    params[4] = np.array([phi_max, theta_max, 1.0], dtype=np.float32)
    return params


def reconstruction_loop(step_fn: Callable, loss_fn: Callable, target, batch_size: int = 5, z_dim: int = 200, max_epochs: int = 10,
                        inner_step: int = 200, seed: int = 0, callback: Optional[Callable] = None,
                        shading: Optional[dict] = None) -> Dict[str, object]:
    """The outer / inner loop of :455-537 over any step function.

    step_fn(state, target) -> (new_state, loss [B], grads): one inner step from `state` {"latent" [B,z_dim], "pose" [B,3] (radians),
    "texture" [B,199], "light" [B,1] (azimuth, radians)}; loss is evaluated at `state`.  loss_fn(state, target) -> loss [B] at a
    state: the reference re-evaluates the loss after the last inner step and keeps the argmin hypothesis (:522-534).

    Epoch 0 starts from five poses around (phi 270, theta 90) in a 60 x 30 degree window, latent 0.5, texture N(0, 1) from
    np.random.default_rng(seed) and light azimuths linspace(230, 320) degrees; every later epoch halves the window around the
    best pose (converted to [phi, 90 - theta, 1] degrees, :533-534) and restarts all five hypotheses from the best latent,
    texture and light.  callback(epoch, step, state, loss, selection_loss) runs after every step with the updated state;
    selection_loss is the re-evaluated loss [B] after the last inner step of an epoch, else None.

    Returns {"latent", "texture", "light", "pose" (radians, the selected hypothesis), "best_param" (the reference's degree
    form), "best_index", "best_loss" (per epoch), "state" (the last state)}.
    shading: the first epoch's {"light_col" [5,3], "ambient" [5]} or None; given, they join the state, later epochs restart from
    the selected hypothesis' values, and the result holds the selected "light_col" [3] and "ambient"."""
    if batch_size != 5:
        raise ValueError(f"the reconstruction loop runs 5 pose hypotheses (create_param_center); batch_size is {batch_size}")
    rng = np.random.default_rng(seed)
    best_param = np.zeros(shape=(3))
    best_vector = np.zeros(shape=(z_dim))
    best_tex = np.zeros(shape=(199))
    best_light = best_shading = None
    best_pose = best_index = None
    best_loss = []
    phi_range = 60
    theta_range = 30
    state = None
    for i in range(max_epochs):
        if i == 0:
            params_batch = create_param_center(phi_mid=270, phi_range=phi_range, theta_mid=90, theta_range=theta_range,
                                               batch_size=batch_size)
            vector_batch = np.ones((batch_size, z_dim)) * 0.5
            tex_batch = rng.standard_normal((batch_size, 199))
            light_batch = np.expand_dims((np.linspace(230, 320, num=5) * math.pi / 180.0), axis=0).T
        else:
            phi_range /= 2
            theta_range /= 2
            params_batch = create_param_center(phi_mid=best_param[0], phi_range=phi_range, theta_mid=best_param[1],
                                               theta_range=theta_range, batch_size=batch_size)
            vector_batch = np.tile(best_vector[np.newaxis, :], (batch_size, 1))
            tex_batch = np.tile(best_tex[np.newaxis, :], (batch_size, 1))
            light_batch = np.tile(best_light[np.newaxis, :], (batch_size, 1))
        # the assign ops of :481 store into float32 variables
        state = dict(latent=np.asarray(vector_batch, np.float32), pose=np.asarray(params_batch, np.float32),
                     texture=np.asarray(tex_batch, np.float32), light=np.asarray(light_batch, np.float32))
        if shading is not None:
            for k in ("light_col", "ambient"):
                state[k] = (np.asarray(shading[k], np.float32).copy() if i == 0 else
                            np.repeat(best_shading[k][np.newaxis], batch_size, 0))
        for idx in range(inner_step):
            state, loss, _ = step_fn(state, target)
            sel = None
            if idx == inner_step - 1:
                sel = np.asarray(loss_fn(state, target))
                j = int(np.argmin(sel))
                best_vector = state["latent"][j]
                best_tex = state["texture"][j]
                best_light = state["light"][j]
                if shading is not None:
                    best_shading = {k: np.asarray(state[k][j], np.float32).copy() for k in ("light_col", "ambient")}
                best_pose = state["pose"][j].copy()
                best_param = state["pose"][j] * 180. / math.pi
                best_param = np.array([best_param[0], 90 - best_param[1], 1])
                best_index = j
                best_loss.append(float(sel[j]))
            if callback is not None:
                callback(i, idx, state, loss, sel)
    out = dict(latent=best_vector, texture=best_tex, light=best_light, pose=best_pose, best_param=best_param,
               best_index=best_index, best_loss=best_loss, state=state)
    if shading is not None:
        out.update(best_shading)
    return out


class FaceReconstruction:
    """The reference's face reconstruction (Reconstruct_RenderNet_Face.py:335-537) on this package's kernels.

        rec = FaceReconstruction(weight_dict, weight_dict_decoder)          # npz-keyed RenderNet and shape-decoder weights
        target = rec.shaded_target(albedo, normal)                          # [5,512,512,3]
        out = rec.run(target)                                               # latent, texture, pose, light, voxels, ...

    The render network runs in `precision` ("exact" or "fast"); the shape and texture decoders run in fp32 in both modes.
    Defaults are those of config_reconstruction_RenderNet.json (RECON_DEFAULTS).

    fit_shading: the state also holds the light colour "light_col" [B,3] and the ambient term "ambient" [B], starting from the
    reference's white light and ambient 0; step descends them with shading_eta (SHADING_ETA: untuned, not in the reference) and
    projects them onto colour >= 0, 0 <= ambient <= 1; run returns the selected values and render shades with the state's.
    k_diffuse stays 1: the composite sees only k_diffuse * colour, which the fitted colour absorbs."""

    def __init__(self, weight_dict, weight_dict_decoder, batch: int = 5, precision: str = "exact", shape_eta: float = 0.8,
                 pose_eta: float = 0.01, tex_eta: float = 0.8, light_eta: float = 0.4, inner_step: int = 200,
                 max_epochs: int = 10, z_dim: int = 200, target_azimuth_light: float = 294.0,
                 target_elevation_light: float = 105.0, seed: int = 0, device: str = "cuda", fit_shading: bool = False,
                 shading_eta: float = SHADING_ETA):
        from .backward import ShapeDecoderGradients, TextureInputGradients
        self.B = int(batch)
        self.eta = dict(latent=float(shape_eta), pose=float(pose_eta), texture=float(tex_eta), light=float(light_eta))
        self.fit_shading = bool(fit_shading)
        if self.fit_shading:
            self.eta["shading"] = float(shading_eta)
        self.inner_step, self.max_epochs, self.z_dim, self.seed = int(inner_step), int(max_epochs), int(z_dim), int(seed)
        self.elevation = (90 - target_elevation_light) * math.pi / 180.0        # :330-331
        self.azimuth = target_azimuth_light * math.pi / 180.0
        self.tig = TextureInputGradients(weight_dict, self.B, precision=precision, model="pretrained", device=device)
        self.sdg = ShapeDecoderGradients(weight_dict_decoder, self.B, device=device)
        self.device = self.tig.device
        self._target = None

    def shaded_target(self, albedo, normal) -> np.ndarray:
        """:435-447: target albedo and normal map (images in [0,1], [512,512,3] or [1,512,512,3]) -> the Phong-shaded target under
        the ground-truth light (NumPy composite, white background, with mask), tiled to the batch.  float32 [B,512,512,3]."""
        from .Phong_shading import np_phong_composite
        target = np.asarray(albedo, np.float64).reshape((1, 512, 512, 3))
        target_normal = np.asarray(normal, np.float64).reshape((1, 512, 512, 3))
        el, az = self.elevation, self.azimuth
        light_dir = np.array([[np.sin(el) * np.cos(az), np.sin(el) * np.sin(az), np.cos(el)]])
        shading = np_phong_composite(target_normal, light_dir, np.array([[1.0, 1.0, 1.0]]), 0., 1.0, background_col="white",
                                     with_mask=True)
        return np.tile(np.multiply(target, shading), (self.B, 1, 1, 1)).astype(np.float32)

    def _target_dev(self, target):
        if isinstance(target, torch.Tensor):
            return target.to(device=self.device, dtype=torch.float32).contiguous()
        if self._target is None or self._target[0] is not target:
            self._target = (target, torch.as_tensor(np.asarray(target, np.float32)).to(self.device).contiguous())
        return self._target[1]

    def initial_shading(self) -> Optional[dict]:
        """The first epoch's {"light_col" [B,3], "ambient" [B]}: the reference's white light and ambient 0 (None without
        fit_shading)."""
        if not self.fit_shading:
            return None
        return dict(light_col=np.ones((self.B, 3), np.float32), ambient=np.zeros(self.B, np.float32))

    def _shading(self, state):
        """(light_col, ambient) at `state`: the reference's constants, or the state's with fit_shading."""
        if not self.fit_shading:
            return (1.0, 1.0, 1.0), 0.
        return (np.asarray(state["light_col"], np.float32),
                torch.as_tensor(np.asarray(state["ambient"], np.float32)).to(self.device))

    def gradients(self, state, target):
        """Loss [B] and the gradients of sum_b loss[b] (tf.gradients of the loss vector, :402) with respect to the latent [B,200],
        the pose [B,3], the texture [B,199] and the light azimuth [B,1], at `state`; with fit_shading also the light colour
        [B,3] and the ambient term [B]."""
        if self.fit_shading:
            vox = self.sdg.forward(state["latent"])
            lcol, amb = self._shading(state)
            loss, dvox, dtex, dpose, dlight, dcol, damb = reconstruction_gradients(
                self.tig, vox, state["texture"], state["pose"], state["light"], self._target_dev(target), self.elevation,
                ambient=amb, light_col=lcol, dvox_on_device=True, want_shading_grad=True)
            return loss, dict(latent=self.sdg.backward(dvox), pose=dpose, texture=dtex, light=dlight, light_col=dcol,
                              ambient=damb)
        vox = self.sdg.forward(state["latent"])
        loss, dvox, dtex, dpose, dlight = reconstruction_gradients(self.tig, vox, state["texture"], state["pose"], state["light"],
                                                                   self._target_dev(target), self.elevation, dvox_on_device=True)
        return loss, dict(latent=self.sdg.backward(dvox), pose=dpose, texture=dtex, light=dlight)

    def step(self, state, target):
        """One inner step (:402-412): the loss at `state`, its gradients, and plain gradient descent var -= eta * grad per
        variable group, in float32 like the reference's variables.  Returns (new_state, loss [B], grads)."""
        loss, grads = self.gradients(state, target)
        new = {k: (np.asarray(state[k], np.float32) - np.float32(self.eta[k]) * np.asarray(grads[k], np.float32)).astype(np.float32)
               for k in ("latent", "pose", "texture", "light")}
        if self.fit_shading:
            eta = np.float32(self.eta["shading"])
            new["light_col"] = np.maximum(np.asarray(state["light_col"], np.float32) -
                                          eta * np.asarray(grads["light_col"], np.float32), np.float32(0)).astype(np.float32)
            new["ambient"] = np.clip(np.asarray(state["ambient"], np.float32) - eta * np.asarray(grads["ambient"], np.float32),
                                     np.float32(0), np.float32(1)).astype(np.float32)
        return new, loss, grads

    def loss(self, state, target) -> np.ndarray:
        """The objective [B] at `state` (forward only)."""
        vox = self.sdg.forward(state["latent"])
        albedo, normal = self.tig.forward(vox, state["texture"], state["pose"])
        B = self.B
        az = np.asarray(state["light"], np.float64).reshape(B, 1)
        with torch.cuda.device(self.device):
            ldir = torch.from_numpy(light_pos(az, self.elevation)).to(self.device)
            if self.fit_shading:
                lc, amb = self._shading(state)
                lcol = torch.from_numpy(lc).to(self.device)
            else:
                lcol, amb = torch.ones((B, 3), device=self.device, dtype=torch.float32), 0.
            loss = ops.phong_recon_loss_grad(albedo, normal, self._target_dev(target), ldir, lcol, amb, 1.,
                                             black_background=False, with_mask=True)[0]
        return loss.cpu().numpy()

    def render(self, state, view_params=None, light_azimuth=None) -> Dict[str, np.ndarray]:
        """The images of a state (what :497-508 fetches every 100 steps): the shape decoder, the Texture+Normal network and the
        shading of :372-378 (rn_phong_shade, TensorFlow's composite, white background, mask, ambient 0, k_d 1, light colour 1),
        i.e. the very image the loss measures.  view_params [B,3] / light_azimuth [B,1] (radians) render the state's face from
        another pose or under another light; None keeps the state's own (with fit_shading the state's colour and ambient term
        shade it).  Returns NumPy albedo, normal, shading, compos
        (float32 [B,512,512,3]), compos_u8 (clip(255 compos) as uint8) and voxels ([B,64,64,64] float32)."""
        B = self.B
        pose = state["pose"] if view_params is None else view_params
        az = state["light"] if light_azimuth is None else light_azimuth
        pose = np.asarray(pose, np.float32).reshape(B, 3)
        az = np.asarray(az, np.float64).reshape(B, 1)
        vox = self.sdg.forward(state["latent"])
        albedo, normal = self.tig.forward(vox, state["texture"], pose)
        with torch.cuda.device(self.device):
            ldir = torch.from_numpy(light_pos(az, self.elevation)).to(self.device)
            lcol, amb = self._shading(state)
            shade, compos, u8 = ops.phong_shade(normal, ldir, lcol, amb, 1., albedo=albedo, composite="tf",
                                                background_white=True, with_mask=True)
        out = dict(albedo=albedo, normal=normal, shading=shade, compos=compos, compos_u8=u8, voxels=vox[..., 0])
        return {k: v.cpu().numpy() for k, v in out.items()}

    def run(self, target, callback: Optional[Callable] = None) -> Dict[str, object]:
        """The whole reconstruction (:455-537) from a shaded target [B,512,512,3]: reconstruction_loop with this object's step and
        loss.  Returns its dictionary plus "voxels" [64,64,64] (the decoded best latent) as NumPy."""
        more = dict(shading=self.initial_shading()) if self.fit_shading else {}
        out = reconstruction_loop(self.step, self.loss, target, batch_size=self.B, z_dim=self.z_dim, max_epochs=self.max_epochs,
                                  inner_step=self.inner_step, seed=self.seed, callback=callback, **more)
        vox = self.sdg.forward(np.tile(np.asarray(out["latent"], np.float32)[None], (self.B, 1)))
        out["voxels"] = vox[0, ..., 0].cpu().numpy()
        return out
