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
The optimisation loop itself (:335-537) is not mirrored.  `rendernet_b200.backward.TextureInputGradients(model="pretrained")`
differentiates this forward path with respect to the voxels, the texture vector and the pose, and `reconstruction_gradients`
adds the reconstruction objective (Phong-shaded albedo vs the target, :358-383) and its light-azimuth gradient: with it, the
reference's inner step (:402-412, plain gradient descent per variable group) is a few host lines.  The shape decoder
(`decoder_3d_pretrained`, :61-75) is not mirrored: callers get dL/dvoxels and chain their own.
"""
from __future__ import annotations

import numpy as np
import torch

from . import ops
from . import tfcompat as tf
from .layer_util import (conv2d, conv2d_transpose, conv3d, conv3d_transpose, fully_connected, prelu, res_block_2d,
                         res_block_3d)
from .tfcompat import realize


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
                             k_diffuse=1., light_col=(1.0, 1.0, 1.0)):
    """Loss and gradients of one reconstruction step (:358-412): compos = albedo * tf_phong_composite(normal, light(azimuth,
    elevation), light_col, ambient, k_diffuse, with_mask=True) (white background), loss[b] = mean (target - compos)^2.
    tig: a backward.TextureInputGradients of the batch size (model "pretrained" for the reference's network).  Returns
    (loss [B] float64, dL/dvoxels [B,64,64,64,1], dL/dtexture [B,199], dL/dview_params [B,3], dL/dlight_azimuth [B,1]); the
    objective and its image gradients run in rn_phong_recon_loss_grad, the azimuth map is differentiated on the host in float64."""
    albedo, normal = tig.forward(voxels, texture, view_params)
    dev = albedo.device
    B = albedo.shape[0]
    az = np.asarray(light_azimuth, np.float64).reshape(B, 1)
    ldir = torch.from_numpy(light_pos(az, light_elevation)).to(dev)
    lcol = torch.as_tensor(np.asarray(light_col, np.float32).reshape(-1, 3)).to(dev).expand(B, 3).contiguous()
    tgt = torch.as_tensor(np.asarray(target, np.float32) if not isinstance(target, torch.Tensor) else target)
    tgt = tgt.to(device=dev, dtype=torch.float32).reshape(tuple(albedo.shape)).contiguous()
    with torch.cuda.device(dev):
        loss, d_albedo, d_normal, d_light = ops.phong_recon_loss_grad(albedo, normal, tgt, ldir, lcol, ambient, k_diffuse,
                                                                      black_background=False, with_mask=True)
    dvox, dtex, dpose = tig.backward(d_albedo, d_normal)
    dl = d_light.double().cpu().numpy()
    el = float(np.float32(light_elevation))
    # d light / d azimuth = (-sin(el) sin(az), sin(el) cos(az), 0)
    dlaz = (dl[:, 0:1] * -np.sin(el) * np.sin(az) + dl[:, 1:2] * np.sin(el) * np.cos(az))
    return loss.cpu().numpy(), dvox, dtex, dpose, dlaz
