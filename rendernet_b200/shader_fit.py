"""Fit the view and the light of a known shape to an image through the Shader network: what a differentiable renderer is for.

The Shader network renders a voxel grid from a pose (azimuth, elevation, scale) as a normal map (RGB) or a greyscale contour
image.  Given a target image of a known shape, this module descends on the pose and, for the RGB network, on the light of the
demo's Phong composite (RenderNet_demo.py:54-58), with the reference's hypothesis search (Reconstruct_RenderNet_Face.py:455-537):

    fit = ShaderPoseFit(weights, voxels, objective="phong")        # voxels [64,64,64]: the known shape
    out = fit.run(target, init=dict(pose=compute_pose_param(250, 60, 3.3)[0]))
    out["pose"], out["light"], fit.render(out["state"])["shaded_u8"]

Objectives (`shader_fit_gradients`):
  * "phong": the network's normal map shaded by np_phong_composite under a light given as (azimuth, elevation) in radians,
    mapped as the demo's generate_light_pos (tools/Phong_shading.py:247-253): l = (-sin(el) cos(az), cos(el), -sin(el) sin(az));
    loss[b] = mean (target - shaded)^2 (rn_phong_composite_loss_grad, whose shading is rn_phong_composite's bit for bit);
  * "mse" / "bce": the raw network output (RGB or greyscale) against the target, per item (rn_image_loss_grad_items; "bce" is
    the loss the shipped greyscale Shader was trained with, RenderNet_Shader.py:158-163).
The image gradient runs back through the network and the resampler (backward.ShaderInputGradients) to dL/d(view_params); the
light map is differentiated on the host in float64.  The voxels are held fixed here: the Shader has no shape prior, so fitting
the shape takes several views and a silhouette hull (shape_fit.py).

Search (`pose_search`, the reference's loop with `create_param_center`): five pose hypotheses at the corners and the centre of a
60 x 30 degree (azimuth x elevation) window around the initial guess, light azimuths linspace(230, 320) degrees unless given;
`inner_step` descent steps; the loss is re-evaluated after the last one, the argmin kept and the window halved around it for the
next epoch.  Unlike the reference, the scale is the initial guess's (create_param_center writes 1.0) and is held fixed unless
`fit_scale`.

Shading (`fit_shading=True`, "phong" only): the light's colour [B,3] and the ambient term [B] join the state, starting from the
constructor's constants (PHONG_DEFAULTS), descend with their own eta and are projected onto colour >= 0 and 0 <= ambient <= 1
after every step.  k_diffuse stays a constant: the composite sees only k_diffuse * colour, and the fitted colour absorbs it.
"""
from __future__ import annotations

import argparse
import json
import math
import os
from typing import Callable, Dict, Optional

import numpy as np
import torch

from . import ops
from .Reconstruct_RenderNet_Face import create_param_center

OBJECTIVES = ("phong", "mse", "bce")
# the demo's shading (RenderNet_demo.py:18-20): ambient 0.1, k_diffuse 0.9, white light, black background with the soft mask
PHONG_DEFAULTS = dict(light_col=(1.0, 1.0, 1.0), ambient=0.1, k_diffuse=0.9, background_white=False, with_mask=True)
FIT_DEFAULTS = dict(pose_eta=0.01, light_eta=0.4, inner_step=200, max_epochs=10)       # config_reconstruction_RenderNet.json
# step size of the light colour and the ambient term (fit_shading): not in the reference and not tuned.  The loss is a pixel
# mean, so its curvature in the ambient term is about twice the masked fraction of the image (up to 2): 0.5 keeps the steps stable
SHADING_ETA = 0.5
LIGHT_AZIMUTHS_DEG = np.linspace(230, 320, num=5)                                       # Reconstruct_RenderNet_Face.py:465


def light_dir(light) -> np.ndarray:
    """[B,2] (azimuth, elevation) radians -> [B,3] float32 light directions, generate_light_pos's map (computed in float64)."""
    L = np.asarray(light, np.float64).reshape(-1, 2)
    az, el = L[:, 0], L[:, 1]
    return np.stack([-np.sin(el) * np.cos(az), np.cos(el), -np.sin(el) * np.sin(az)], 1).astype(np.float32)


def light_dir_jacobian(light) -> np.ndarray:
    """d light_dir / d(azimuth, elevation): [B,3,2] float64."""
    L = np.asarray(light, np.float64).reshape(-1, 2)
    az, el = L[:, 0], L[:, 1]
    z = np.zeros_like(az)
    return np.stack([np.stack([np.sin(el) * np.sin(az), -np.cos(el) * np.cos(az)], 1),
                     np.stack([z, -np.sin(el)], 1),
                     np.stack([-np.sin(el) * np.cos(az), -np.cos(el) * np.sin(az)], 1)], 1)


def check_objective(objective: str, is_greyscale: bool) -> None:
    if objective not in OBJECTIVES:
        raise ValueError(f"objective must be one of {OBJECTIVES}, not {objective!r}")
    if objective == "phong" and is_greyscale:
        raise ValueError("objective 'phong' shades a normal map: the greyscale network renders none (use 'bce' or 'mse')")


def _target_on(target, shape, device) -> torch.Tensor:
    t = target if isinstance(target, torch.Tensor) else torch.as_tensor(np.asarray(target, np.float32))
    if t.numel() != int(np.prod(shape)):
        raise ValueError(f"target {tuple(t.shape)} does not hold an image of shape {tuple(shape)}")
    return t.to(device=device, dtype=torch.float32).reshape(tuple(shape)).contiguous()


def shader_fit_gradients(ig, voxels, view_params, target, objective: str, light=None, light_col=PHONG_DEFAULTS["light_col"],
                         ambient: float = PHONG_DEFAULTS["ambient"], k_diffuse: float = PHONG_DEFAULTS["k_diffuse"],
                         background_white: bool = PHONG_DEFAULTS["background_white"],
                         with_mask: bool = PHONG_DEFAULTS["with_mask"], want_dvox: bool = False, want_dpose: bool = True,
                         dvox_on_device: bool = False, want_shading_grad: bool = False):
    """Loss [B] (float64) and the gradients of sum_b loss[b] at (voxels, view_params[, light]).

    ig: a backward.ShaderInputGradients of the batch size.  objective "phong" (RGB network only; light [B,2] = (azimuth,
    elevation) radians, required), "mse" or "bce" (raw output; light must be None).  target: [B,512,512,C] image (NumPy or
    tensor).  Returns (loss, {"pose": dL/dview_params [B,3] if want_dpose else None, "light": dL/d(azimuth, elevation) [B,2] or
    None, "voxels": dL/dvoxels [B,64,64,64,1] if want_dvox else None}), NumPy float64 except dL/dvoxels (float32; a CUDA tensor
    if dvox_on_device).  light_col: 1 or B rows of 3; ambient: a float or a [1|B] tensor.  want_shading_grad ("phong"): the
    dictionary also holds "light_col" [B,3] and "ambient" [B] (rn_phong_composite_loss_grad_params)."""
    check_objective(objective, ig.is_greyscale)
    B = ig.B
    if objective == "phong":
        if light is None:
            raise ValueError("objective 'phong' needs the light (azimuth, elevation) [B,2]")
        light = np.asarray(light, np.float64)
        if light.shape not in ((B, 2), (2,)):
            raise ValueError(f"light must be [{B},2] or [2] (azimuth, elevation), not {light.shape}")
        light = np.broadcast_to(light.reshape(-1, 2), (B, 2))
    elif light is not None:
        raise ValueError(f"objective {objective!r} has no light")
    if want_shading_grad and objective != "phong":
        raise ValueError(f"objective {objective!r} has no shading")
    img = ig.forward(voxels, view_params)
    tgt = _target_on(target, img.shape, img.device)
    dlight = None
    shading = {}
    with torch.cuda.device(img.device):
        if objective == "phong":
            ld = torch.from_numpy(light_dir(light)).to(img.device)
            out = ops.phong_composite_loss_grad(img, tgt, ld, light_col, ambient, k_diffuse, background_white, with_mask,
                                                **(dict(want_shading_grad=True) if want_shading_grad else {}))
            loss, dimg, dl = out[:3]
            dlight = np.einsum("bi,bij->bj", dl.double().cpu().numpy(), light_dir_jacobian(light))
            if want_shading_grad:
                shading = dict(light_col=out[3].double().cpu().numpy(), ambient=out[4].double().cpu().numpy())
        else:
            loss, dimg = ops.image_loss_grad_items(img, tgt, objective)
    dvox, dpose = ig.backward(dimg, want_dvox=want_dvox, want_dpose=want_dpose, dvox_on_device=dvox_on_device)
    return loss.cpu().numpy(), dict(pose=np.asarray(dpose, np.float64) if want_dpose else None, light=dlight, voxels=dvox,
                                    **shading)


def _deg(x):
    return float(x) * 180.0 / math.pi


def pose_window(pose) -> Dict[str, float]:
    """The (phi, theta) form create_param_center takes, in degrees, of a pose [3] in radians: phi = azimuth, theta = 90 - elevation
    parameter (Reconstruct_RenderNet_Face.py:533-534)."""
    return dict(phi=_deg(pose[0]), theta=90.0 - _deg(pose[1]))


def in_window(pose, window, slack_deg: float = 0.0) -> bool:
    """Whether a pose [3] (radians) lies in a searched window {"phi_mid", "phi_range", "theta_mid", "theta_range"} (degrees; the
    azimuth modulo 360)."""
    p = pose_window(pose)
    dphi = (p["phi"] - window["phi_mid"] + 180.0) % 360.0 - 180.0
    return (abs(dphi) <= window["phi_range"] / 2 + slack_deg and
            abs(p["theta"] - window["theta_mid"]) <= window["theta_range"] / 2 + slack_deg)


def pose_search(step_fn: Callable, loss_fn: Callable, target, init_pose, light=None, batch_size: int = 5, max_epochs: int = 10,
                inner_step: int = 200, callback: Optional[Callable] = None, shading: Optional[dict] = None) -> Dict[str, object]:
    """The reference's outer / inner loop (Reconstruct_RenderNet_Face.py:455-537) over the pose and, optionally, the light.

    step_fn(state, target) -> (new_state, loss [B], grads): one descent step from `state` {"pose" [B,3] radians, "light" [B,2]
    radians (only when `light` is given)}, loss evaluated at `state`.  loss_fn(state, target) -> loss [B] at a state.
    init_pose [3] (azimuth, elevation parameter, scale) centres the first 60 x 30 degree window; its scale is every hypothesis'.
    light: the first epoch's [5,2] lights, or None (no light in the state).  After the last inner step of an epoch the loss is
    re-evaluated, the argmin hypothesis kept, and the next epoch restarts five hypotheses in the halved window around its pose,
    with its scale and light.  callback(epoch, step, state, loss, selection_loss) runs after every step (selection_loss: the
    re-evaluated loss [B] after the last inner step, else None).

    Returns {"pose" [3], "light" [2] or None (the selected hypothesis), "best_param" (degrees, the reference's form),
    "best_index", "best_loss" (per epoch), "windows" (per epoch: phi_mid, phi_range, theta_mid, theta_range, degrees),
    "state" (the last state)}.  shading: the first epoch's {"light_col" [5,3], "ambient" [5]}, or None; given, they join the state,
    later epochs restart from the selected hypothesis' values, and the result holds the selected "light_col" [3] and "ambient"."""
    if batch_size != 5:
        raise ValueError(f"the pose search runs 5 hypotheses (create_param_center); batch_size is {batch_size}")
    if int(max_epochs) < 1 or int(inner_step) < 1:
        raise ValueError(f"max_epochs ({max_epochs}) and inner_step ({inner_step}) must be at least 1")
    init_pose = np.asarray(init_pose, np.float64).reshape(3)
    w = pose_window(init_pose)
    best_param = np.array([w["phi"], w["theta"], 1.0])
    scale = np.float32(init_pose[2])
    if light is not None:
        light = np.asarray(light, np.float32)
        if light.shape != (batch_size, 2):
            raise ValueError(f"light must be [{batch_size},2] (azimuth, elevation), not {light.shape}")
    best_light = best_pose = best_index = best_shading = None
    best_loss, windows = [], []
    phi_range, theta_range = 60.0, 30.0
    state = None
    for i in range(int(max_epochs)):
        if i > 0:
            phi_range /= 2
            theta_range /= 2
        params = create_param_center(phi_mid=best_param[0], phi_range=phi_range, theta_mid=best_param[1], theta_range=theta_range,
                                     batch_size=batch_size)
        params[:, 2] = scale
        windows.append(dict(phi_mid=float(best_param[0]), phi_range=phi_range, theta_mid=float(best_param[1]),
                            theta_range=theta_range))
        state = dict(pose=params)
        if light is not None:
            state["light"] = light.copy() if i == 0 else np.tile(best_light[np.newaxis, :], (batch_size, 1))
        if shading is not None:
            for k in ("light_col", "ambient"):
                v = np.asarray(shading[k], np.float32) if i == 0 else best_shading[k]
                state[k] = v.copy() if i == 0 else np.repeat(v[np.newaxis], batch_size, 0)
        for idx in range(int(inner_step)):
            state, loss, _ = step_fn(state, target)
            sel = None
            if idx == inner_step - 1:
                sel = np.asarray(loss_fn(state, target))
                j = int(np.argmin(sel))
                best_pose = np.asarray(state["pose"][j], np.float32).copy()
                best_light = None if light is None else np.asarray(state["light"][j], np.float32).copy()
                if shading is not None:
                    best_shading = {k: np.asarray(state[k][j], np.float32).copy() for k in ("light_col", "ambient")}
                w = pose_window(best_pose)
                best_param = np.array([w["phi"], w["theta"], 1.0])
                scale = best_pose[2]
                best_index = j
                best_loss.append(float(sel[j]))
            if callback is not None:
                callback(i, idx, state, loss, sel)
    out = dict(pose=best_pose, light=best_light, best_param=best_param, best_index=best_index, best_loss=best_loss,
               windows=windows, state=state)
    if shading is not None:
        out.update(best_shading)
    return out


def weights_are_greyscale(weights) -> Optional[bool]:
    """What the stored e_conv11 filter says (RenderNet_Shader.py:125-131; transposed filter [kh,kw,Cout,Cin]), None if absent."""
    if weights is None:
        return None
    last = [v for k, v in weights.items() if k.replace("/", "_").endswith("e_conv11_weights")]
    return (int(np.shape(last[0])[2]) == 1) if last else None


class ShaderPoseFit:
    """Pose (and light) fit of a known shape to a target image through the Shader network.

        fit = ShaderPoseFit(weights, voxels, objective="phong")      # weights: {tf name: array} or None (seeded)
        out = fit.run(target, init=dict(pose=[az, theta, scale], light=[az, el]))

    `gradients`, `step` (plain descent, var -= eta * grad in float32 like FaceReconstruction.step), `loss` and `render` work on a
    state {"pose" [5,3], "light" [5,2] ("phong" only)}; `run` is `pose_search` over them.  The voxels ([64,64,64], [1|5,...,1])
    are held fixed.  is_greyscale: None takes it from the weights' e_conv11 filter (False for seeded weights).

    fit_shading ("phong" only): the state also holds "light_col" [5,3] and "ambient" [5], starting from light_col / ambient;
    step descends them with shading_eta (SHADING_ETA: untuned) and projects them onto colour >= 0, 0 <= ambient <= 1; run
    returns the selected hypothesis' values and render shades with the state's."""

    def __init__(self, weights, voxels, objective: str = "phong", batch: int = 5, precision: str = "exact",
                 pose_eta: float = FIT_DEFAULTS["pose_eta"], light_eta: float = FIT_DEFAULTS["light_eta"],
                 inner_step: int = FIT_DEFAULTS["inner_step"], max_epochs: int = FIT_DEFAULTS["max_epochs"],
                 fit_scale: bool = False, is_greyscale: Optional[bool] = None, light_col=PHONG_DEFAULTS["light_col"],
                 ambient: float = PHONG_DEFAULTS["ambient"], k_diffuse: float = PHONG_DEFAULTS["k_diffuse"],
                 background_white: bool = PHONG_DEFAULTS["background_white"], with_mask: bool = PHONG_DEFAULTS["with_mask"],
                 loss_scale=None, seed: int = 0, device: str = "cuda", fit_shading: bool = False,
                 shading_eta: float = SHADING_ETA):
        if int(batch) != 5:
            raise ValueError(f"the pose search runs 5 hypotheses (create_param_center); batch is {batch}")
        found = weights_are_greyscale(weights)
        if is_greyscale is None:
            is_greyscale = bool(found)
        elif found is not None and found != bool(is_greyscale):
            raise ValueError(f"is_greyscale={is_greyscale}, but the weights' e_conv11 filter says {found}")
        check_objective(objective, is_greyscale)
        if fit_shading and objective != "phong":
            raise ValueError(f"fit_shading fits the Phong composite's light; objective {objective!r} has none")
        v = np.asarray(voxels, np.float32)
        if v.size not in (64 ** 3, 5 * 64 ** 3):
            raise ValueError(f"voxels must hold one or 5 grids of 64^3, not shape {v.shape}")
        self.voxels = np.ascontiguousarray(np.broadcast_to(v.reshape(-1, 64, 64, 64, 1), (5, 64, 64, 64, 1)))
        self.B, self.objective, self.is_greyscale = 5, objective, bool(is_greyscale)
        self.eta = dict(pose=float(pose_eta), light=float(light_eta))
        self.fit_shading = bool(fit_shading)
        if self.fit_shading:
            self.eta["shading"] = float(shading_eta)
        self.inner_step, self.max_epochs, self.fit_scale = int(inner_step), int(max_epochs), bool(fit_scale)
        self.phong = dict(light_col=light_col, ambient=float(ambient), k_diffuse=float(k_diffuse),
                          background_white=bool(background_white), with_mask=bool(with_mask))
        from .backward import ShaderInputGradients
        self.ig = ShaderInputGradients(weights, self.B, precision=precision, is_greyscale=self.is_greyscale, loss_scale=loss_scale,
                                       seed=seed, device=device)
        self.device = self.ig.device
        self._target = None

    def _target_dev(self, target):
        if isinstance(target, torch.Tensor):
            return target
        if self._target is None or self._target[0] is not target:
            self._target = (target, torch.as_tensor(np.asarray(target, np.float32)).to(self.device))
        return self._target[1]

    def _light(self, state):
        return state["light"] if self.objective == "phong" else None

    def _phong(self, state) -> dict:
        """The shading arguments at `state`: the constants, or with fit_shading the state's colour and ambient terms."""
        if not self.fit_shading:
            return self.phong
        return dict(self.phong, light_col=np.asarray(state["light_col"], np.float32),
                    ambient=torch.as_tensor(np.asarray(state["ambient"], np.float32)).to(self.device))

    def initial_shading(self) -> Optional[dict]:
        """The first epoch's {"light_col" [5,3], "ambient" [5]} (the constructor's constants), or None without fit_shading."""
        if not self.fit_shading:
            return None
        lc = np.asarray(self.phong["light_col"], np.float32).reshape(-1, 3)
        return dict(light_col=np.ascontiguousarray(np.broadcast_to(lc, (self.B, 3))),
                    ambient=np.full(self.B, self.phong["ambient"], np.float32))

    def gradients(self, state, target):
        """Loss [B] and dL/d(pose) [B,3], dL/d(light) [B,2] ("phong"; else None) of sum_b loss[b] at `state`; with fit_shading
        also dL/d(light_col) [B,3] and dL/d(ambient) [B]."""
        if self.fit_shading:
            return shader_fit_gradients(self.ig, self.voxels, state["pose"], self._target_dev(target), self.objective,
                                        light=self._light(state), want_shading_grad=True, **self._phong(state))
        return shader_fit_gradients(self.ig, self.voxels, state["pose"], self._target_dev(target), self.objective,
                                    light=self._light(state), **(self.phong if self.objective == "phong" else {}))

    def step(self, state, target):
        """One descent step: pose -= pose_eta * dpose (the scale only if fit_scale), light -= light_eta * dlight, in float32.
        Returns (new_state, loss [B] at `state`, grads)."""
        loss, grads = self.gradients(state, target)
        g = np.asarray(grads["pose"], np.float32).copy()
        if not self.fit_scale:
            g[:, 2] = 0.0
        new = dict(pose=(np.asarray(state["pose"], np.float32) - np.float32(self.eta["pose"]) * g).astype(np.float32))
        if self.objective == "phong":
            new["light"] = (np.asarray(state["light"], np.float32) -
                            np.float32(self.eta["light"]) * np.asarray(grads["light"], np.float32)).astype(np.float32)
        if self.fit_shading:
            eta = np.float32(self.eta["shading"])
            new["light_col"] = np.maximum(np.asarray(state["light_col"], np.float32) -
                                          eta * np.asarray(grads["light_col"], np.float32), np.float32(0)).astype(np.float32)
            new["ambient"] = np.clip(np.asarray(state["ambient"], np.float32) - eta * np.asarray(grads["ambient"], np.float32),
                                     np.float32(0), np.float32(1)).astype(np.float32)
        return new, loss, grads

    def loss(self, state, target) -> np.ndarray:
        """The objective [B] at `state` (forward and the loss kernel; no backward walk)."""
        img = self.ig.forward(self.voxels, state["pose"])
        tgt = _target_on(self._target_dev(target), img.shape, img.device)
        with torch.cuda.device(self.device):
            if self.objective == "phong":
                ld = torch.from_numpy(light_dir(state["light"])).to(self.device)
                p = self._phong(state)
                loss = ops.phong_composite_loss_grad(img, tgt, ld, p["light_col"], p["ambient"], p["k_diffuse"],
                                                     p["background_white"], p["with_mask"], want_light_grad=False)[0]
            else:
                loss = ops.image_loss_grad_items(img, tgt, self.objective, want_grad=False)[0]
        return loss.cpu().numpy()

    def render(self, state) -> Dict[str, np.ndarray]:
        """The fitted images of a state, NumPy: "image" (the raw network output [B,512,512,C] float32) and, for "phong", "shaded"
        (rn_phong_composite: the very image the loss measures) and "shaded_u8" (clip(255 x) as uint8, RenderNet_demo.py:58);
        otherwise "image_u8"."""
        img = self.ig.forward(self.voxels, state["pose"])
        out = dict(image=img)
        with torch.cuda.device(self.device):
            if self.objective == "phong" and self.fit_shading:
                p = self._phong(state)
                ld = torch.from_numpy(light_dir(state["light"])).to(self.device)
                out["shaded"], _, out["shaded_u8"] = ops.phong_shade(img, ld, p["light_col"], p["ambient"], p["k_diffuse"],
                                                                     composite="numpy", background_white=p["background_white"],
                                                                     with_mask=p["with_mask"])
            elif self.objective == "phong":
                p = self.phong
                ld = torch.from_numpy(light_dir(state["light"])).to(self.device)
                lc = ops._light_rows(p["light_col"], self.B, img.device, "light_col")
                out["shaded"], out["shaded_u8"] = ops.phong_composite(img, ld, lc, p["ambient"], p["k_diffuse"],
                                                                      p["background_white"], p["with_mask"], want_u8=True)
            else:
                out["image_u8"] = (255.0 * img).clamp(0, 255).to(torch.uint8)
        return {k: v.cpu().numpy() for k, v in out.items()}

    def initial_light(self, init) -> Optional[np.ndarray]:
        """The first epoch's lights [5,2]: init["light"] ([2] or [5,2], radians) if given, else azimuths linspace(230, 320)
        degrees at init["light_elevation"] (radians; the demo's 60 degrees by default).  None unless the objective is "phong"."""
        if self.objective != "phong":
            return None
        if init.get("light") is not None:
            L = np.asarray(init["light"], np.float32)
            if L.shape not in ((2,), (self.B, 2)):
                raise ValueError(f"init light must be [2] or [{self.B},2] (azimuth, elevation), not {L.shape}")
            return np.ascontiguousarray(np.broadcast_to(L.reshape(-1, 2), (self.B, 2)))
        el = float(init.get("light_elevation", math.radians(60.0)))
        return np.stack([LIGHT_AZIMUTHS_DEG * math.pi / 180.0, np.full(self.B, el)], 1).astype(np.float32)

    def run(self, target, init: Optional[dict] = None, callback: Optional[Callable] = None) -> Dict[str, object]:
        """The search from init {"pose": [3] radians (default: azimuth 270 degrees, elevation parameter 0, scale 1 -- the
        reference's first window), "light" or "light_elevation" (see initial_light)}.  Returns pose_search's dictionary."""
        init = dict(init or {})
        pose = np.asarray(init.get("pose", [math.radians(270.0), 0.0, 1.0]), np.float64).reshape(3)
        if self.fit_shading:
            return pose_search(self.step, self.loss, target, pose, light=self.initial_light(init), batch_size=self.B,
                               max_epochs=self.max_epochs, inner_step=self.inner_step, callback=callback,
                               shading=self.initial_shading())
        return pose_search(self.step, self.loss, target, pose, light=self.initial_light(init), batch_size=self.B,
                           max_epochs=self.max_epochs, inner_step=self.inner_step, callback=callback)


# ------------------------------------------------------------------------------------------ command line
def main(argv=None):
    from .RenderNet_demo import compute_pose_param, load_graph
    from . import binvox_rw
    parser = argparse.ArgumentParser(description="Fit the view (and light) of a known voxel shape to an image through the Shader "
                                                 "network.", formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    parser.add_argument('--voxel_path', type=str, required=True, help="Path to the input voxel (.binvox, 64^3).")
    parser.add_argument('--target', type=str, required=True, help="Target image (512x512 PNG; RGB, or greyscale for bce/mse).")
    parser.add_argument('--model', type=str, default="./model/3d2d_renderer.pb",
                        help="Weights as RenderNet_demo loads them; seeded random weights if missing.")
    parser.add_argument('--is_greyscale', action='store_true', help="Seeded weights: the greyscale network.")
    parser.add_argument('--objective', type=str, default="phong", choices=OBJECTIVES)
    parser.add_argument('--azimuth', type=float, default=250, help="Initial guess: azimuth (degrees), as RenderNet_demo.")
    parser.add_argument('--elevation', type=float, default=60, help="Initial guess: elevation (degrees), as RenderNet_demo.")
    parser.add_argument('--radius', type=float, default=3.3, help="Radius (held fixed unless --fit_scale).")
    parser.add_argument('--light_azimuth', type=float, default=None,
                        help="Initial light azimuth (degrees); default: five hypotheses linspace(230, 320).")
    parser.add_argument('--light_elevation', type=float, default=60, help="Initial light elevation (degrees).")
    parser.add_argument('--precision', type=str, default="exact", choices=("exact", "fast"))
    parser.add_argument('--inner_step', type=int, default=FIT_DEFAULTS["inner_step"])
    parser.add_argument('--max_epochs', type=int, default=FIT_DEFAULTS["max_epochs"])
    parser.add_argument('--pose_eta', type=float, default=FIT_DEFAULTS["pose_eta"])
    parser.add_argument('--light_eta', type=float, default=FIT_DEFAULTS["light_eta"])
    parser.add_argument('--fit_scale', action='store_true')
    parser.add_argument('--fit_shading', action='store_true',
                        help="Also fit the light colour and the ambient term (objective phong; k_diffuse stays 0.9).")
    parser.add_argument('--shading_eta', type=float, default=SHADING_ETA, help="Step size of the colour and ambient terms.")
    parser.add_argument('--out_dir', type=str, default="./fit", help="Where the JSON and the PNG of the fit go.")
    args = parser.parse_args(argv)
    from PIL import Image

    have_model = os.path.exists(args.model) or os.path.exists(args.model + ".index")
    graph = load_graph(args.model if have_model else None, is_greyscale=None if have_model else args.is_greyscale)
    with open(args.voxel_path, 'rb') as f:
        voxel = np.reshape(binvox_rw.read_as_3d_array(f).data.astype(np.float32), (1, 64, 64, 64, 1))
    target = np.asarray(Image.open(args.target).convert("L" if graph.is_greyscale else "RGB"), np.float32) / 255.0
    target = np.tile(target.reshape((1, 512, 512, -1)), (5, 1, 1, 1))
    fit = ShaderPoseFit(graph.weights, voxel, objective=args.objective, precision=args.precision, pose_eta=args.pose_eta,
                        light_eta=args.light_eta, inner_step=args.inner_step, max_epochs=args.max_epochs,
                        fit_scale=args.fit_scale, is_greyscale=graph.is_greyscale,
                        **(dict(fit_shading=True, shading_eta=args.shading_eta) if args.fit_shading else {}))
    init = dict(pose=compute_pose_param(args.azimuth, args.elevation, args.radius)[0],
                light_elevation=math.radians(args.light_elevation))
    if args.light_azimuth is not None:
        init["light"] = [math.radians(args.light_azimuth), math.radians(args.light_elevation)]
    first = []
    out = fit.run(target, init=init, callback=lambda e, i, s, loss, sel: first.append(np.asarray(loss)) if not first else None)
    pose, light = out["pose"], out["light"]
    res = dict(azimuth=_deg(pose[0]) % 360.0, elevation=90.0 - _deg(pose[1]), radius=3.3 / float(pose[2]),
               pose=[float(v) for v in pose], objective=args.objective, best_loss=out["best_loss"], best_index=out["best_index"],
               first_step_loss=[float(v) for v in first[0]], windows=out["windows"])
    if light is not None:
        res.update(light_azimuth=_deg(light[0]) % 360.0, light_elevation=_deg(light[1]), light=[float(v) for v in light])
    if args.fit_shading:
        res.update(light_col=[float(v) for v in out["light_col"]], ambient=float(out["ambient"]))
    imgs = fit.render(out["state"])                  # the selected hypothesis is out["best_index"] of the last state
    u8 = (imgs["shaded_u8"] if args.objective == "phong" else imgs["image_u8"])[out["best_index"]][None]
    os.makedirs(args.out_dir, exist_ok=True)
    stem = os.path.join(args.out_dir, os.path.basename(args.voxel_path).split('.binvox')[0] + "_fit")
    Image.fromarray(u8[0, ..., 0] if u8.shape[-1] == 1 else u8[0]).save(stem + ".png")
    with open(stem + ".json", "w") as f:
        json.dump(res, f, indent=1)
    print(stem + ".json", json.dumps({k: res[k] for k in res if k not in ("windows",)}))
    return res


if __name__ == "__main__":
    main()
