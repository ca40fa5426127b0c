"""Reconstruct a voxel shape from posed images through the Shader network: multi-view occupancy fit with silhouette carving.

The Shader has no shape prior, so what stands in for one is the usual set-up of a differentiable renderer used for shape:
several views at known poses, a silhouette hull to start from, occupancy kept in [0, 1], and two regularisers that push toward
what the network was trained on (smooth, binary grids):

    fit = ShaderShapeFit(weights, poses, objective="phong", light=[az, el])      # poses [V,3] (radians, scale), known
    out = fit.run(targets, masks=masks, steps=100)                              # targets [V,512,512,C], masks [V,512,512]
    fit.save(out["occupancy"], "shape.binvox")                                 # thresholded at 0.1, as the reference saves

Objective, over one occupancy grid occ [64,64,64] that every view renders:
    L(occ) = sum_v loss_v(occ) + lambda_smooth R_s(occ) + lambda_bin R_b(occ)
with loss_v the objective of `shader_fit.shader_fit_gradients` ("phong", "mse" or "bce") of view v, R_s the mean squared difference
of axis neighbours and R_b = mean occ (1 - occ) (rn_voxel_fit_grad).  Views run in chunks of `batch` through one
ShaderInputGradients; each chunk's dL/dvoxels stays on the device, one rn_voxel_fit_grad launch sums the views, adds the
regularisers and zeroes the carved voxels, then rn_adam_step updates occ and a clamp projects it onto [0, 1].  Carved voxels have
a zero gradient, so their Adam moments stay 0 and they never move.

Carving (`carve`): a voxel is kept iff some view observes it (a sample of the network's 128^3 grid reads it with a nonzero
trilinear weight) and every view that observes it reads it from inside that view's silhouette.  Both tests are resampler
backwards (rn_resample_backward_f32) of an indicator: sums of non-negative weights cannot cancel, so "> 0" is an exact support test.

The default lambda_smooth, lambda_bin, lr and betas are untuned starting values: tuning them needs trained Shader weights, which
the package does not ship.  Reconstruction quality on real data is therefore unverified; the tests pin the gradients, the carving
and the mechanics.
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
from .shader_fit import OBJECTIVES, PHONG_DEFAULTS, _target_on, check_objective, light_dir, shader_fit_gradients, weights_are_greyscale

SIZE, NEW_SIZE, IMAGE = 64, 128, 512
# untuned starting values (see the module docstring)
SHAPE_FIT_DEFAULTS = dict(lambda_smooth=0.1, lambda_bin=0.01, lr=0.01, betas=(0.9, 0.999), eps=1e-8, steps=100)
SAVE_THRESHOLD = 0.1                 # Reconstruct_RenderNet_Face.py:516 saves vox > 0.1


# ------------------------------------------------------------------------------------------ carving
def mask_columns(masks, margin: int = 1) -> np.ndarray:
    """[V,512,512] silhouettes -> [V,128,128] bool columns of the network's grid: a column is inside if any of its 4 x 4 pixels
    is, then the inside is dilated by `margin` columns (a square of side 2 margin + 1), because the learned geometry blurs."""
    m = np.asarray(masks, bool)
    if m.ndim != 3 or m.shape[1:] != (IMAGE, IMAGE):
        raise ValueError(f"masks must be [V,{IMAGE},{IMAGE}], not {m.shape}")
    if int(margin) < 0:
        raise ValueError(f"margin must be >= 0, not {margin}")
    f = IMAGE // NEW_SIZE
    cols = m.reshape(m.shape[0], NEW_SIZE, f, NEW_SIZE, f).any(axis=(2, 4))
    for axis in (1, 2):
        out = cols.copy()
        for s in range(1, int(margin) + 1):
            lo = [slice(None)] * 3
            hi = [slice(None)] * 3
            lo[axis], hi[axis] = slice(s, None), slice(None, -s)
            out[tuple(lo)] |= cols[tuple(hi)]
            out[tuple(hi)] |= cols[tuple(lo)]
        cols = out
    return cols


def carve_rule(observed, inside) -> np.ndarray:
    """observed, inside [V, ...] (resampler backwards of ones and of the silhouette) -> uint8 keep: observed by at least one view,
    and inside (> 0) in every view that observes it."""
    seen = np.asarray(observed) > 0
    ok = ~seen | (np.asarray(inside) > 0)
    return (seen.any(0) & ok.all(0)).astype(np.uint8)


def _device_resample_backward(minv: torch.Tensor, gout: torch.Tensor, size: int) -> torch.Tensor:
    V = int(minv.shape[0])
    # the scatter reads no voxel value when only dvox is asked for; the buffer gives the kernel its shape
    vox = torch.zeros((V, size, size, size, 1), device=gout.device, dtype=torch.float32)
    return ops.resample_backward(vox, minv, gout, True, want_dvox=True, want_dminv=False)[0]


def carve(poses, masks, margin: int = 1, size: int = SIZE, device: str = "cuda",
          resample_backward: Optional[Callable] = None) -> np.ndarray:
    """The silhouette hull, uint8 [size,size,size] (1 = kept).  poses [V,3] (azimuth, elevation, scale; radians), masks [V,512,512]
    bool.  Each mask is reduced to the network's 128^2 columns (mask_columns), broadcast along depth in the axis-transformed
    layout the network reads ([V,128,128,128,1]), and pushed back through the resampler twice: observed_v = backward(ones),
    inside_v = backward(mask).  resample_backward(minv [V,3,4], gout [V,128,128,128,1]) -> dvox [V,size^3...] replaces the device
    scatter (tests)."""
    from .engine import pose_to_matrix
    poses = np.asarray(poses, np.float32).reshape(-1, 3)
    cols = mask_columns(masks, margin)
    if cols.shape[0] != poses.shape[0]:
        raise ValueError(f"{poses.shape[0]} poses but {cols.shape[0]} masks")
    V = poses.shape[0]
    minv = torch.from_numpy(pose_to_matrix(poses, size, NEW_SIZE)).to(device)
    back = resample_backward or (lambda m, g: _device_resample_backward(m, g, size))
    ones = torch.ones((V, NEW_SIZE, NEW_SIZE, NEW_SIZE, 1), device=device, dtype=torch.float32)
    observed = back(minv, ones).reshape(V, -1)
    del ones
    grid = torch.from_numpy(cols).to(device=device, dtype=torch.float32)[:, :, :, None, None]
    inside = back(minv, grid.expand(V, NEW_SIZE, NEW_SIZE, NEW_SIZE, 1).contiguous()).reshape(V, -1)
    keep = carve_rule(observed.cpu().numpy(), inside.cpu().numpy())
    return keep.reshape(size, size, size)


# ------------------------------------------------------------------------------------------ the fit
class ShaderShapeFit:
    """Occupancy fit of one 64^3 grid to V posed target images through the Shader network (see the module docstring).

        fit = ShaderShapeFit(weights, poses, objective="phong", light=[az, el])      # weights: {tf name: array} or None (seeded)
        loss, reg, g = fit.gradients(occ, targets)                                   # loss [V], reg (R_s, R_b), g CUDA [64,64,64]
        state = fit.init_state(occ); fit.step(state, targets)                        # one Adam step + clamp, in place
        out = fit.run(targets, masks=masks, steps=100)

    poses [V,3] (azimuth, elevation, scale; radians), known.  light [V,2] or [2] (azimuth, elevation; radians), "phong" only and
    required there.  `keep` (uint8 [64,64,64] or None) restricts the fit to a hull; `run` sets it from the masks."""

    def __init__(self, weights, poses, objective: str = "phong", batch: int = 8, precision: str = "exact",
                 is_greyscale: bool = False, light=None, lambda_smooth: float = SHAPE_FIT_DEFAULTS["lambda_smooth"],
                 lambda_bin: float = SHAPE_FIT_DEFAULTS["lambda_bin"], lr: float = SHAPE_FIT_DEFAULTS["lr"],
                 betas=SHAPE_FIT_DEFAULTS["betas"], eps: float = SHAPE_FIT_DEFAULTS["eps"], loss_scale=None, seed: int = 0,
                 device: str = "cuda"):
        found = weights_are_greyscale(weights)
        if found is not None and found != bool(is_greyscale):
            raise ValueError(f"is_greyscale={is_greyscale}, but the weights' e_conv11 filter says {found}")
        check_objective(objective, bool(is_greyscale))
        poses = np.asarray(poses, np.float32)
        if poses.ndim != 2 or poses.shape[1] != 3 or poses.shape[0] < 1:
            raise ValueError(f"poses must be [V,3] (azimuth, elevation, scale), not {poses.shape}")
        V = poses.shape[0]
        if objective == "phong":
            if light is None:
                raise ValueError("objective 'phong' needs the light (azimuth, elevation): [V,2] or [2]")
            light = np.asarray(light, np.float64)
            if light.shape not in ((V, 2), (2,)):
                raise ValueError(f"light must be [{V},2] or [2] (azimuth, elevation), not {light.shape}")
            light = np.ascontiguousarray(np.broadcast_to(light.reshape(-1, 2), (V, 2)))
        elif light is not None:
            raise ValueError(f"objective {objective!r} has no light")
        for name, lam in (("lambda_smooth", lambda_smooth), ("lambda_bin", lambda_bin)):
            if not (math.isfinite(float(lam)) and float(lam) >= 0.0):
                raise ValueError(f"{name} must be a finite number >= 0, not {lam}")
        b1, b2 = (float(b) for b in betas)
        if not (0.0 <= b1 < 1.0 and 0.0 <= b2 < 1.0) or not (float(lr) > 0.0 and math.isfinite(float(lr))) or not float(eps) > 0:
            raise ValueError(f"need lr > 0, 0 <= betas < 1 and eps > 0, not lr={lr}, betas={betas}, eps={eps}")
        if int(batch) < 1:
            raise ValueError(f"batch must be >= 1, not {batch}")
        self.V, self.B = V, min(int(batch), V)
        self.poses, self.light, self.objective, self.is_greyscale = poses, light, objective, bool(is_greyscale)
        self.lambda_smooth, self.lambda_bin = float(lambda_smooth), float(lambda_bin)
        self.lr, self.betas, self.eps = float(lr), (b1, b2), float(eps)
        self.phong = dict(PHONG_DEFAULTS)
        self.keep = None
        from .backward import ShaderInputGradients
        self.ig = ShaderInputGradients(weights, self.B, precision=precision, is_greyscale=self.is_greyscale, loss_scale=loss_scale,
                                       seed=seed, device=device)
        self.device = self.ig.device
        self._target = None

    # ---------------------------------------------------------------------------------- plumbing
    def _chunks(self):
        """(first view, number of real views, row indices [B]) per chunk; the last chunk repeats its last view to fill the batch
        (those rows are computed and dropped)."""
        for v0 in range(0, self.V, self.B):
            n = min(self.B, self.V - v0)
            yield v0, n, np.minimum(np.arange(v0, v0 + self.B), self.V - 1)

    def _occ(self, occ) -> torch.Tensor:
        t = occ if isinstance(occ, torch.Tensor) else torch.as_tensor(np.asarray(occ, np.float32))
        if t.numel() != SIZE ** 3:
            raise ValueError(f"occupancy must hold a 64^3 grid, not shape {tuple(t.shape)}")
        return t.to(device=self.device, dtype=torch.float32).reshape(SIZE, SIZE, SIZE).contiguous()

    def _voxels(self, occ: torch.Tensor) -> torch.Tensor:
        return occ.reshape(1, SIZE, SIZE, SIZE, 1).expand(self.B, SIZE, SIZE, SIZE, 1)

    def _targets(self, target) -> torch.Tensor:
        if self._target is not None and self._target[0] is target:
            return self._target[1]
        C = 1 if self.is_greyscale else 3
        t = _target_on(target, (self.V, IMAGE, IMAGE, C), self.device)
        self._target = (target, t)
        return t

    def _keep(self) -> Optional[torch.Tensor]:
        if self.keep is None:
            return None
        k = np.asarray(self.keep)
        if k.dtype != np.uint8 or k.size != SIZE ** 3:
            raise ValueError(f"keep must be uint8 with 64^3 elements, not {k.dtype} {k.shape}")
        return torch.from_numpy(np.ascontiguousarray(k.reshape(-1))).to(self.device)

    def _light(self, rows):
        return self.light[rows] if self.objective == "phong" else None

    # ---------------------------------------------------------------------------------- objective
    def gradients(self, occ, target):
        """(loss [V] float64 NumPy, reg [2] float64 NumPy = (R_s, R_b), g fp32 CUDA [64,64,64]) at occ: the data term's loss per
        view and the gradient of sum_v loss_v + lambda_smooth R_s + lambda_bin R_b (zero outside `keep`)."""
        occ = self._occ(occ)
        tgt = self._targets(target)
        vox = self._voxels(occ)
        loss = np.zeros(self.V, np.float64)
        dvox = torch.empty((self.V, SIZE, SIZE, SIZE), device=self.device, dtype=torch.float32)
        extra = self.phong if self.objective == "phong" else {}
        for v0, n, rows in self._chunks():
            lc, g = shader_fit_gradients(self.ig, vox, self.poses[rows], tgt[torch.from_numpy(rows).to(self.device)], self.objective,
                                         light=self._light(rows), want_dvox=True, want_dpose=False, dvox_on_device=True, **extra)
            loss[v0:v0 + n] = lc[:n]
            dvox[v0:v0 + n] = g["voxels"][:n].reshape(n, SIZE, SIZE, SIZE)
        with torch.cuda.device(self.device):
            g, reg = ops.voxel_fit_grad(dvox, occ, self._keep(), self.lambda_smooth, self.lambda_bin)
        return loss, reg.cpu().numpy(), g

    def init_state(self, occ) -> Dict[str, object]:
        """A fit state: the occupancy (fp32 CUDA [64,64,64], a copy) and zero Adam moments."""
        occ = self._occ(occ).clone()
        return dict(occ=occ, m=torch.zeros_like(occ), v=torch.zeros_like(occ), t=0)

    def step(self, state, target):
        """One Adam step (tf.train.AdamOptimizer's form, rn_adam_step) on state["occ"], in place, then the clamp onto [0, 1].
        Returns (loss [V], reg [2]) at the occupancy before the step."""
        loss, reg, g = self.gradients(state["occ"], target)
        state["t"] += 1
        b1, b2 = self.betas
        t = state["t"]
        lr_t = self.lr * math.sqrt(1.0 - b2 ** t) / (1.0 - b1 ** t)
        with torch.cuda.device(self.device):
            ops.adam_step(state["occ"], g, state["m"], state["v"], lr_t, b1, b2, self.eps)
            state["occ"].clamp_(0.0, 1.0)
        return loss, reg

    def loss(self, occ, target) -> np.ndarray:
        """The data term [V] at occ (forward and the loss kernel; no backward walk)."""
        occ = self._occ(occ)
        tgt = self._targets(target)
        vox = self._voxels(occ)
        out = np.zeros(self.V, np.float64)
        p = self.phong
        for v0, n, rows in self._chunks():
            img = self.ig.forward(vox, self.poses[rows])
            t = tgt[torch.from_numpy(rows).to(self.device)]
            with torch.cuda.device(self.device):
                if self.objective == "phong":
                    ld = torch.from_numpy(light_dir(self.light[rows])).to(self.device)
                    lc = ops.phong_composite_loss_grad(img, t, ld, p["light_col"], p["ambient"], p["k_diffuse"], p["background_white"],
                                                       p["with_mask"], want_light_grad=False)[0]
                else:
                    lc = ops.image_loss_grad_items(img, t, self.objective, want_grad=False)[0]
            out[v0:v0 + n] = lc.cpu().numpy()[:n]
        return out

    def render(self, occ) -> Dict[str, np.ndarray]:
        """The images of occ in every view, NumPy: "image" (raw network output [V,512,512,C]) and, for "phong", "shaded" (the
        composite the loss measures) and "shaded_u8"; otherwise "image_u8"."""
        occ = self._occ(occ)
        vox = self._voxels(occ)
        parts: Dict[str, list] = {}
        p = self.phong
        for v0, n, rows in self._chunks():
            img = self.ig.forward(vox, self.poses[rows])
            out = dict(image=img)
            with torch.cuda.device(self.device):
                if self.objective == "phong":
                    ld = torch.from_numpy(light_dir(self.light[rows])).to(self.device)
                    lc = ops._light_rows(p["light_col"], self.B, img.device, "light_col")
                    out["shaded"], out["shaded_u8"] = ops.phong_composite(img, ld, lc, p["ambient"], p["k_diffuse"],
                                                                          p["background_white"], p["with_mask"], want_u8=True)
                else:
                    out["image_u8"] = (255.0 * img).clamp(0, 255).to(torch.uint8)
            for k, t in out.items():
                parts.setdefault(k, []).append(t[:n].cpu().numpy())
        return {k: np.concatenate(v) for k, v in parts.items()}

    def run(self, target, masks=None, init=None, steps: int = SHAPE_FIT_DEFAULTS["steps"], margin: int = 1,
            callback: Optional[Callable] = None) -> Dict[str, object]:
        """Fit from init ([64^3] occupancy; default: the carved hull at 0.5, or 0.5 everywhere without masks).  masks [V,512,512]
        bool: the silhouettes `carve` turns into `keep` (None: no carving, `keep` is left as it is).  callback(step, loss, reg,
        occ) runs after every step (loss [V] and reg [2] at the occupancy before the step, occ the CUDA state after it).
        Returns {"occupancy": fp32 [64,64,64], "loss": [steps, V], "reg": [steps, 2], "keep": uint8 or None}."""
        if masks is not None:
            m = np.asarray(masks, bool)
            if m.shape[0] != self.V:
                raise ValueError(f"{self.V} views but {m.shape[0]} masks")
            self.keep = carve(self.poses, m, margin=margin, device=self.device)
        if init is None:
            init = (0.5 * self.keep.astype(np.float32) if self.keep is not None else np.full((SIZE,) * 3, 0.5, np.float32))
        state = self.init_state(init)
        losses, regs = [], []
        for k in range(int(steps)):
            loss, reg = self.step(state, target)
            losses.append(loss)
            regs.append(reg)
            if callback is not None:
                callback(k, loss, reg, state["occ"])
        return dict(occupancy=state["occ"].cpu().numpy(), loss=np.array(losses).reshape(-1, self.V),
                    reg=np.array(regs).reshape(-1, 2), keep=self.keep)

    @staticmethod
    def save(occ, path, threshold: float = SAVE_THRESHOLD) -> None:
        """Write occ > threshold as a .binvox (binvox_rw.save_binvox; the reference saves its reconstructions at 0.1)."""
        from . import binvox_rw
        o = occ.cpu().numpy() if isinstance(occ, torch.Tensor) else np.asarray(occ)
        binvox_rw.save_binvox(o.reshape(SIZE, SIZE, SIZE) > threshold, path)


# ------------------------------------------------------------------------------------------ command line
def main(argv=None):
    from PIL import Image
    from .RenderNet_demo import load_graph
    from .data_util import extract_param_from_names
    parser = argparse.ArgumentParser(description="Reconstruct a 64^3 voxel shape from posed images through the Shader network.",
                                     formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    parser.add_argument("targets", nargs="+", help="Target images (512x512 PNG), named ..._p<az>_t<el>_r<r>... unless --poses.")
    parser.add_argument("--poses", type=str, default=None,
                        help="JSON list of [azimuth, elevation, scale] per target (radians; extract_param_from_names' form).")
    parser.add_argument("--weights", type=str, default="./model/3d2d_renderer.pb",
                        help="Weights as RenderNet_demo loads them; seeded random weights if missing.")
    parser.add_argument("--greyscale", action="store_true", help="Seeded weights: the greyscale network.")
    parser.add_argument("--objective", type=str, default="phong", choices=OBJECTIVES)
    parser.add_argument("--light", type=float, nargs=2, default=[275.0, 60.0], metavar=("AZ", "EL"),
                        help="Light azimuth and elevation (degrees) of the 'phong' objective.")
    parser.add_argument("--steps", type=int, default=SHAPE_FIT_DEFAULTS["steps"])
    parser.add_argument("--batch", type=int, default=8, help="Views per network pass.")
    parser.add_argument("--precision", type=str, default="exact", choices=("exact", "fast"))
    parser.add_argument("--mask-threshold", type=float, default=0.05,
                        help="Silhouette = pixels whose luminance (0..1) exceeds this; the hull is carved from them.")
    parser.add_argument("--out", type=str, default="./shape_fit", help="Output directory.")
    args = parser.parse_args(argv)

    have_model = os.path.exists(args.weights) or os.path.exists(args.weights + ".index")
    graph = load_graph(args.weights if have_model else None, is_greyscale=None if have_model else args.greyscale)
    if args.poses is not None:
        with open(args.poses) as f:
            poses = np.asarray(json.load(f), np.float32).reshape(-1, 3)
    else:
        poses = np.concatenate([extract_param_from_names(os.path.basename(p)) for p in args.targets]).astype(np.float32)
    if poses.shape[0] != len(args.targets):
        raise ValueError(f"{len(args.targets)} targets but {poses.shape[0]} poses")
    imgs = [np.asarray(Image.open(p).convert("RGB"), np.float32) / 255.0 for p in args.targets]
    rgb = np.stack(imgs)
    lum = rgb @ np.array([0.299, 0.587, 0.114], np.float32)
    masks = lum > args.mask_threshold
    target = lum[..., None] if graph.is_greyscale else rgb
    light = [math.radians(args.light[0]), math.radians(args.light[1])] if args.objective == "phong" else None
    fit = ShaderShapeFit(graph.weights, poses, objective=args.objective, batch=args.batch, precision=args.precision,
                         is_greyscale=graph.is_greyscale, light=light)
    out = fit.run(target, masks=masks, steps=args.steps)
    occ = out["occupancy"]
    os.makedirs(args.out, exist_ok=True)
    fit.save(occ, os.path.join(args.out, "shape.binvox"))
    np.save(os.path.join(args.out, "occupancy.npy"), occ)
    renders = fit.render(occ)
    u8 = renders["shaded_u8"] if args.objective == "phong" else renders["image_u8"]
    for v in range(fit.V):
        Image.fromarray(u8[v, ..., 0] if u8.shape[-1] == 1 else u8[v]).save(os.path.join(args.out, f"render_{v}.png"))
    res = dict(objective=args.objective, targets=list(args.targets), poses=poses.tolist(), light_deg=list(args.light),
               loss=out["loss"].sum(1).tolist(), loss_per_view=out["loss"].tolist(), R_s=out["reg"][:, 0].tolist(),
               R_b=out["reg"][:, 1].tolist(), hull_size=int(out["keep"].sum()),
               occupied_at_threshold=int((occ > SAVE_THRESHOLD).sum()), threshold=SAVE_THRESHOLD,
               lambda_smooth=fit.lambda_smooth, lambda_bin=fit.lambda_bin, lr=fit.lr, steps=args.steps)
    with open(os.path.join(args.out, "fit.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(os.path.join(args.out, "fit.json"), json.dumps({k: res[k] for k in ("hull_size", "occupied_at_threshold")}),
          "loss", res["loss"][0], "->", res["loss"][-1])
    return res


if __name__ == "__main__":
    main()
