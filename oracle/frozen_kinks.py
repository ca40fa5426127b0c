"""PReLU with frozen kinks, for comparing whole-network gradients element by element.

Two fp32 implementations of the Shader graph differ by ~1e-6 relative per layer, so a few units per layer sit on opposite sides
of a PReLU kink in the two; each such unit changes its gradient by a whole term (1 vs alpha).  With the branch of every unit
taken from one implementation, both differentiate the same piecewise-linear function and their gradients agree to rounding.
"""
import contextlib

import numpy as np
import torch

from . import rendernet_oracle as orc


@contextlib.contextmanager
def prelu_kinks(W, masks=None, record=None):
    """Inside the block, every `orc.prelu(z, alpha)` call (looked up at call time, so projection_unit's too) identifies its layer
    by the identity of `alpha` among the "/alpha" values of W -- the model functions pass W[name] through unchanged.
    masks {alpha name: bool tensor of z's shape}: the call returns where(mask, z, alpha * z) instead.
    record: a dict filled with {alpha name: z > 0} of every call."""
    names = {id(v): n for n, v in W.items() if n.endswith("/alpha")}
    plain = orc.prelu

    def prelu(x, alpha):
        name = names[id(alpha)]
        x = orc._t(x).float()
        if record is not None:
            record[name] = (x > 0).detach()
        if masks is None:
            return plain(x, alpha)
        a = alpha.float() if isinstance(alpha, torch.Tensor) else torch.from_numpy(np.asarray(alpha, np.float32))
        m = torch.as_tensor(masks[name]).to(device=x.device, dtype=torch.bool)
        if tuple(m.shape) != tuple(x.shape):
            raise ValueError(f"kink mask of {name}: shape {tuple(m.shape)} != pre-activation shape {tuple(x.shape)}")
        return torch.where(m, x, a * x)

    orc.prelu = prelu
    try:
        yield
    finally:
        orc.prelu = plain


def tape_prelu_masks(tape):
    """{alpha name: pre-activation > 0} of every PReLU layer recorded on a rendernet_b200 tape: the branch its backward pass took
    (rec["rerun"]() returns the layer's pre-activation, kept or recomputed)."""
    return {rec["alpha"]._rn_name: (rec["rerun"]().float() > 0).cpu() for rec in tape
            if rec.get("act") == "prelu" and not isinstance(rec["alpha"], str)}


def kink_flips(masks, signs):
    """(units on opposite sides of the kink, units compared) between two {alpha name: bool tensor} maps."""
    n = sum(int((masks[k].cpu() != signs[k].cpu()).sum()) for k in signs)
    return n, sum(int(signs[k].numel()) for k in signs)
