"""LAMB and LARS as ``torch.optim.Optimizer`` subclasses: the torch-op engine's optimizers for ``--optimizer lamb|lars``
and the reference the native kernels are tested against.

torch has neither.  The semantics are those of the most widely used PyTorch implementations, timm's ``Lamb`` and
``Lars``, at the settings this project uses (``config.TRAIN``): for a tensor p with gradient g and decay wd,

LAMB (bias correction on, grad_averaging, no global clipping, no trust clipping)::

    m = b1 m + (1 - b1) g        v = b2 v + (1 - b2) g^2
    u = (m / (1 - b1^t)) / (sqrt(v) / sqrt(1 - b2^t) + eps) + wd p
    r = |p| / |u|  if wd != 0 and |p| > 0 and |u| > 0, else 1
    p = p - lr r u

LARS (no dampening, no Nesterov, no trust clipping)::

    r = coeff |p| / (|g| + wd |p| + eps)  if wd != 0 and |p| > 0 and |g| > 0, else 1
    d = r (g + wd p)             (d = g when wd == 0)
    buf = d on the first step, else momentum buf + d
    p = p - lr buf

Only tensors with a nonzero decay are adapted, as timm does without ``always_adapt``.
"""
from __future__ import annotations

import math

import torch

from ..config import TRAIN

LAYERWISE = ("lamb", "lars")


def check_layerwise_decay(optimizer: str, weight_decay: float) -> None:
    """Refuse LAMB / LARS without a weight decay: no tensor would be adapted, and the run would silently be plain
    Adam / SGD with momentum."""
    if optimizer in LAYERWISE and not weight_decay > 0.0:
        raise ValueError("--optimizer %s adapts only tensors with a nonzero weight decay: with --weight-decay 0 it is "
                         "plain %s; give --weight-decay > 0 (--bias-weight-decay 0 keeps the biases unadapted)"
                         % (optimizer, "Adam" if optimizer == "lamb" else "SGD with momentum"))


class Lamb(torch.optim.Optimizer):
    def __init__(self, params, lr: float = 1e-3, betas=(TRAIN.lamb_beta1, TRAIN.lamb_beta2), eps: float = TRAIN.lamb_eps,
                 weight_decay: float = 0.0):
        if not lr >= 0.0 or not eps >= 0.0 or not weight_decay >= 0.0:
            raise ValueError("Lamb: lr, eps and weight_decay must be >= 0")
        super().__init__(params, dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay))

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for group in self.param_groups:
            group["step"] = group.get("step", 0) + 1
            b1, b2 = group["betas"]
            wd, t = group["weight_decay"], group["step"]
            bc1, bc2 = 1.0 - b1 ** t, 1.0 - b2 ** t
            for p in group["params"]:
                if p.grad is None:
                    continue
                g = p.grad
                st = self.state[p]
                if not st:
                    st["exp_avg"] = torch.zeros_like(p)
                    st["exp_avg_sq"] = torch.zeros_like(p)
                m, v = st["exp_avg"], st["exp_avg_sq"]
                m.mul_(b1).add_(g, alpha=1.0 - b1)
                v.mul_(b2).addcmul_(g, g, value=1.0 - b2)
                denom = (v.sqrt() / math.sqrt(bc2)).add_(group["eps"])
                u = (m / bc1).div_(denom)
                if wd != 0:
                    u.add_(p, alpha=wd)
                    pn, un = p.norm(2.0), u.norm(2.0)
                    one = torch.ones_like(pn)
                    u.mul_(torch.where(pn > 0, torch.where(un > 0, pn / un, one), one))
                p.add_(u, alpha=-group["lr"])
        return loss


class Lars(torch.optim.Optimizer):
    def __init__(self, params, lr: float = 1e-3, momentum: float = TRAIN.momentum, weight_decay: float = 0.0,
                 trust_coeff: float = TRAIN.lars_trust_coeff, eps: float = TRAIN.lars_eps):
        if not lr >= 0.0 or not momentum >= 0.0 or not weight_decay >= 0.0:
            raise ValueError("Lars: lr, momentum and weight_decay must be >= 0")
        super().__init__(params, dict(lr=lr, momentum=momentum, weight_decay=weight_decay, trust_coeff=trust_coeff,
                                      eps=eps))

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for group in self.param_groups:
            wd, mom = group["weight_decay"], group["momentum"]
            for p in group["params"]:
                if p.grad is None:
                    continue
                d = p.grad
                if wd != 0:
                    pn, gn = p.norm(2.0), d.norm(2.0)
                    one = torch.ones_like(pn)
                    r = group["trust_coeff"] * pn / (gn + pn * wd + group["eps"])
                    r = torch.where(pn > 0, torch.where(gn > 0, r, one), one)
                    d = d.add(p, alpha=wd).mul_(r)
                if mom != 0:
                    st = self.state[p]
                    if "momentum_buffer" not in st:
                        st["momentum_buffer"] = d.clone().detach()
                    else:
                        st["momentum_buffer"].mul_(mom).add_(d)
                    d = st["momentum_buffer"]
                p.add_(d, alpha=-group["lr"])
        return loss
