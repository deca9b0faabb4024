"""The learning rate of every epoch, for both engines.

torchvision's classification recipe steps its schedulers once per epoch: ``SequentialLR(warmup, main,
milestones=[W])`` when ``--lr-warmup-epochs W > 0``, else ``main`` alone, where ``warmup`` is
``LinearLR(start_factor=decay, total_iters=W)`` or ``ConstantLR(factor=decay, total_iters=W)`` and
``main`` is ``StepLR(step, gamma)`` or ``CosineAnnealingLR(T_max=epochs - W, eta_min=lr_min)``.  The
native engine has no torch optimizer to attach schedulers to, so the rate is computed here in closed
form and handed to both engines: ``lr_at(k)`` is the rate after k scheduler steps, i.e. the rate of
epoch k + 1.  StepLR without warmup is ``base_lr * gamma ** (k // step)``, bit for bit; ``--lr-step 0``
keeps the rate constant, as it always has.
"""
from __future__ import annotations

import dataclasses
import math


@dataclasses.dataclass(frozen=True)
class LRSchedule:
    base_lr: float
    epochs: int
    scheduler: str = "step"           # step | cosine
    step: int = 0                     # StepLR period in epochs (0: constant)
    gamma: float = 0.1
    lr_min: float = 0.0               # CosineAnnealingLR's eta_min
    warmup_epochs: int = 0
    warmup_method: str = "constant"   # linear | constant
    warmup_decay: float = 0.01

    @classmethod
    def from_args(cls, args) -> "LRSchedule":
        return cls(base_lr=args.learning_rate, epochs=args.epochs,
                   scheduler=getattr(args, "lr_scheduler", "step"), step=args.lr_step, gamma=args.lr_gamma,
                   lr_min=getattr(args, "lr_min", 0.0), warmup_epochs=getattr(args, "lr_warmup_epochs", 0),
                   warmup_method=getattr(args, "lr_warmup_method", "constant"),
                   warmup_decay=getattr(args, "lr_warmup_decay", 0.01))

    @property
    def constant(self) -> bool:
        """True when every epoch runs at base_lr (the default): nothing needs setting."""
        return self.scheduler == "step" and not self.step and not self.warmup_epochs

    def _main(self, k: int) -> float:
        if self.scheduler == "cosine":
            t_max = self.epochs - self.warmup_epochs
            return self.lr_min + (self.base_lr - self.lr_min) * (1 + math.cos(math.pi * k / t_max)) / 2
        if not self.step:
            return self.base_lr
        return self.base_lr * (self.gamma ** (k // self.step))

    def lr_at(self, k: int) -> float:
        """The rate after k per-epoch scheduler steps: the rate of (1-based) epoch k + 1."""
        W = self.warmup_epochs
        if W and k < W:
            if self.warmup_method == "linear":
                return self.base_lr * (self.warmup_decay + (1.0 - self.warmup_decay) * k / W)
            return self.base_lr * self.warmup_decay
        return self._main(k - W)
