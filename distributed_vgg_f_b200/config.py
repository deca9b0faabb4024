"""Framework-wide defaults.

Parity notes (reference: distributedUtil.py:12-25): the reference keeps its defaults as module
constants -- 20 epochs, Adam lr 1e-3, mini-batch 16, the ``TrainData`` / ``ValidationData``
directory names -- plus three vestigial SGD/StepLR constants it never reads.  We keep the same
defaults, but grouped in frozen dataclasses, and the SGD/StepLR values are *live* here: they
configure the optional fused SGD optimizer and the optional step LR schedule.
"""
from __future__ import annotations

import dataclasses


@dataclasses.dataclass(frozen=True)
class TrainDefaults:
    epochs: int = 20               # distributedUtil.py:14
    learning_rate: float = 1e-3    # distributedUtil.py:15
    mini_batch: int = 16           # distributedUtil.py:20
    # Optional SGD path (the reference defines these but never uses them, distributedUtil.py:16-18).
    momentum: float = 0.9
    decay_step_size: int = 7
    decay_gamma: float = 0.1
    # Adam hyper-parameters = torch.optim.Adam defaults (distributedVggf.py:230).
    adam_beta1: float = 0.9
    adam_beta2: float = 0.999
    adam_eps: float = 1e-8
    # LAMB and LARS (--optimizer lamb|lars) as timm's Lamb / Lars with their defaults: bias correction on,
    # no trust clipping, only tensors with a nonzero decay adapted.
    lamb_beta1: float = 0.9
    lamb_beta2: float = 0.999
    lamb_eps: float = 1e-6
    lars_trust_coeff: float = 1e-3
    lars_eps: float = 1e-8


@dataclasses.dataclass(frozen=True)
class DataDefaults:
    train_dir: str = "TrainData"          # distributedUtil.py:22-25
    val_dir: str = "ValidationData"
    resize: int = 256                     # distributedVggf.py:89, :104
    crop: int = 224                       # distributedVggf.py:92, :105
    crop_scale: tuple = (0.8, 1.0)        # distributedVggf.py:89
    crop_ratio: tuple = (3.0 / 4.0, 4.0 / 3.0)
    rotation_deg: float = 10.0            # distributedVggf.py:90
    mean: tuple = (0.485, 0.456, 0.406)   # distributedVggf.py:94
    std: tuple = (0.229, 0.224, 0.225)


TRAIN = TrainDefaults()
DATA = DataDefaults()

# Control-plane backend used for rendezvous.  The reference hard-codes "gloo"
# (distributedUtil.py:12); we pick nccl when every rank owns a GPU and gloo otherwise.
CPU_BACKEND = "gloo"
GPU_BACKEND = "nccl"

# Compile target for every CUDA source in csrc/.
CUDA_ARCH_FLAGS = ("-gencode", "arch=compute_90a,code=sm_90a")
