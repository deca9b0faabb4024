"""Checkpoint save / resume.

The reference has no checkpointing at all (no torch.save / load / state_dict anywhere; SURVEY D1,
5.4).  The only layout that is "the same" as anything the reference could produce is the
``state_dict()`` of its wrapped model: both ``DistributedDataParallel`` (ws > 1,
distributedVggf.py:225) and ``DataParallel`` (ws == 1, :227) prefix every key with ``module.``, and
the tensors carry torchvision's VGG names and shapes plus the funnel
(``module.features.0.weight`` ... ``module.classifier.6.3.bias``, 34 tensors).  We therefore write

    {"model": {module.<torchvision name>: fp32 tensor in torch layout},
     "optimizer": {"name", "step", "exp_avg": {...}, "exp_avg_sq": {...} | "momentum_buffer": {...}},
     "epoch": int, "args": dict, "format": "distributed-vgg-f_b200/1"}

with ``torch.save`` on rank 0 only.  ``strip_module_prefix(ckpt["model"])`` loads directly into the
reference's *unwrapped* model object (``vgg_funnel_model(C).load_state_dict``).  The native engine
stores conv weights as OHWI and FC-1 columns in NHWC-flatten order; conversion to / from the torch
layout happens here (``engine.export_state`` / ``import_state``).

With ``--model-ema`` the payload also holds ``"model_ema"``: ``{"n_averaged": int64 tensor,
module.<torchvision name>: fp32 tensor, ...}``, the keys of torchvision's
``AveragedModel(vgg_funnel_model(C)).state_dict()``, so that it loads into one directly.
"""
from __future__ import annotations

import os
from typing import Any, Dict, Optional

import torch

FORMAT = "distributed-vgg-f_b200/1"


def add_module_prefix(state: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    return {(k if k.startswith("module.") else "module." + k): v for k, v in state.items()}


def strip_module_prefix(state: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    return {(k[len("module."):] if k.startswith("module.") else k): v for k, v in state.items()}


def model_state(model) -> Dict[str, torch.Tensor]:
    if hasattr(model, "export_state"):              # NativeEngine
        state = model.export_state()
    else:
        state = model.state_dict()
    return add_module_prefix({k: v.detach().to("cpu", torch.float32) for k, v in state.items()})


def frozen_layers_of(model) -> int:
    """The --freeze-layers count of a native engine or of a torch model (leading layers without gradients)."""
    if hasattr(model, "freeze_layers"):
        return int(model.freeze_layers)
    module = model.module if hasattr(model, "module") and not hasattr(model, "features") else model
    if not hasattr(module, "spec"):
        return 0
    from ..models.vggf import count_frozen_layers
    return count_frozen_layers(module)


def optimizer_state(model, optimizer) -> Dict[str, Any]:
    if hasattr(model, "export_optimizer_state"):
        return model.export_optimizer_state()
    if optimizer is None:
        return {}
    st = optimizer.state_dict()
    frozen = frozen_layers_of(model)
    if frozen:                 # as the native engine records it; absent without frozen layers
        st["frozen_layers"] = frozen
    return st


def _check_frozen(path: str, st: dict, model) -> bool:
    """Does the optimizer state ``st`` belong to this run's frozen layers?  Raises when it does not."""
    theirs, mine = int(st.get("frozen_layers", 0)), frozen_layers_of(model)
    if theirs != mine:
        raise ValueError("%s: its optimizer state was written with --freeze-layers %d, this run has --freeze-layers "
                         "%d: resume with %d (or evaluate it with --eval-only)" % (path, theirs, mine, theirs))
    return True


def ema_state(model, model_ema) -> Dict[str, torch.Tensor]:
    """The ``"model_ema"`` entry: an AveragedModel's state dict (torch path), or the native engine's EMA
    (``model_ema`` is then True) under the same keys."""
    if isinstance(model_ema, torch.nn.Module):
        return {k: (v.detach().cpu() if k == "n_averaged" else v.detach().to("cpu", torch.float32))
                for k, v in model_ema.state_dict().items()}
    state = {"n_averaged": torch.tensor(model.ema_updates, dtype=torch.int64)}
    state.update(add_module_prefix(model.export_ema_state()))
    return state


def save_checkpoint(path: str, model, optimizer, epoch: int, args: Optional[dict] = None,
                    is_rank0: bool = True, model_ema=None) -> None:
    if hasattr(model, "prepare_export"):     # collective: engines with sharded optimizer state gather it
        model.prepare_export()
    if not is_rank0:
        return
    payload = {"format": FORMAT, "model": model_state(model),
               "optimizer": optimizer_state(model, optimizer), "epoch": int(epoch),
               "args": dict(args or {})}
    if model_ema is not None:
        payload["model_ema"] = ema_state(model, model_ema)
    tmp = path + ".tmp"
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    torch.save(payload, tmp)
    os.replace(tmp, path)


def load_checkpoint(path: str, model, optimizer=None, model_ema=None, ema_required: bool = False,
                    skip_frozen_mismatch: bool = False) -> int:
    """Restore model (+ optimizer, + the EMA when ``model_ema`` is given) and return the epoch to resume
    *after*.  A checkpoint without an EMA leaves the EMA fresh, or fails with ``ema_required``.  An optimizer
    state written with a different --freeze-layers count is refused (per-parameter Adam step counts make
    "unfreeze and continue" a different optimizer), or with ``skip_frozen_mismatch`` (evaluation) not loaded."""
    # our files hold tensors and plain containers only: no need to unpickle arbitrary objects
    payload = torch.load(path, map_location="cpu", weights_only=True)
    if model_ema is not None:
        ema = payload.get("model_ema") if isinstance(payload, dict) else None
        if ema is None:
            if ema_required:
                raise ValueError("%s holds no model EMA (it was not saved with --model-ema)" % path)
            print("[Info] %s holds no model EMA: the EMA starts fresh" % path, flush=True)
        elif isinstance(model_ema, torch.nn.Module):
            model_ema.load_state_dict(ema)
        else:
            model.import_ema_state(strip_module_prefix({k: v for k, v in ema.items() if k != "n_averaged"}),
                                   int(ema["n_averaged"]))
    state = payload["model"] if "model" in payload else payload
    opt = payload.get("optimizer") if isinstance(payload, dict) else None
    if opt and skip_frozen_mismatch and int(opt.get("frozen_layers", 0)) != frozen_layers_of(model):
        opt = None
    if hasattr(model, "import_state"):
        model.import_state(strip_module_prefix(state))
        if "optimizer" in payload and opt:
            model.import_optimizer_state(opt)
    else:
        target = model.module if hasattr(model, "module") and not hasattr(model, "features") else model
        target.load_state_dict(strip_module_prefix(state))
        if optimizer is not None and opt and _check_frozen(path, opt, model):
            optimizer.load_state_dict({k: v for k, v in opt.items() if k != "frozen_layers"})
    return int(payload.get("epoch", 0))


def load_teacher_state(path: str, num_classes: int, model: Optional[str] = None, student_model: str = "vggf"):
    """The teacher of --distill-teacher: (model name, torch-layout fp32 state dict).  ``path`` holds a checkpoint of
    this project (``{"model": {"module.<name>": ...}, "args": {...}}``) or a plain state dict with torchvision names.
    The model is ``model`` when given, else the checkpoint's ``args["model"]``, else ``student_model``.  Unlike
    --pretrained, the file must be the whole model: a missing, unexpected or misshapen tensor is refused, and so is
    a class count other than ``num_classes``."""
    from ..models.vggf import get_spec

    if not os.path.isfile(path):
        raise FileNotFoundError("--distill-teacher %s: no such file" % path)
    payload = torch.load(path, map_location="cpu", weights_only=True)
    if not isinstance(payload, dict):
        raise ValueError("--distill-teacher %s: not a checkpoint or a state dict" % path)
    ours = isinstance(payload.get("model"), dict)
    state = strip_module_prefix(payload["model"] if ours else payload)
    saved = payload.get("args") if ours and isinstance(payload.get("args"), dict) else {}
    name = model or saved.get("model") or student_model
    spec = get_spec(name, num_classes)
    head = spec.fcs[-1].name + ".weight"
    if head in state and state[head].dim() == 2 and state[head].shape[0] != num_classes:
        raise ValueError("--distill-teacher %s: the teacher has %d classes, the student %d"
                         % (path, state[head].shape[0], num_classes))
    missing = [n for n in spec.param_names if n not in state]
    unexpected = sorted(set(state) - set(spec.param_names))
    wrong = [n for n in spec.param_names if n in state and tuple(state[n].shape) != tuple(spec.param_shape(n))]
    if missing or unexpected or wrong:
        raise ValueError("--distill-teacher %s does not hold a whole %s: missing %s, unexpected %s, wrong shape %s"
                         % (path, name, missing[:4] or "none", unexpected[:4] or "none",
                            ["%s %s (want %s)" % (n, tuple(state[n].shape), tuple(spec.param_shape(n)))
                             for n in wrong[:4]] or "none"))
    return name, {n: state[n].detach().to(torch.float32) for n in spec.param_names}
