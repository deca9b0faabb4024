"""Orchestration: data -> model -> parallel wrapper -> optimizer -> Trainer.fit.

Reference: ``manage_training(args)`` (distributedVggf.py:200-236) -- pick the device, build the
train / validation DataManagers, derive ``num_classes`` from the training folder, print three
``[Info]`` banner lines (+ one when distributed), build the model, wrap it (DDP when the process
group exists, DataParallel otherwise), build Adam(lr) and run ``Trainer.fit``.

Same sequence and same banner here.  What changes: rank -> GPU binding, the single-GPU path is a
plain engine (no DataParallel), the engine is either ``NativeEngine`` (sm_90a kernels, fused
gradient all-reduce over peer memory) or the torch-op oracle, and checkpoint / resume / LR step /
JSONL logging are available as additive options.
"""
from __future__ import annotations

import json
import math
import os
import time

import torch

from .cli import input_sizes
from .data.loader import DataManager
from .models.vggf import build_oracle, freeze_leading_layers_, get_spec
from .parallel.ddp import FlatDDP
from .parallel.process_group import (device_name, distributed_is_initialized, init_distributed,
                                     pick_device)
from .trainer import Trainer
from .utils import checkpoint as ckpt
from .utils.lr_schedule import LRSchedule


def _want_native(args, device: torch.device) -> bool:
    if args.engine == "oracle":
        return False
    native_ok = device.type == "cuda" and torch.cuda.get_device_capability(device) == (9, 0)
    if args.engine == "native" and not native_ok:
        raise RuntimeError("--engine native needs an sm_90 (H100) GPU (got %s)" % device)
    if native_ok and getattr(args, "dtype", "bf16") == "fp32":
        # The sm_90a kernels compute in bf16 (fp32 master weights, moments and accumulators).  The reference's
        # fp32 arithmetic (distributedVggf.py:162-172) is served by the torch-op engine -- same model, same
        # bucketed gradient averaging (FlatDDP) -- until a wgmma tf32 path exists (DESIGN 2.3).
        if args.engine == "native":
            raise RuntimeError("--engine native computes in bf16; --dtype fp32 runs on --engine oracle (torch ops)")
        print("[Info] --dtype fp32: using the torch-op engine (the native kernels compute in bf16)", flush=True)
        return False
    return native_ok


def model_ema_decay(decay: float, world_size: int, mini_batch: int, accum_steps: int, ema_steps: int,
                    epochs: int) -> float:
    """The decay of one EMA update, as torchvision's classification reference adjusts --model-ema-decay
    (a decay per image) to the images seen between two updates; K = accum_steps = 1 is its formula."""
    adjust = world_size * mini_batch * accum_steps * ema_steps / epochs
    alpha = min(1.0, (1.0 - decay) * adjust)
    return 1.0 - alpha


def build_model_ema(module: torch.nn.Module, decay: float):
    """torchvision's ExponentialMovingAverage: AveragedModel with ema_avg, buffers averaged too."""
    from torch.optim.swa_utils import AveragedModel

    def ema_avg(avg_model_param, model_param, num_averaged):
        return decay * avg_model_param + (1 - decay) * model_param

    return AveragedModel(module, avg_fn=ema_avg, use_buffers=True)


def parameter_groups(model: torch.nn.Module, weight_decay: float, bias_weight_decay=None):
    """torchvision's set_weight_decay(custom_keys_weight_decay=[("bias", bias_weight_decay)]): the
    ``*.bias`` tensors in a group of their own at ``bias_weight_decay``, everything else at
    ``weight_decay``.  Without a bias decay, one group (the parent's layout of the optimizer state).
    Frozen parameters (``requires_grad`` off: --freeze-layers) are in no group, as a torch fine-tuning
    script leaves them out."""
    if bias_weight_decay is None:
        return [{"params": [p for p in model.parameters() if p.requires_grad], "weight_decay": weight_decay}]
    named = [(n, p) for n, p in model.named_parameters() if p.requires_grad]
    return [{"params": [p for n, p in named if not n.endswith(".bias")], "weight_decay": weight_decay},
            {"params": [p for n, p in named if n.endswith(".bias")], "weight_decay": bias_weight_decay}]


def build_optimizer(model_or_params, args):
    """The torch-op engine's optimizer.  The decay is always passed: AdamW's own default is 0.01."""
    wd = getattr(args, "weight_decay", 0.0)
    if isinstance(model_or_params, torch.nn.Module):
        params = parameter_groups(model_or_params, wd, getattr(args, "bias_weight_decay", None))
    else:
        params = [{"params": [p for p in model_or_params if p.requires_grad], "weight_decay": wd}]
    if args.optimizer == "sgd":
        return torch.optim.SGD(params, lr=args.learning_rate, momentum=args.momentum, weight_decay=wd)
    if args.optimizer == "adamw":
        return torch.optim.AdamW(params, lr=args.learning_rate, weight_decay=wd)
    if args.optimizer in ("lamb", "lars"):
        from .utils.optim import Lamb, Lars, check_layerwise_decay
        check_layerwise_decay(args.optimizer, wd)
        if args.optimizer == "lamb":
            return Lamb(params, lr=args.learning_rate, weight_decay=wd)
        return Lars(params, lr=args.learning_rate, momentum=args.momentum, weight_decay=wd)
    return torch.optim.Adam(params, lr=args.learning_rate, weight_decay=wd)     # distributedVggf.py:230


def manage_training(args) -> Trainer:
    device = pick_device(args.rank, args.no_cuda)
    if args.world_size > 1 and not distributed_is_initialized():
        init_distributed(args.init_url, args.rank, args.world_size, device,
                         getattr(args, "backend", None))

    if getattr(args, "synthetic", 0):
        # Rank 0 alone decides whether the set has to be generated, writes it into a temporary
        # directory and renames it into place; EVERY rank then passes the same barrier.  (A per-rank
        # isdir() test races with rank 0 creating the directory: a late rank would skip the barrier,
        # scan a half-written folder and pair rank 0's barrier with some other collective.)
        if args.rank == 0 and not os.path.isdir(os.path.join(args.root_dir, "TrainData")):
            import shutil

            from .data.synthetic import make_synthetic_imagefolder
            tmp = args.root_dir.rstrip("/") + ".tmp%d" % os.getpid()
            make_synthetic_imagefolder(tmp, train_per_class=args.synthetic,
                                       val_per_class=max(args.synthetic // 4, 1), seed=args.seed)
            os.makedirs(args.root_dir, exist_ok=True)
            for sub in sorted(os.listdir(tmp), reverse=True):     # TrainData last
                os.replace(os.path.join(tmp, sub), os.path.join(args.root_dir, sub))
            shutil.rmtree(tmp, ignore_errors=True)
        if distributed_is_initialized():
            torch.distributed.barrier()

    dm_kw = dict(world_size=args.world_size, rank=args.rank, pipeline=args.pipeline,
                 seed=args.seed, reference_order=args.reference_order,
                 decode_threads=getattr(args, "decode_threads", 8))
    sizes = input_sizes(args)
    train_data_mngr = DataManager(args.root_dir, args.mini_batch, train=True,
                                  mixup_alpha=getattr(args, "mixup_alpha", 0.0),
                                  cutmix_alpha=getattr(args, "cutmix_alpha", 0.0),
                                  resize_size=sizes["train_resize_size"], crop_size=sizes["train_crop_size"], **dm_kw)
    val_tta = getattr(args, "val_tta", "none")
    valid_data_mngr = DataManager(args.root_dir, args.mini_batch, train=False,
                                  shard_eval=getattr(args, "shard_eval", False),
                                  resize_size=sizes["val_resize_size"], crop_size=sizes["val_crop_size"],
                                  **dm_kw, **({} if val_tta == "none" else dict(tta=val_tta)))
    train_loader, valid_loader = train_data_mngr.get_loader(), valid_data_mngr.get_loader()

    num_classes = args.num_classes or train_data_mngr.number_classes
    print("[Info] number of classes: {}".format(num_classes))
    print("[Info] class labels: {}".format(train_data_mngr.class_names))
    print("[Info] Running instance {} using {}".format(args.rank, device_name(device)))
    if sizes != input_sizes(None):
        print("[Info] input sizes: train RandomResizedCrop {} -> crop {}, eval Resize {} -> crop {}".format(
            sizes["train_resize_size"], sizes["train_crop_size"], sizes["val_resize_size"], sizes["val_crop_size"]))
    stream = None
    if train_data_mngr.pipeline == "stream":
        stream = dict(pipeline="stream", decode_threads=train_loader.threads,
                      stream_fallback=train_loader.other_count + valid_loader.other_count)
        print("[Info] input pipeline: stream ({} decode threads, {} file(s) decoded by PIL at start-up)".format(
            stream["decode_threads"], stream["stream_fallback"]))
    if val_tta != "none":
        from .data.transforms import tta_views
        print("[Info] test-time augmentation: {} ({} views per image, mean of their softmaxes)".format(
            val_tta, len(tta_views(val_tta))))

    spec = get_spec(args.model, num_classes)
    pretrained = torch.load(args.pretrained, map_location="cpu") if args.pretrained else None
    freeze = spec.check_freeze_layers(getattr(args, "freeze_layers", 0))
    if freeze:
        frozen = spec.frozen_param_names(freeze)
        print("[Info] frozen layers: {} .. {} ({} layers, {} parameters)".format(
            frozen[0].rsplit(".", 1)[0], frozen[-1].rsplit(".", 1)[0], freeze,
            sum(math.prod(spec.param_shape(n)) for n in frozen)))

    if distributed_is_initialized():
        print("[Info] distributed training has been initialized")

    ema_decay = None
    if getattr(args, "model_ema", False):
        ema_decay = model_ema_decay(args.model_ema_decay, args.world_size, args.mini_batch,
                                    getattr(args, "accum_steps", 1), args.model_ema_steps, args.epochs)

    if _want_native(args, device):
        from .engine.native_engine import NativeEngine

        model = NativeEngine(spec, device=device, batch=args.mini_batch, lr=args.learning_rate,
                             optimizer=args.optimizer, momentum=args.momentum,
                             compute_dtype=args.dtype, allreduce=args.allreduce,
                             wire_dtype=args.wire_dtype, bucket_mb=args.bucket_mb, seed=args.seed,
                             pretrained_state=pretrained, profile=args.profile,
                             zero1={"auto": "auto", "on": True, "off": False}[getattr(args, "zero1", "auto")],
                             label_smoothing=getattr(args, "label_smoothing", 0.0), ema_decay=ema_decay,
                             weight_decay=getattr(args, "weight_decay", 0.0),
                             bias_weight_decay=getattr(args, "bias_weight_decay", None),
                             deterministic=getattr(args, "deterministic", False), freeze_layers=freeze,
                             powersgd_rank=getattr(args, "powersgd_rank", 0),
                             powersgd_start_iter=getattr(args, "powersgd_start_iter", 1000),
                             input_hw=sizes["train_crop_size"], eval_hw=sizes["val_crop_size"])
        optimizer = None            # fused into the engine
        model_ema = True if ema_decay is not None else None       # kept by the engine's optimizer kernels
        if model.world > 1:
            model.comm_timing(True)   # [Perf] line: all-reduce GB/s and fraction of the NVLink rate per epoch
    else:
        if getattr(args, "deterministic", False):
            torch.use_deterministic_algorithms(True)
            # dropout draws from the global generator, which nothing else seeds (each rank its own masks)
            torch.manual_seed(args.seed * 1000003 + args.rank)
        model = build_oracle(spec, seed=args.seed, pretrained_state=pretrained).to(device)
        freeze_leading_layers_(model, freeze)            # before FlatDDP: it buckets trainable tensors only
        if distributed_is_initialized():
            state = None
            if getattr(args, "powersgd_rank", 0):
                from .parallel import powersgd
                state = powersgd.make_state(args.powersgd_rank, args.powersgd_start_iter, args.seed)
            model = FlatDDP(model, bucket_cap_mb=args.bucket_mb, powersgd=state)
        optimizer = build_optimizer(model.module if isinstance(model, FlatDDP) else model, args)
        model_ema = None
        if ema_decay is not None:
            model_ema = build_model_ema(model.module if isinstance(model, FlatDDP) else model, ema_decay)

    teacher, distill = None, None
    if getattr(args, "distill_teacher", None):
        teacher, distill = build_teacher(args, spec, device, native=optimizer is None, crop=sizes["train_crop_size"],
                                         eval_crop=sizes["val_crop_size"])
        if optimizer is None:
            model.set_distillation(teacher, args.distill_alpha, args.distill_temperature)
            if val_tta != "none":
                teacher.set_val_tta(val_tta)          # its one-time score is taken like the student's

    if getattr(args, "eval_only", False) and model_ema is not None and not args.resume:
        raise ValueError("--eval-only --model-ema scores a checkpoint's EMA: pass --resume <checkpoint>")
    start_epoch = 1
    if args.resume:
        kw = {} if model_ema is None else dict(model_ema=model_ema, ema_required=getattr(args, "eval_only", False))
        if getattr(args, "eval_only", False):   # scoring needs no optimizer state: any frozen count will do
            kw["skip_frozen_mismatch"] = True
        start_epoch = ckpt.load_checkpoint(args.resume, model, optimizer, **kw) + 1
        print("[Info] resumed from {} at epoch {}".format(args.resume, start_epoch))

    schedule = LRSchedule.from_args(args)

    def set_lr(lr: float) -> None:
        if optimizer is not None:
            for g in optimizer.param_groups:
                g["lr"] = lr
        else:
            model.set_lr(lr)

    def current_lr() -> float:
        return optimizer.param_groups[0]["lr"] if optimizer is not None else model.lr

    if not schedule.constant:
        # the rate of the first epoch to run, on BOTH back ends: a warmup's first rate, or a resumed
        # run's rate behind the schedule's steps
        set_lr(schedule.lr_at(start_epoch - 1))

    def on_epoch_end(epoch: int, trainer: Trainer) -> None:
        epoch_lr = current_lr()
        if not schedule.constant:
            set_lr(schedule.lr_at(epoch))
        if args.save:
            kw = {} if model_ema is None else dict(model_ema=model_ema)
            ckpt.save_checkpoint(args.save, model, optimizer, epoch, vars(args),
                                 is_rank0=(args.rank == 0), **kw)
            # rank 0 is busy with a ~1.6 GB D2H copy + torch.save: hold the other ranks HERE, on the
            # host, instead of letting them spin inside the next epoch's first all-reduce kernel
            if distributed_is_initialized():
                torch.distributed.barrier()
        if args.log_jsonl and args.rank == 0:
            rec = dict(trainer.history[-1], time=time.time(), world_size=args.world_size)
            if sizes != input_sizes(None):
                rec["input_sizes"] = sizes
            if val_tta != "none":
                rec["val_tta"] = val_tta
            if stream is not None:
                rec.update(stream)
            if not schedule.constant:
                rec["lr"] = epoch_lr
            if hasattr(model, "phase_times"):
                rec["phase_ms"] = model.phase_times()
            if distill is not None:
                rec.update(distill=distill, teacher_test_acc=teacher_acc.accuracy)
            for key in ("epoch_host_times", "epoch_allreduce"):       # set by Trainer for native engines
                if getattr(trainer, key, None):
                    rec[key[len("epoch_"):]] = getattr(trainer, key)
            with open(args.log_jsonl, "a") as f:
                f.write(json.dumps(rec) + "\n")

    cw = None
    if getattr(args, "class_weights", None):
        cw = torch.tensor([float(v) for v in args.class_weights.split(",")], dtype=torch.float32)
        if cw.numel() != num_classes:
            raise ValueError("--class-weights needs %d comma-separated values" % num_classes)
    trainer = Trainer(model, optimizer, train_loader, valid_loader, device, class_weights=cw,
                      on_epoch_end=on_epoch_end, shard_eval=getattr(args, "shard_eval", False),
                      accum_steps=getattr(args, "accum_steps", 1),
                      label_smoothing=getattr(args, "label_smoothing", 0.0), model_ema=model_ema,
                      model_ema_steps=getattr(args, "model_ema_steps", 32),
                      teacher=teacher if optimizer is not None else None,
                      distill_alpha=getattr(args, "distill_alpha", 0.5),
                      distill_temperature=getattr(args, "distill_temperature", 4.0), val_tta=val_tta,
                      val_metrics=getattr(args, "val_metrics", False),
                      class_names=val_class_names(valid_data_mngr.class_names, num_classes))
    trainer.profile_timeline = getattr(args, "profile", None) == "timeline"
    if getattr(args, "eval_only", False):        # score a checkpoint: one validation pass, no training
        test_loss, test_acc = trainer._evaluate()
        print("[Info] Evaluation: test loss: {}, test acc: {}.".format(test_loss, test_acc), flush=True)
        rec = dict(epoch=start_epoch - 1, test_loss=test_loss.average, test_acc=test_acc.accuracy)
        if val_tta != "none":
            rec["val_tta"] = val_tta
        classes = {}
        trainer.report_classes("Evaluation: ", "test", test_acc, classes, "test")
        if model_ema is not None:
            ema_loss, ema_acc = trainer._evaluate(ema=True)
            print("[Info] Evaluation: EMA test loss: {}, EMA test acc: {}.".format(ema_loss, ema_acc), flush=True)
            rec.update(ema_test_loss=ema_loss.average, ema_test_acc=ema_acc.accuracy)
            trainer.report_classes("Evaluation: ", "EMA test", ema_acc, classes, "ema_test")
        rec.update(classes)
        trainer.history.append(rec)
        return trainer
    if teacher is not None:
        # a teacher trained on another class order scores near chance here
        teacher_loss, teacher_acc = trainer._evaluate(model=teacher)
        print("[Info] distillation: teacher {} from {} (alpha {}, temperature {}): test loss {}, test acc {}.".format(
            distill["model"], distill["path"], distill["alpha"], distill["temperature"], teacher_loss, teacher_acc),
            flush=True)
    trainer.fit(args.epochs, start_epoch=start_epoch)
    return trainer


def val_class_names(names, num_classes: int) -> list:
    """The --val-metrics row names: the validation folder's classes (its order numbers the labels), by index past
    them when --num-classes asks for more."""
    names = list(names)[:num_classes]
    return names + [str(c) for c in range(len(names), num_classes)]


def build_teacher(args, spec, device: torch.device, native: bool, crop: int, eval_crop: int):
    """The --distill-teacher model, loaded whole by this rank (every rank reads the same file, as --pretrained):
    a forward-only ``TeacherEngine`` on the native engine, an eval-mode ``VGGOracle`` without gradients on the
    torch-op engine (fp32).  Returns (teacher, the JSONL record's ``distill`` entry)."""
    name, state = ckpt.load_teacher_state(args.distill_teacher, spec.num_classes,
                                          getattr(args, "distill_teacher_model", None), args.model)
    tspec = get_spec(name, spec.num_classes)
    info = dict(path=args.distill_teacher, model=name, alpha=args.distill_alpha, temperature=args.distill_temperature)
    if native:
        from .engine.native_engine import TeacherEngine
        try:
            teacher = TeacherEngine(tspec, device, args.mini_batch, state, input_hw=crop, eval_hw=eval_crop,
                                    deterministic=getattr(args, "deterministic", False))
        except ValueError as e:
            raise ValueError("--distill-teacher-model %s: the native engine cannot run it (%s)" % (name, e)) from None
        print("[Info] distillation teacher: {} ({} parameters), {:.1f} MB of device memory, forward only".format(
            name, tspec.num_params, teacher.device_bytes() / 1e6), flush=True)
        return teacher, info
    teacher = build_oracle(tspec, seed=0).to(device)       # its own generator: the global RNG stays untouched
    teacher.load_state_dict(state)
    teacher.eval().requires_grad_(False)
    return teacher, info
