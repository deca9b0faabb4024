"""Training / evaluation loops.

Reference (distributedVggf.py:126-197): ``Trainer(model, optimizer, train_loader, test_loader,
device).fit(epochs)`` -- per batch: H2D, forward, cross-entropy, zero_grad, backward, step, two
``.item()`` syncs; per epoch: a full (unsharded) validation pass on every rank and one report line
``[Info] Epoch: e/E, train loss: .., train acc: ..%, test loss: .., test acc: ..%.``.

``Trainer`` keeps the constructor, ``fit`` and the report line, for two interchangeable back ends:
  * a torch ``nn.Module`` (optionally wrapped in ``parallel.ddp.FlatDDP``) -- the oracle / CPU path;
  * ``engine.NativeEngine`` -- the sm_90a path, where forward, loss, backward, gradient
    all-reduce and optimizer are one ``train_step`` call and metrics stay on the device.
Differences kept on purpose: metrics accumulate on the device and are read once per epoch
(``DeviceMeter``), ``set_epoch`` is called so shuffling changes between epochs, and throughput is
reported on an extra line.

``label_smoothing`` and batches that carry a MixUp / CutMix draw (``data.transforms.MixDraw``): on the
torch path the images are mixed by torchvision and the loss is ``F.cross_entropy(outputs, targets,
weight=, label_smoothing=)`` with torchvision's probability targets, as its classification reference
script does; the native engine does the same in its kernels.  The test loss stays plain cross-entropy.

``accum_steps=K`` (gradient accumulation): one optimizer update per group of K consecutive training
mini-batches, and after the epoch's last one, so the last group of an epoch may be shorter (k' < K) and
no group crosses an epoch boundary.  Each mini-batch's loss is its own mean; the update uses the sum of
the group's gradients divided by k'.  Metrics count every mini-batch.

``teacher`` (knowledge distillation, torch path; the native engine has its own, ``set_distillation``): an
eval-mode module without gradients run under ``no_grad`` on the (mixed) training inputs; the training loss is
(1 - a) CE + a T^2 F.kl_div(log_softmax(s / T), log_softmax(t / T), "batchmean", log_target=True) with CE as above,
and the train meter accumulates it.  Accuracy and the test loss stay those of the labels.

``model_ema`` (torchvision's --model-ema): after the optimizer update whose 0-based index u within the
epoch has u % model_ema_steps == 0, the moving average of the weights is updated -- by the native engine's
optimizer kernels (``model_ema=True``, ``train_step(ema=True)``), or on the torch path by
``model_ema.update_parameters`` (an ``AveragedModel``) after ``optimizer.step()``.  Every epoch the
average is evaluated after the raw weights: ``[Info] Epoch: e/E, EMA test loss: .., EMA test acc: ..%.``

``val_metrics`` (--val-metrics): the validation passes of the weights and of the EMA count a confusion matrix and
the top-5 hits (``DeviceMeter(num_classes=)``), and each of their report lines is followed by the lines of
``utils.metrics.class_report``; the history gets ``test_*`` / ``ema_test_*`` keys of ``utils.metrics.class_metrics``.
``class_names`` name the rows (the validation folder's classes, which number the labels).
"""
from __future__ import annotations

import time
from typing import Optional

import torch
import torch.nn.functional as F

from .config import DATA
from .data import transforms as T
from .data.loader import DEVICE_BATCHES
from .utils.metrics import DeviceMeter, class_report


def _bf16_peak() -> float:
    """bf16 TFLOP/s to report utilisation against: MEASURED_PEAKS.json next to the package when a
    measurement of this machine is there, else the H100 SXM data-sheet dense bf16 rate."""
    import json
    import os
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")
    try:
        with open(path) as f:
            d = json.load(f)
        for key in ("bf16_tflops_sustained", "cublas_bf16_tflops_sustained", "bf16_tflops"):
            if key in d:
                return float(d[key])
    except (OSError, ValueError):
        pass
    return 989.0


def sys_stdout_flush() -> None:
    import sys
    sys.stdout.flush()


def distill_loss(student: torch.Tensor, teacher: torch.Tensor, ce: torch.Tensor, alpha: float,
                 temperature: float) -> torch.Tensor:
    """(1 - alpha) ce + alpha T^2 KL(softmax(teacher / T) || softmax(student / T)), the KL a batch mean."""
    T = float(temperature)
    kl = F.kl_div(F.log_softmax(student / T, 1), F.log_softmax(teacher / T, 1), reduction="batchmean", log_target=True)
    return (1.0 - alpha) * ce + alpha * T * T * kl


def _is_native(model) -> bool:
    return hasattr(model, "train_step") and hasattr(model, "eval_step")


class Trainer:
    def __init__(self, model, optimizer, train_loader, test_loader, device,
                 class_weights: Optional[torch.Tensor] = None, verbose_throughput: bool = True,
                 on_epoch_end=None, shard_eval: bool = False, accum_steps: int = 1,
                 label_smoothing: float = 0.0, model_ema=None, model_ema_steps: int = 32, teacher=None,
                 distill_alpha: float = 0.5, distill_temperature: float = 4.0, val_tta: str = "none",
                 val_metrics: bool = False, class_names=None) -> None:
        if accum_steps < 1:
            raise ValueError("accum_steps must be >= 1 (got %d)" % accum_steps)
        if accum_steps > 1 and not hasattr(train_loader, "__len__"):
            raise ValueError("accum_steps > 1 needs a training loader with __len__: the last group of an epoch "
                             "ends at its last batch")
        self.accum_steps = int(accum_steps)
        self.label_smoothing = float(label_smoothing)      # torch path; the native engine has its own
        if model_ema_steps < 1:
            raise ValueError("model_ema_steps must be >= 1 (got %d)" % model_ema_steps)
        if model_ema is not None and _is_native(model) and getattr(model, "ema32", None) is None:
            raise ValueError("model_ema on the native engine needs NativeEngine(ema_decay=...)")
        self.model_ema = model_ema          # AveragedModel (torch path), True (native engine) or None
        self.model_ema_steps = int(model_ema_steps)
        self.teacher = teacher              # torch path: the distillation teacher (an eval-mode module)
        self.distill_alpha, self.distill_temperature = float(distill_alpha), float(distill_temperature)
        self.model = model
        self.optimizer = optimizer
        self.train_loader = train_loader
        self.test_loader = test_loader
        self.device = device
        # The reference carries a commented-out class-weighted loss (distributedVggf.py:164-166).
        self.class_weights = class_weights.to(device) if class_weights is not None else None
        self.verbose_throughput = verbose_throughput
        self.on_epoch_end = on_epoch_end
        self.shard_eval = shard_eval
        if self.class_weights is not None and _is_native(model):
            model.set_class_weights(self.class_weights)
        # --val-tta: every validation pass scores the mean softmax of the mode's views (the native engine loops them
        # itself once told; the torch path below); training is untouched
        T.tta_views(val_tta)
        self.val_tta = val_tta
        if val_tta != "none" and _is_native(model):
            model.set_val_tta(val_tta)
        if val_metrics and not class_names:
            raise ValueError("val_metrics needs the class names, one per class")
        self.val_metrics = bool(val_metrics)
        self.class_names = list(class_names) if class_names is not None else None
        self.history = []

    def report_classes(self, head: str, what: str, acc, rec: dict, key: str) -> None:
        """--val-metrics: print the per-class lines of an evaluation pass after its report line and add its
        ``<key>_*`` entries to ``rec``."""
        if acc.classes is None:
            return
        for line in class_report(head, what, acc.classes, self.class_names):
            print(line)
        sys_stdout_flush()
        rec.update({key + "_" + k: v for k, v in acc.classes.items()})

    # ------------------------------------------------------------------------------------------
    def fit(self, epochs: int, start_epoch: int = 1) -> None:
        for epoch in range(start_epoch, epochs + 1):
            for ld in (self.train_loader, self.test_loader):
                if hasattr(ld, "set_epoch"):
                    ld.set_epoch(epoch - 1)
            t0 = time.perf_counter()
            train_loss, train_acc = self._train()
            t1 = time.perf_counter()
            test_loss, test_acc = self._evaluate()
            print(
                "[Info] Epoch: {}/{},".format(epoch, epochs),
                "train loss: {}, train acc: {},".format(train_loss, train_acc),
                "test loss: {}, test acc: {}.".format(test_loss, test_acc),
                flush=True,
            )
            head = "Epoch: {}/{}, ".format(epoch, epochs)
            classes = {}
            self.report_classes(head, "test", test_acc, classes, "test")
            ema_s = 0.0
            if self.model_ema is not None:
                te = time.perf_counter()
                ema_loss, ema_acc = self._evaluate(ema=True)
                print("[Info] Epoch: {}/{}, EMA test loss: {}, EMA test acc: {}.".format(epoch, epochs, ema_loss,
                                                                                      ema_acc), flush=True)
                self.report_classes(head, "EMA test", ema_acc, classes, "ema_test")
                ema_s = time.perf_counter() - te
            if self.verbose_throughput and train_loss.count:
                print("[Perf] Epoch: {}/{}, train images/sec (this rank): {:.1f}{}{}".format(
                    epoch, epochs, train_loss.count / max(t1 - t0, 1e-9),
                    self._utilisation(train_loss.count, t1 - t0), self._comm_line()), flush=True)
                ht = getattr(self, "epoch_host_times", None)
                if ht:
                    print("[Perf] Epoch: {}/{}, host: first batch after {:.1f} ms, steps enqueued in {:.1f} ms, "
                          "GPU drained {:.1f} ms later; validation pass {:.1f} ms".format(
                              epoch, epochs, ht["first_batch_ms"], ht["enqueue_ms"], ht["drain_ms"],
                              1e3 * (time.perf_counter() - t1 - ema_s)), flush=True)
            self.history.append(dict(epoch=epoch, train_loss=train_loss.average,
                                     train_acc=train_acc.accuracy, test_loss=test_loss.average,
                                     test_acc=test_acc.accuracy))
            if self.model_ema is not None:
                self.history[-1].update(ema_test_loss=ema_loss.average, ema_test_acc=ema_acc.accuracy)
            self.history[-1].update(classes)
            if self.on_epoch_end is not None:
                self.on_epoch_end(epoch, self)

    @staticmethod
    def _print_timeline(rows) -> None:
        """--profile timeline: one line per mark, compute stream first, then the side streams."""
        if not rows:
            return
        print("[Timeline] last training step of the epoch, ms since its start (CUDA events)", flush=True)
        prev = 0.0
        for name, lane, ms in rows:
            if lane == "compute":
                print("[Timeline]   compute %-26s %8.3f  +%.3f" % (name, ms, ms - prev))
                prev = ms
        for name, lane, ms in rows:
            if lane != "compute":
                print("[Timeline]   %-7s %-26s %8.3f" % (lane, name, ms))
        sys_stdout_flush()

    def _comm_line(self) -> str:
        """Gradient all-reduce of the epoch as the step saw it: bus GB/s and fraction of the NVLink rate
        (SURVEY 5.5).  Needs ``engine.comm_timing(True)`` (the CLI's --profile comm)."""
        rep = getattr(self.model, "comm_report", None)
        steps = len(self.train_loader) if hasattr(self.train_loader, "__len__") else 0
        updates = -(-steps // self.accum_steps)          # the all-reduces run once per update
        r = rep(max(updates, 1)) if rep is not None else None
        self.epoch_allreduce = r
        if not r:
            return ""
        return ", grad all-reduce {:.0f} MB/{} in {:.2f} ms = {:.0f} GB/s bus ({:.0f}% of 450 nominal)".format(
            r["wire_MB_per_step"], "step" if self.accum_steps == 1 else "update", r["ms_per_step"], r["bus_GBs"],
            100 * r["frac_of_450_nominal"])

    def _utilisation(self, images: int, seconds: float) -> str:
        """Native engine only: achieved training TFLOP/s (3 x forward FLOPs of the layer table) and
        its fraction of the measured bf16 peak (MEASURED_PEAKS.json next to the package, if any)."""
        spec, hw = getattr(self.model, "spec", None), getattr(self.model, "HW", None)
        if not _is_native(self.model) or spec is None or not hw or seconds <= 0:
            return ""
        tflops = 3.0 * spec.flops_per_image(hw) * images / seconds / 1e12
        return ", {:.0f} TFLOP/s ({:.0f}% of the bf16 peak)".format(tflops, 100.0 * tflops / _bf16_peak())

    # ------------------------------------------------------------------------------------------
    def _to_device(self, batch, loader=None):
        if isinstance(batch, DEVICE_BATCHES):     # cut to the network input its loader is set to
            return batch.to_float(self.device, out_hw=getattr(loader, "crop", DATA.crop))
        inputs, targets = batch[0], batch[1]
        return inputs.to(self.device, non_blocking=True), targets.to(self.device, non_blocking=True)

    def _mixed_to_device(self, batch):
        """(inputs, integer targets, probability targets or None) of a training batch: the batch's
        MixUp / CutMix draw applied by torchvision (the reference pipeline has applied it already)."""
        mix = batch.mix if isinstance(batch, DEVICE_BATCHES) else (batch[2] if len(batch) > 2 else None)
        inputs, targets = self._to_device(batch, self.train_loader)
        if mix is None:
            return inputs, targets, None
        if isinstance(batch, DEVICE_BATCHES):
            inputs = T.apply_mix(inputs, targets, mix)
        return inputs, targets, mix

    def _updates_after(self, k: int, n_steps: int) -> bool:
        """Does the (k+1)-th training batch of an epoch of ``n_steps`` end its accumulation group?"""
        return (k + 1) % self.accum_steps == 0 or k + 1 == n_steps

    def _ema_after(self, u: int) -> bool:
        """Does the epoch's optimizer update of 0-based index ``u`` update the EMA?"""
        return self.model_ema is not None and u % self.model_ema_steps == 0

    def _train(self):
        meter = DeviceMeter(self.device)
        if _is_native(self.model):
            self.model.set_meter(meter)
            t0 = time.perf_counter()
            first = None
            want_tl = getattr(self, "profile_timeline", False) and hasattr(self.model, "timeline")
            n_steps = len(self.train_loader) if hasattr(self.train_loader, "__len__") else 0
            u = 0                                          # optimizer updates so far in this epoch
            for k, batch in enumerate(self.train_loader):
                if first is None:
                    first = time.perf_counter() - t0       # loader start-up: time to the first batch
                if want_tl and k == n_steps - 1:           # trace the epoch's last step
                    self.model.sync()
                    self.model.timeline(True)
                if self.accum_steps == 1 or self._updates_after(k, n_steps):
                    if self._ema_after(u):
                        self.model.train_step(batch, ema=True)
                    else:
                        self.model.train_step(batch)
                    u += 1
                else:
                    self.model.train_step(batch, update=False)
            t1 = time.perf_counter()
            self.model.sync()
            if want_tl:
                self._print_timeline(self.model.timeline_report())
                self.model.timeline(False)
            self.epoch_host_times = {"first_batch_ms": 1e3 * (first or 0.0), "enqueue_ms": 1e3 * (t1 - t0),
                                     "drain_ms": 1e3 * (time.perf_counter() - t1)}
            return meter.snapshot()

        self.model.train()
        wrapper = self.model if hasattr(self.model, "finish_backward") else None
        n_steps = len(self.train_loader) if self.accum_steps > 1 else 0
        pending = 0                                      # mini-batches accumulated since the last update
        u = 0                                            # optimizer updates so far in this epoch
        module = self.model.module if wrapper is not None else self.model
        for k, batch in enumerate(self.train_loader):
            update = self.accum_steps == 1 or self._updates_after(k, n_steps)
            inputs, targets, mix = self._mixed_to_device(batch)
            outputs = self.model(inputs)
            soft = None if mix is None else T.mixed_targets(targets, outputs.shape[1], mix)
            loss = F.cross_entropy(outputs, targets if soft is None else soft, weight=self.class_weights,
                                   label_smoothing=self.label_smoothing)
            if self.teacher is not None:
                with torch.no_grad():
                    t_out = self.teacher(inputs)
                loss = distill_loss(outputs, t_out, loss, self.distill_alpha, self.distill_temperature)
            if pending == 0:                             # zeroed once per group, before its first backward
                if wrapper is not None:
                    wrapper.zero_grad()
                else:
                    self.optimizer.zero_grad()
            if wrapper is not None:
                wrapper._require_sync = update           # all-reduce each bucket once, on the updating batch
            loss.backward()
            pending += 1
            if wrapper is not None:
                wrapper.finish_backward()
            if update:
                if pending > 1 and not getattr(wrapper, "averages_group", False):      # the group's mean
                    with torch.no_grad():
                        for p in self.model.parameters():
                            if p.grad is not None:
                                p.grad.mul_(1.0 / pending)
                self.optimizer.step()
                if self._ema_after(u):
                    self.model_ema.update_parameters(module)
                u += 1
                pending = 0
            meter.add_reference(outputs.detach(), targets, self.class_weights, soft_target=soft,
                                label_smoothing=self.label_smoothing,
                                loss=loss.detach() if self.teacher is not None else None)
        return meter.snapshot()

    def _reduce_eval(self, meter: DeviceMeter):
        """--shard-eval: every rank saw a disjoint slice of the validation set; sum the counters."""
        import torch.distributed as dist

        if self.shard_eval and dist.is_available() and dist.is_initialized():
            dist.all_reduce(meter.buf)
            if meter.counts is not None:
                dist.all_reduce(meter.counts)
        return meter.snapshot()

    def _evaluate(self, ema: bool = False, model=None):
        """One validation pass over the weights, or with ``ema`` over their moving average, or over ``model`` (a
        distillation teacher: an engine or module of the same kind; its score is counted without --val-metrics)."""
        counted = self.val_metrics and model is None
        meter = DeviceMeter(self.device, len(self.class_names) if counted else None)
        model = self.model if model is None else model
        if _is_native(model):
            model.set_meter(meter)
            if ema:
                model.prepare_ema()             # collective under ZeRO-1: gathers the owned EMA cells
            for batch in self.test_loader:
                if ema:
                    model.eval_step(batch, ema=True)
                else:
                    model.eval_step(batch)
            model.sync()
            return self._reduce_eval(meter)

        net = self.model_ema if ema else model
        net.eval()
        with torch.no_grad():
            for batch in self.test_loader:
                if self.val_tta != "none":
                    meter.add_tta(*self._views_forward(net, batch))
                    continue
                inputs, targets = self._to_device(batch, self.test_loader)
                outputs = net(inputs)
                meter.add_reference(outputs, targets)
        return self._reduce_eval(meter)

    def _views_forward(self, net, batch):
        """([logits of each --val-tta view], targets) of a validation batch on the torch path: a fused batch is
        evaluated at each view, the reference pipeline's [b][V][3][H][W] batch is cut into its views."""
        views = T.tta_views(self.val_tta)
        if isinstance(batch, DEVICE_BATCHES):
            crop = getattr(self.test_loader, "crop", DATA.crop)
            targets = batch.labels.to(self.device)
            return [net(batch.to_float(self.device, out_hw=crop, view=v)[0]) for v in views], targets
        x, targets = batch[0].to(self.device, non_blocking=True), batch[1].to(self.device, non_blocking=True)
        if x.dim() != 5 or x.shape[1] != len(views):
            raise ValueError("the validation batches do not carry the %s views: build the validation DataManager "
                             "with tta=%r" % (self.val_tta, self.val_tta))
        return [net(x[:, i]) for i in range(len(views))], targets
