"""Running metrics.

``Average`` / ``Accuracy2`` keep the reference's public surface and string formats
(distributedUtil.py:31-99: ``'{:.6f}'`` for the loss mean, ``'{:.2f}%'`` for accuracy) so that the
per-epoch report line is byte-compatible.  The reference feeds them with two ``.item()`` host
syncs per step (distributedVggf.py:174-175); ``DeviceMeter`` is the H100-native replacement: the
fused cross-entropy kernel adds (loss_sum, correct, count) into a 3-float device buffer and the
host reads it once per epoch.
"""
from __future__ import annotations

import torch


class Average:
    """Sample-weighted running mean (reference: distributedUtil.py:31-58)."""

    def __init__(self) -> None:
        self.sum = 0.0
        self.count = 0

    def __str__(self) -> str:
        return "{:.6f}".format(self.average)

    @property
    def average(self) -> float:
        return self.sum / self.count if self.count else float("nan")

    def update(self, value, number) -> None:
        self.sum += float(value) * number
        self.count += number


class Accuracy2:
    """Running top-1 accuracy (reference: distributedUtil.py:61-99)."""

    def __init__(self) -> None:
        self.correct = 0
        self.count = 0

    def __str__(self) -> str:
        return "{:.2f}%".format(self.accuracy * 100)

    @property
    def accuracy(self) -> float:
        return self.correct / self.count if self.count else float("nan")

    def update(self, output: torch.Tensor, target: torch.Tensor) -> None:
        with torch.no_grad():
            self.correct += int(output.argmax(dim=1).eq(target).sum().item())
        self.count += output.size(0)

    def update_counts(self, correct: int, number: int) -> None:
        self.correct += int(correct)
        self.count += int(number)


class DeviceMeter:
    """Three fp32 device accumulators: [sum of per-sample loss, #correct, #samples].

    The native engine's cross-entropy kernel atomically adds into ``buf``; nothing touches the
    host until ``snapshot`` is called (once per epoch).
    """

    def __init__(self, device) -> None:
        self.buf = torch.zeros(4, dtype=torch.float32, device=device)

    def reset(self) -> None:
        self.buf.zero_()

    def add_reference(self, logits: torch.Tensor, target: torch.Tensor, weight=None,
                      soft_target: torch.Tensor = None, label_smoothing: float = 0.0, loss=None) -> None:
        """Torch-op fallback used by the oracle path (same arithmetic as the kernel): accumulates
        ``loss * batch`` exactly like ``Average.update(loss.item(), batch)`` in the reference's loop,
        where ``loss`` is the (optionally class-weighted) mean torch reports.

        ``soft_target`` (probability targets [B][C], MixUp / CutMix) and ``label_smoothing``: the loss is
        F.cross_entropy's with them, and a sample is correct when argmax(logits) == argmax(soft_target)
        (torchvision's classification reference, ``utils.accuracy`` on 2-D targets).

        ``loss`` (a scalar, e.g. the distillation objective): accumulated instead of the cross-entropy; the
        accuracy is counted as without it."""
        if loss is not None:
            with torch.no_grad():
                cls = soft_target.argmax(dim=1) if soft_target is not None else target
                self.buf[0] += loss.float() * logits.shape[0]
                self.buf[1] += logits.argmax(dim=1).eq(cls).sum()
                self.buf[2] += logits.shape[0]
            return
        if soft_target is not None or label_smoothing:
            with torch.no_grad():
                tgt = soft_target if soft_target is not None else target
                loss = torch.nn.functional.cross_entropy(logits.float(), tgt, weight=weight,
                                                         label_smoothing=label_smoothing)
                self.buf[0] += loss * logits.shape[0]
                cls = soft_target.argmax(dim=1) if soft_target is not None else target
                self.buf[1] += logits.argmax(dim=1).eq(cls).sum()
                self.buf[2] += logits.shape[0]
            return
        with torch.no_grad():
            logp = torch.log_softmax(logits.float(), dim=1)
            nll = -logp.gather(1, target.view(-1, 1)).view(-1)
            if weight is None:
                self.buf[0] += nll.sum()
            else:
                w = weight.to(nll.device, nll.dtype)[target]
                self.buf[0] += (w * nll).sum() / w.sum() * logits.shape[0]
            self.buf[1] += logits.argmax(dim=1).eq(target).sum()
            self.buf[2] += logits.shape[0]

    def add_tta(self, view_logits, target: torch.Tensor) -> None:
        """Torch-op form of the --val-tta reduction (the native engine's tta_accumulate): logits of each view of the
        batch ([b][C] each, in view order) -> the mean of their fp32 softmaxes, added in view order; a sample's loss
        is -log of its label's mean probability, and it is correct when the first maximum of the mean is its label."""
        with torch.no_grad():
            acc = None
            for z in view_logits:
                p = torch.softmax(z.float(), dim=1)
                acc = p if acc is None else acc + p
            mean = acc / len(view_logits)
            self.buf[0] += -torch.log(mean.gather(1, target.view(-1, 1))).sum()
            self.buf[1] += mean.argmax(dim=1).eq(target).sum()
            self.buf[2] += mean.shape[0]

    def snapshot(self):
        loss_sum, correct, count, _ = self.buf.tolist()
        avg, acc = Average(), Accuracy2()
        avg.sum, avg.count = loss_sum, int(count)
        acc.correct, acc.count = int(correct), int(count)
        return avg, acc
