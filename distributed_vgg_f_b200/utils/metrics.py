"""Running metrics.

``Average`` / ``Accuracy2`` keep the reference's public surface and string formats
(distributedUtil.py:31-99: ``'{:.6f}'`` for the loss mean, ``'{:.2f}%'`` for accuracy) so that the
per-epoch report line is byte-compatible.  The reference feeds them with two ``.item()`` host
syncs per step (distributedVggf.py:174-175); ``DeviceMeter`` is the H100-native replacement: the
fused cross-entropy kernel adds (loss_sum, correct, count) into a 3-float device buffer and the
host reads it once per epoch.

``DeviceMeter(device, num_classes)`` also counts a confusion matrix and the top-5 hits of an evaluation pass
(--val-metrics) in int64; ``class_metrics`` derives per-class recall, precision, support, balanced accuracy and
acc@5 from them.
"""
from __future__ import annotations

from typing import Optional

import numpy as np
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
        self.classes: Optional[dict] = None     # class_metrics of an evaluation pass counted with a class count

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


def _ratio(num: int, den: int):
    return num / den if den else None


def class_metrics(confusion, top5: Optional[int] = None) -> dict:
    """Everything --val-metrics reports, from the counts of a pass: ``confusion`` [C][C] (rows labels, columns
    predictions) and the top-5 hits.  Returns a dict of JSON-ready values: confusion (list of rows), support (row
    sums), recall (diagonal / row sum), precision (diagonal / column sum), balanced_acc (the mean recall over classes
    with support, scikit-learn's balanced_accuracy_score) and, when C > 5, acc5 (top-5 hits / samples).  A ratio
    with a zero denominator is None."""
    m = np.asarray(confusion, dtype=np.int64)
    C = m.shape[0]
    diag, rows, cols = np.diag(m), m.sum(1), m.sum(0)
    recall = [_ratio(int(diag[c]), int(rows[c])) for c in range(C)]
    defined = [r for r in recall if r is not None]
    out = dict(confusion=m.tolist(), support=[int(n) for n in rows], recall=recall,
               precision=[_ratio(int(diag[c]), int(cols[c])) for c in range(C)],
               balanced_acc=sum(defined) / len(defined) if defined else None)
    if C > 5:
        out["acc5"] = _ratio(int(top5), int(rows.sum()))
    return out


def _pct(r) -> str:
    return "-" if r is None else "{:.2f}%".format(r * 100)


def class_report(head: str, what: str, m: dict, class_names=None) -> list:
    """The report lines of ``class_metrics`` ``m``: ``[Info] <head><what> balanced acc: ..%`` (and ``<what> acc@5``
    when C > 5), then for C <= 32 one line per class with its support, recall, precision and confusion row.  An
    undefined ratio prints ``-``."""
    C = len(m["support"])
    names = list(class_names) if class_names is not None else []
    names += [str(c) for c in range(len(names), C)]
    first = "[Info] {}{} balanced acc: {}".format(head, what, _pct(m["balanced_acc"]))
    if "acc5" in m:
        first += ", {} acc@5: {}".format(what, _pct(m["acc5"]))
    lines = [first + "."]
    if C <= 32:
        for c in range(C):
            lines.append("[Info] {}{} class {}: support {}, recall {}, precision {}, confusion row {}.".format(
                head, what, names[c], m["support"][c], _pct(m["recall"][c]), _pct(m["precision"][c]),
                m["confusion"][c]))
    return lines


class DeviceMeter:
    """Three fp32 device accumulators: [sum of per-sample loss, #correct, #samples].

    The native engine's cross-entropy kernel atomically adds into ``buf``; nothing touches the
    host until ``snapshot`` is called (once per epoch).

    With ``num_classes`` C the meter also holds int64 ``counts`` [C * C + 1]: ``confusion`` (a [C][C] view, rows
    labels, columns first-maximum predictions) and ``top5`` (the last element: labels ranked among the first five).
    The native engine launches ``ops.class_metrics`` into them when they exist, and the evaluation reductions
    (``add_reference`` with integer targets, ``add_tta``) count with torch ops; ``snapshot`` then attaches
    ``class_metrics`` to the accuracy it returns.
    """

    def __init__(self, device, num_classes: Optional[int] = None) -> None:
        self.buf = torch.zeros(4, dtype=torch.float32, device=device)
        self.counts = self.confusion = self.top5 = None
        if num_classes is not None:
            C = int(num_classes)
            if C < 1:
                raise ValueError("num_classes must be >= 1 (got %d)" % C)
            self.counts = torch.zeros(C * C + 1, dtype=torch.int64, device=device)
            self.confusion = self.counts[:C * C].view(C, C)
            self.top5 = self.counts[C * C:]

    def reset(self) -> None:
        self.buf.zero_()
        if self.counts is not None:
            self.counts.zero_()

    def _count_classes(self, scores: torch.Tensor, target: torch.Tensor, pred: torch.Tensor) -> None:
        """Add a batch to ``confusion`` and ``top5`` (torch ops): ``pred`` is the prediction the correct-count used;
        the label y ranks #{c : s_c > s_y} + #{c < y : s_c == s_y}."""
        if self.counts is None:
            return
        C = self.confusion.shape[0]
        t = target.view(-1).to(self.counts.device, torch.int64)
        s = scores.float().to(self.counts.device)
        self.confusion.view(-1).add_(torch.bincount(t * C + pred.to(t.device), minlength=C * C))
        sy = s.gather(1, t.view(-1, 1))
        ahead = (s > sy) | ((s == sy) & (torch.arange(C, device=s.device) < t.view(-1, 1)))
        self.top5.add_((ahead.sum(1) < 5).sum())

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
            pred = logits.argmax(dim=1)
            self.buf[1] += pred.eq(target).sum()
            self.buf[2] += logits.shape[0]
            self._count_classes(logits, target, pred)

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
            pred = mean.argmax(dim=1)
            self.buf[1] += pred.eq(target).sum()
            self.buf[2] += mean.shape[0]
            self._count_classes(mean, target, pred)

    def snapshot(self):
        loss_sum, correct, count, _ = self.buf.tolist()
        avg, acc = Average(), Accuracy2()
        avg.sum, avg.count = loss_sum, int(count)
        acc.correct, acc.count = int(correct), int(count)
        if self.counts is not None:
            counts = self.counts.tolist()
            C = self.confusion.shape[0]
            acc.classes = class_metrics(np.array(counts[:C * C], dtype=np.int64).reshape(C, C), counts[-1])
        return avg, acc
