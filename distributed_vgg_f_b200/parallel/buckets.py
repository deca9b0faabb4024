"""Gradient bucket plan over a flat, ready-ordered arena.

What the reference gets from torch DDP's C++ Reducer (distributedVggf.py:225; SURVEY N3): after
the first iteration, parameters are regrouped in gradient-ready order into buckets capped at
1 MiB (first) / 25 MiB (rest); a tensor larger than the cap sits alone (the 411 MB
``classifier.0.weight`` gradient becomes one message).

We own the plan instead.  Parameters are laid out in ONE flat arena in the order their gradients
become ready (reverse of forward), every tensor aligned to ``align`` elements, and a bucket is
simply a half-open element range ``[start, end)`` of that arena:
  * no copy-in / copy-out: wgrad kernels write straight into the arena, the fused all-reduce
    kernel reads and writes ranges of it;
  * a tensor larger than the cap is *split* across several buckets so the reduction of the first
    chunk overlaps with everything behind it (the reference cannot do that);
  * bucket boundaries are multiples of ``align`` so every rank-slice of a two-shot / NVLS
    reduction is 16-byte aligned for any world size up to 16.
"""
from __future__ import annotations

import dataclasses
from typing import Dict, List, Optional, Sequence, Tuple


@dataclasses.dataclass(frozen=True)
class Bucket:
    index: int
    start: int                 # element offset into the arena
    end: int
    tensors: Tuple[str, ...]   # names of tensors that overlap this range

    @property
    def numel(self) -> int:
        return self.end - self.start


@dataclasses.dataclass
class BucketPlan:
    offsets: Dict[str, int]        # tensor name -> element offset (ready order)
    numels: Dict[str, int]
    order: List[str]               # gradient-ready order
    total: int                     # arena length in elements (aligned)
    buckets: List[Bucket]
    align: int

    def bucket_of(self, name: str) -> List[int]:
        return [b.index for b in self.buckets if name in b.tensors]

    def last_tensor_of_bucket(self, b: Bucket) -> str:
        """The tensor whose gradient completes the bucket (latest in ready order)."""
        return max(b.tensors, key=self.order.index)

    @property
    def grad_total(self) -> int:
        """Length of the arena prefix the buckets cover: the tensors that have gradients.  ``total``
        unless the plan was made for frozen layers (engine_bucket_plan(trainable=))."""
        return self.buckets[-1].end if self.buckets else 0


def _round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


def make_bucket_plan(ready_order: Sequence[Tuple[str, int]], cap_elems: int = 16 * 1024 * 1024,
                     first_cap_elems: int = 0, align: int = 2048, late_cap_elems: int = 0,
                     late_from: str = "", tail_elems: int = 0, exclude: Sequence[str] = ()) -> BucketPlan:
    """``ready_order``: (name, numel) in the order gradients are produced by backward.

    ``late_cap_elems`` / ``late_from``: from tensor ``late_from`` on, buckets are capped at the smaller
    ``late_cap_elems``.  The big early tensors (the FC weights: 88 % of VGG-F, all ready in the first
    tenth of backward) want large messages; the convolution gradients trickle in over the rest of
    backward and the LAST bucket's reduction + optimizer step is the only part of the whole gradient
    exchange that nothing can hide, so the late buckets are one layer each and the final one is
    additionally held to ``tail_elems`` (the first convolutions: a few hundred KB, latency-bound).

    ``exclude``: tensors that keep their offsets but belong to no bucket (exchanged some other way: PowerSGD);
    a bucket never spans one.
    """
    exclude = frozenset(exclude)
    if cap_elems % align:
        cap_elems = _round_up(cap_elems, align)
    if late_cap_elems and late_cap_elems % align:
        late_cap_elems = _round_up(late_cap_elems, align)
    offsets, numels, order, pos = {}, {}, [], 0
    for name, n in ready_order:
        offsets[name], numels[name] = pos, n
        order.append(name)
        pos += _round_up(n, align)
    total = pos

    buckets: List[Bucket] = []
    cur_start, cur_names = 0, []

    def close(end: int) -> None:
        nonlocal cur_start, cur_names
        if end > cur_start:
            buckets.append(Bucket(len(buckets), cur_start, end, tuple(cur_names)))
        cur_start, cur_names = end, []

    # the tail: the longest suffix of the ready order that fits ``tail_elems`` gets its own bucket
    tail_start = total
    if tail_elems:
        for name in reversed(order):
            if total - offsets[name] > tail_elems:
                break
            tail_start = offsets[name]
    late = False
    for name in order:
        t0, t1 = offsets[name], offsets[name] + _round_up(numels[name], align)
        late = late or (bool(late_from) and name == late_from)
        cap = first_cap_elems if (first_cap_elems and not buckets) else cap_elems
        if late and late_cap_elems:
            cap = late_cap_elems
        if name in exclude:
            close(t0)
            cur_start = t1
            continue
        if t0 == tail_start and cur_names:
            close(t0)
        if (t1 - t0) > cap:
            close(t0)                       # flush what we have, then split the big tensor
            p = t0
            while p < t1:
                q = min(p + cap, t1)
                cur_names = [name]
                close(q)
                p = q
            continue
        if cur_names and (t1 - cur_start) > cap:
            close(t0)
        cur_names.append(name)
    close(total)
    return BucketPlan(offsets, numels, order, total, buckets, align)


def engine_bucket_plan(ready_order: Sequence[Tuple[str, int]], bucket_mb: float = 32.0, conv_bucket_mb: float = 9.5,
                       tail_bucket_kb: float = 2400.0, trainable: Optional[int] = None,
                       exclude: Sequence[str] = ()) -> BucketPlan:
    """The plan NativeEngine uses (sizes in MB / KB of fp32 gradient): ``bucket_mb`` messages for the FC weights
    that are ready first, ``conv_bucket_mb`` (one big conv layer) from the first ``features.*`` tensor on, and a
    final bucket of at most ``tail_bucket_kb``.  Also what ``python -m distributed_vgg_f_b200.tools.plan`` prints.

    ``trainable``: only the first ``trainable`` tensors of the ready order have gradients (frozen leading layers
    are a suffix of it).  Every tensor keeps the offset of the full plan; the buckets, and the tail rule, cover
    the trainable prefix ``[0, grad_total)`` alone.  None: every tensor trains.

    ``exclude``: trainable tensors left out of every bucket, offsets unchanged (the PowerSGD-compressed ones)."""
    trainable = len(ready_order) if trainable is None else int(trainable)
    if not 0 < trainable <= len(ready_order):
        raise ValueError("trainable must lie in [1, %d] (got %d)" % (len(ready_order), trainable))
    cap = int(bucket_mb * 1024 * 1024 / 4)
    head = list(ready_order[:trainable])
    first_conv = next((n for n, _ in head if n.startswith("features.")), "")
    plan = make_bucket_plan(head, cap_elems=cap, late_cap_elems=min(cap, int(conv_bucket_mb * 1024 * 1024 / 4)),
                            late_from=first_conv, tail_elems=int(tail_bucket_kb * 1024 / 4), exclude=exclude)
    for name, n in ready_order[trainable:]:          # frozen: offsets and sizes only, in no bucket
        plan.offsets[name], plan.numels[name] = plan.total, n
        plan.order.append(name)
        plan.total += _round_up(n, plan.align)
    return plan
