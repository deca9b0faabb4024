"""Launch plan of the layer-wise adaptive optimizers (LAMB, LARS) over the engine's gradient buckets.

A trust ratio needs the norms of a whole tensor, and the buckets cut tensors apart (VGG-F's ``classifier.0.weight``
spans 13 buckets; a conv bucket may end with the bias of the layer after it).  So each update takes two kinds of
launch (DESIGN 3.2):

* phase 1, once per update unit (a bucket, or a PowerSGD-compressed tensor) right where the Adam launch of that unit
  goes: one segment per tensor piece, each CTA inside one segment, each CTA's partial sums stored at a slot of its
  own.  A tensor's slots are numbered by a running CTA index over its phase-1 pieces, in issue order;
* phase 2, right after the phase 1 of the unit that holds a tensor's last piece: one segment per tensor completed
  there, every CTA of a segment adding that tensor's slots in the same order before it updates its slice.

Everything here is pure host arithmetic on the bucket plan, so ``tools.plan --optimizer lamb`` prints it without a
GPU and the tests check it on the CPU.
"""
from __future__ import annotations

import dataclasses
from typing import Callable, Dict, List, Sequence, Tuple

from .buckets import BucketPlan

THREADS = 256            # threads per CTA of the layer-wise kernels
CTAS_PER_SM = 4          # the optimizer launches' grid cap (csrc: layerwise_max_grid)
MAX_SEGMENTS = 16        # segments per launch (csrc: LW_MAX_SEGMENTS)


def _round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


@dataclasses.dataclass(frozen=True)
class Segment:
    start: int           # element offset within the launch's range
    tensor: int          # index into LayerwisePlan.tensors (and the engine's ratio array)
    ctas: int
    slot: int            # phase 1: slot of the segment's first CTA; phase 2: the tensor's first slot
    nslots: int          # phase 2: the tensor's slot count (phase 1: 0)
    wd: float


@dataclasses.dataclass(frozen=True)
class Launch:
    start: int           # arena range [start, end)
    end: int
    segments: Tuple[Segment, ...]

    @property
    def grid(self) -> int:
        return sum(s.ctas for s in self.segments)


@dataclasses.dataclass
class LayerwisePlan:
    tensors: List[str]                       # trainable tensors in arena order
    ranges: Dict[str, Tuple[int, int]]       # tensor -> arena range, padding included
    units: List[Tuple[int, int]]             # update units in issue order
    phase1: Dict[int, List[Launch]]          # unit start -> its phase-1 launches
    phase2: Dict[int, List[Launch]]          # unit start -> the phase-2 launches issued after them
    slots: Dict[str, Tuple[int, int]]        # tensor -> (first slot, slot count)
    total_slots: int

    def phase2_count(self) -> int:
        return sum(len(v) for v in self.phase2.values())

    def workspace_elems(self) -> int:
        """fp32 elements of the partial-sum workspace: a pair per slot."""
        return 2 * self.total_slots


def _ctas(elems: int, per_segment_cap: int) -> int:
    return max(1, min(-(-(elems // 4) // THREADS), per_segment_cap))


def _chunks(items: Sequence, n: int) -> List[Sequence]:
    return [items[k:k + n] for k in range(0, len(items), n)]


def update_units(plan: BucketPlan, compressed: Sequence[str] = ()) -> List[Tuple[int, int]]:
    """The arena ranges the engine updates one launch group at a time: the buckets, and each PowerSGD-compressed
    tensor's aligned range (in no bucket)."""
    units = [(b.start, b.end) for b in plan.buckets]
    return units + [(plan.offsets[n], plan.offsets[n] + _round_up(plan.numels[n], plan.align)) for n in compressed]


def layerwise_plan(plan: BucketPlan, decay_of: Callable[[str], float], sms: int,
                   units: Sequence[Tuple[int, int]] = None, max_segments: int = MAX_SEGMENTS) -> LayerwisePlan:
    """The phase-1 and phase-2 launches of every update unit.  ``units``: the arena ranges updated one launch group
    at a time (default: the buckets); under PowerSGD also each compressed tensor's range.  ``decay_of``: a tensor's
    weight decay.  ``sms``: SMs of the GPU planned for; a launch uses at most ``CTAS_PER_SM * sms`` CTAs."""
    units = sorted((int(s), int(e)) for s, e in (update_units(plan) if units is None else units))
    cap = CTAS_PER_SM * int(sms)
    ranges = {n: (plan.offsets[n], plan.offsets[n] + _round_up(plan.numels[n], plan.align)) for n in plan.order}
    # the trainable tensors: those the units cover (frozen ones lie behind every bucket and unit)
    tensors = [n for n in plan.order if any(ranges[n][0] < e and ranges[n][1] > s for s, e in units)]
    ranges = {n: ranges[n] for n in tensors}
    tid = {n: i for i, n in enumerate(tensors)}
    used: Dict[str, int] = {n: 0 for n in tensors}
    phase1: Dict[int, List[Launch]] = {}
    last_unit: Dict[str, int] = {}
    for s, e in units:
        pieces = []                        # (start, end, tensor) within [s, e), arena order
        for n in tensors:
            a, b = ranges[n]
            if a < e and b > s:
                pieces.append((max(a, s), min(b, e), n))
                last_unit[n] = s
        launches = []
        for part in _chunks(pieces, max_segments):
            lo, per = part[0][0], max(1, cap // len(part))
            segs = []
            for a, b, n in part:
                c = _ctas(b - a, per)
                segs.append(Segment(a - lo, tid[n], c, used[n], 0, float(decay_of(n))))
                used[n] += c
            launches.append(Launch(lo, part[-1][1], tuple(segs)))
        phase1[s] = launches
    base, slots = 0, {}
    for n in tensors:                      # dense: tensor after tensor, each its pieces' CTAs in issue order
        slots[n] = (base, used[n])
        base += used[n]
    phase1 = {s: [Launch(L.start, L.end, tuple(dataclasses.replace(g, slot=g.slot + slots[tensors[g.tensor]][0])
                                                for g in L.segments)) for L in ls] for s, ls in phase1.items()}
    phase2: Dict[int, List[Launch]] = {}
    for s, _ in units:
        done = [n for n in tensors if last_unit.get(n) == s]
        launches = []
        for part in _chunks(done, max_segments):
            lo, per = ranges[part[0]][0], max(1, cap // len(part))
            segs = tuple(Segment(ranges[n][0] - lo, tid[n], _ctas(ranges[n][1] - ranges[n][0], per), slots[n][0],
                                 slots[n][1], float(decay_of(n))) for n in part)
            launches.append(Launch(lo, ranges[part[-1]][1], segs))
        phase2[s] = launches
    return LayerwisePlan(tensors, ranges, list(units), phase1, phase2, slots, base)


def describe(lw: LayerwisePlan, kind: str) -> List[str]:
    """Text of ``tools.plan --optimizer lamb|lars``: per unit, the phase-1 pieces and the tensors it completes."""
    out = ["%s: %d phase-1 launches, %d phase-2 launches, %d partial-sum slots (%.1f KB of workspace)"
           % (kind, sum(len(v) for v in lw.phase1.values()), lw.phase2_count(), lw.total_slots,
              lw.workspace_elems() * 4 / 1e3)]
    out.append("%3s %11s %-40s %s" % ("#", "start", "phase 1 (tensor: CTAs = slots)", "phase 2 after it"))
    for u, (s, _) in enumerate(lw.units):
        p1 = "; ".join("%s: %d" % (lw.tensors[g.tensor], g.ctas) for L in lw.phase1[s] for g in L.segments)
        p2 = ", ".join(lw.tensors[g.tensor] for L in lw.phase2[s] for g in L.segments)
        n2 = len(lw.phase2[s])
        out.append("%3d %11d %-40s %s" % (u, s, p1, ("%d launch%s: %s" % (n2, "" if n2 == 1 else "es", p2)) if n2 else "-"))
    return out


def engine_layerwise_plans(spec, sms: int, decay_of: Callable[[str], float] = lambda name: 0.0,
                           freeze_layers: int = 0, powersgd_rank: int = 0, bucket_mb: float = 32.0,
                           conv_bucket_mb: float = 9.5, tail_bucket_kb: float = 2400.0) -> Dict[bool, LayerwisePlan]:
    """The plans NativeEngine makes for a model (``NativeEngine.layerwise_plans``) from the spec alone: key False
    for uncompressed updates, True (with ``powersgd_rank``) for the updates PowerSGD compresses."""
    from ..models import layout as L
    from . import powersgd
    from .buckets import engine_bucket_plan

    ready = L.ready_order(spec)
    trainable = len(ready) - len(spec.frozen_param_names(freeze_layers))
    plan = engine_bucket_plan(ready, bucket_mb, conv_bucket_mb, tail_bucket_kb, trainable=trainable)
    plans = {False: layerwise_plan(plan, decay_of, sms)}
    if powersgd_rank:
        comp = [t.name for t in powersgd.plan(spec, powersgd_rank, freeze_layers) if t.compressed]
        plan2 = engine_bucket_plan(ready, bucket_mb, conv_bucket_mb, tail_bucket_kb, trainable=trainable, exclude=comp)
        plans[True] = layerwise_plan(plan2, decay_of, sms, update_units(plan2, comp))
    return plans
