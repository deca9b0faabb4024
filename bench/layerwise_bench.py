"""What LAMB and LARS cost on the native engine, one GPU.

Prints one JSON line per measurement, each with the card's name and power limit read in the same run:
  * "step": VGG-F training step time at batch 64 and 224^2 with Adam (the default), SGD, LAMB and LARS (the last two
    at --weight-decay 0.05, biases 0), in alternating blocks of --steps steps, median over --runs blocks;
  * "phase": device time of LAMB's and LARS's phase-1 launches over FC-1 (its 13 bucket pieces, summed) and of its
    phase-2 launch (median of --reps each), against the HBM bound of the bytes each moves at the H100 SXM data
    sheet's 3.35 TB/s.
Usage: ``python bench/layerwise_bench.py [--steps 10] [--runs 5] [--reps 20]``.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from distributed_vgg_f_b200 import ops  # noqa: E402
from distributed_vgg_f_b200.config import TRAIN  # noqa: E402
from ema_bench import _batch, _card, _time  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
RECIPE = dict(weight_decay=0.05, bias_weight_decay=0.0)
# bytes per element: LAMB phase 1 reads p, g, m, v, writes m, v and clears g; phase 2 reads p, m, v and writes p and
# the bf16 shadow.  LARS phase 1 reads p and g; phase 2 reads p, m, g, writes p, m, the shadow and clears g.
BYTES = {("lamb", 1): 28, ("lamb", 2): 18, ("lars", 1): 8, ("lars", 2): 26}


def _engine(b: int, **kw):
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine
    from distributed_vgg_f_b200.models.vggf import vggf_spec

    return NativeEngine(vggf_spec(3), device=torch.device("cuda"), batch=b, distributed=False, **kw)


def phase_times(eng, reps: int, card: dict) -> None:
    """Phase 1 over FC-1's pieces (fp32 gradient, cleared by LAMB) and its phase 2, as the engine launches them."""
    kind, lamb = eng.opt_name, eng.opt_name == "lamb"
    plan = eng.layerwise_plans()[False]
    t = plan.tensors.index("classifier.0.weight")
    lo, hi = plan.ranges["classifier.0.weight"]
    hyper = dict(beta1=TRAIN.lamb_beta1, beta2=TRAIN.lamb_beta2, eps=TRAIN.lamb_eps, step=10) if lamb else \
        dict(momentum=eng.momentum, trust_coeff=TRAIN.lars_trust_coeff, trust_eps=TRAIN.lars_eps)
    p1 = [L for s in plan.phase1 for L in plan.phase1[s] if any(g.tensor == t for g in L.segments)]
    p2 = [L for s in plan.phase2 for L in plan.phase2[s] if any(g.tensor == t for g in L.segments)]
    eng.g32.normal_().mul_(1e-3)

    def launch(phase, L):
        a, b = L.start, L.end
        kw = dict(g32=eng.g32[a:b]) if (phase == 1 or not lamb) else {}
        if (phase == 1) == lamb:
            kw["zero"] = eng.g32[a:b]
        extra = dict(shadow=eng.w16[a:b], ratio=eng.trust_ratio) if phase == 2 else {}
        ops.layerwise_step(phase, kind, eng.p32[a:b], eng.m32[a:b], eng.v32[a:b] if lamb else None, ws=eng._lw_ws,
                           lr=1e-9, segments=L.segments, **kw, **extra, **hyper)

    for phase, launches in ((1, p1), (2, p2)):
        ms = sum(_time(lambda L=L: launch(phase, L), reps) for L in launches)
        n = sum(L.end - L.start for L in launches)
        bound_ms = n * BYTES[(kind, phase)] / HBM_BYTES_PER_S * 1e3
        print(json.dumps(dict(card, what="phase", optimizer=kind, phase=phase, tensor="classifier.0.weight",
                              launches=len(launches), elements=n, bytes_per_element=BYTES[(kind, phase)],
                              ms=round(ms, 4), hbm_bound_ms=round(bound_ms, 4),
                              frac_of_hbm_bound=round(bound_ms / ms, 3))), flush=True)
    assert hi - lo >= sum(L.end - L.start for L in p2) > 0


def step_times(engines: dict, batch, steps: int, runs: int, card: dict) -> None:
    res = {k: [] for k in engines}
    for eng in engines.values():
        for _ in range(3):
            eng.train_step(batch)
        eng.sync()
    for _ in range(runs):
        for name, eng in engines.items():
            a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(steps):
                eng.train_step(batch)
            e.record()
            e.synchronize()
            res[name].append(a.elapsed_time(e) / steps)
    base = statistics.median(res["adam"])
    for name, ts in res.items():
        ms = statistics.median(ts)
        print(json.dumps(dict(card, what="step", case=name, batch=batch.labels.shape[0], steps_per_block=steps,
                              blocks=runs, ms_per_step=round(ms, 3), img_s=round(batch.labels.shape[0] / (ms * 1e-3), 1),
                              vs_adam=round(ms / base, 4), all_blocks_ms=[round(t, 3) for t in ts])), flush=True)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    ops.require()
    card = _card()
    batch = _batch(args.batch)
    engines = {"adam": _engine(args.batch), "sgd": _engine(args.batch, optimizer="sgd"),
               "lamb": _engine(args.batch, optimizer="lamb", **RECIPE),
               "lars": _engine(args.batch, optimizer="lars", **RECIPE)}
    step_times(engines, batch, args.steps, args.runs, card)
    for name in ("lamb", "lars"):
        phase_times(engines[name], args.reps, card)


if __name__ == "__main__":
    main()
