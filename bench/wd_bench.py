"""What weight decay, AdamW and per-tensor decay cost on the native engine, one GPU.

Prints one JSON line per measurement, each with the card's name and power limit read in the same run:
  * "optimizer": summed device time of one optimizer launch per bucket of the VGG-F plan (fp32-gradient
    entry, median of --reps launches each) for Adam at decay 0 (the default), Adam with each bucket's
    segment table (decay 0.05, biases 0), and AdamW with the same tables;
  * "step": VGG-F training step time at batch 64 and 224^2 with the default flags and with
    ``--optimizer adamw --weight-decay 0.05 --bias-weight-decay 0`` (cases alternated, median over --runs
    runs of --steps steps each).  Three more cases separate the code from the numbers it trains on: Adam
    with a uniform L2 decay of 0.05 (the scalar launches of before, different weights), AdamW at decay 0
    (the default's weights bit for bit, through the decoupled kernels), and a second default engine,
    built last, for the spread between two engines of one configuration.
Usage: ``python bench/wd_bench.py [--steps 32] [--runs 5] [--reps 20]``.
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
from ema_bench import _batch, _card, _time  # noqa: E402

RECIPE = dict(optimizer="adamw", weight_decay=0.05, bias_weight_decay=0.0)


def _engine(b: int, **kw):
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine
    from distributed_vgg_f_b200.models.vggf import vggf_spec

    return NativeEngine(vggf_spec(3), device=torch.device("cuda"), batch=b, distributed=False, **kw)


def optimizer_launches(eng, reps: int, card: dict) -> None:
    """``eng`` was built with RECIPE: its buckets carry the segment tables."""
    eng.g32.normal_().mul_(1e-3)
    cases = {"adam_wd0": lambda s, segs: dict(weight_decay=0.0),
             "adam_segments": lambda s, segs: dict(weight_decay=segs[0][1], wd_segments=segs),
             "adamw_segments": lambda s, segs: dict(weight_decay=segs[0][1], wd_segments=segs, decoupled=True)}
    for name, kw_of in cases.items():
        ms = 0.0
        for bk in eng.plan.buckets:
            s, e = bk.start, bk.end
            kw = kw_of(s, eng._wd_segments[s])

            def run():
                ops.adam_step(eng.p32[s:e], eng.m32[s:e], eng.v32[s:e], g32=eng.g32[s:e], zero=eng.g32[s:e],
                              shadow=eng.w16[s:e], lr=1e-9, step=10, **kw)
            ms += _time(run, reps)
        print(json.dumps(dict(card, what="optimizer", case=name, launches=len(eng.plan.buckets),
                              max_segments=max(len(v) for v in eng._wd_segments.values()), params=eng.plan.total,
                              ms=round(ms, 4))), flush=True)


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
    for name, ts in res.items():
        ms = statistics.median(ts)
        print(json.dumps(dict(card, what="step", case=name, batch=batch.labels.shape[0], steps_per_run=steps, runs=runs,
                              ms_per_step=round(ms, 3), img_s=round(batch.labels.shape[0] / (ms * 1e-3), 1),
                              all_runs_ms=[round(t, 3) for t in ts])), flush=True)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=32)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    ops.require()
    card = _card()
    batch = _batch(args.batch)
    engines = {"default": _engine(args.batch), "adamw_wd0.05_bias0": _engine(args.batch, **RECIPE),
               "adam_wd0.05": _engine(args.batch, weight_decay=0.05), "adamw_wd0": _engine(args.batch, optimizer="adamw"),
               "default_again": _engine(args.batch)}
    optimizer_launches(engines["adamw_wd0.05_bias0"], args.reps, card)
    step_times(engines, batch, args.steps, args.runs, card)


if __name__ == "__main__":
    main()
