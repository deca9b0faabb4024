"""What the moving average of the weights (--model-ema) costs on the native engine, one GPU.

Prints one JSON line per measurement, each with the card's name and power limit read in the same run:
  * "optimizer": device time of every Adam launch of the VGG-F bucket plan, with and without the EMA, on
    the fp32-gradient entry (g32) and on the bf16-wire entry (g16); bytes are counted from the streams
    each launch moves (g32: p, m, v read + written, g32 read, shadow written, gradient re-zeroed = 34 B
    per parameter; g16: 28 B; the EMA adds 8 B) and divided by the time, against 3.35 TB/s;
  * "step": VGG-F training step time at batch 64 and 224^2 with the EMA off, at --model-ema-steps 32 and
    at 1 (cases alternated, median over --runs runs of --steps steps each);
  * "eval": one EMA evaluation's preparation (cast ema32 -> ema16; no ZeRO-1 on one GPU) and its
    validation pass, next to the pass over the raw weights.
Usage: ``python bench/ema_bench.py [--steps 32] [--runs 5] [--reps 20] [--eval-batches 20]``.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from distributed_vgg_f_b200 import ops  # noqa: E402
from distributed_vgg_f_b200.data import transforms as T  # noqa: E402
from distributed_vgg_f_b200.data.loader import FusedBatch  # noqa: E402

HBM_GBS = 3350.0
DECAY = 0.999


def _card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    name, _, power = q.stdout.strip().partition(",")
    return {"gpu": name.strip() or torch.cuda.get_device_name(), "power_limit": power.strip()}


def _batch(b: int) -> FusedBatch:
    g = torch.Generator().manual_seed(0)
    src = torch.randint(0, 256, (b, 128, 128, 3), dtype=torch.uint8, generator=g)
    return FusedBatch(src.pin_memory(), T.sample_train_params(b, 128, 128, g).pin_memory(),
                      torch.randint(0, 3, (b,), generator=g).pin_memory(), T.resized_dims(True, 128, 128), None)


def _engine(b: int, ema_decay):
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine
    from distributed_vgg_f_b200.models.vggf import vggf_spec

    return NativeEngine(vggf_spec(3), device=torch.device("cuda"), batch=b, distributed=False, ema_decay=ema_decay)


def _time(run, reps: int) -> float:
    """Median device time (ms) of ``run`` over ``reps`` launches, after warm-up."""
    for _ in range(3):
        run()
    times = []
    for _ in range(reps):
        a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        run()
        e.record()
        e.synchronize()
        times.append(a.elapsed_time(e))
    return statistics.median(times)


def optimizer_launches(eng, reps: int, card: dict) -> None:
    g16 = torch.randn(eng.plan.total, device="cuda").mul_(1e-3).to(torch.bfloat16)
    eng.g32.normal_().mul_(1e-3)
    for entry, base in (("g32", 34), ("g16", 28)):
        for ema in (False, True):
            ms = 0.0
            for bk in eng.plan.buckets:
                s, e = bk.start, bk.end
                kw = dict(ema=eng.ema32[s:e], ema_decay=DECAY) if ema else {}
                grads = dict(g32=eng.g32[s:e], zero=eng.g32[s:e]) if entry == "g32" else dict(g16=g16[s:e])

                def run():
                    ops.adam_step(eng.p32[s:e], eng.m32[s:e], eng.v32[s:e], shadow=eng.w16[s:e], lr=1e-9,
                                  step=10, **grads, **kw)
                ms += _time(run, reps)
            nbytes = eng.plan.total * (base + (8 if ema else 0))
            gbs = nbytes / (ms * 1e-3) / 1e9
            print(json.dumps(dict(card, what="optimizer", entry=entry, ema=ema, launches=len(eng.plan.buckets),
                                  params=eng.plan.total, bytes_per_param_counted=base + (8 if ema else 0),
                                  ms=round(ms, 4), GBs=round(gbs, 1), frac_of_3350=round(gbs / HBM_GBS, 3))),
                  flush=True)


def step_times(engines: dict, batch, steps: int, runs: int, card: dict) -> None:
    res = {k: [] for k in engines}
    for eng, _ in engines.values():
        for _ in range(3):
            eng.train_step(batch)
        eng.sync()
    for _ in range(runs):
        for name, (eng, every) in engines.items():
            a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for u in range(steps):
                if every and u % every == 0:
                    eng.train_step(batch, ema=True)
                else:
                    eng.train_step(batch)
            e.record()
            e.synchronize()
            res[name].append(a.elapsed_time(e) / steps)
    for name, ts in res.items():
        ms = statistics.median(ts)
        print(json.dumps(dict(card, what="step", case=name, batch=batch.labels.shape[0], steps_per_run=steps, runs=runs,
                              ms_per_step=round(ms, 3), img_s=round(batch.labels.shape[0] / (ms * 1e-3), 1),
                              all_runs_ms=[round(t, 3) for t in ts])), flush=True)


def evaluation(eng, batch, n_batches: int, reps: int, card: dict) -> None:
    from distributed_vgg_f_b200.utils.metrics import DeviceMeter

    eng.train_step(batch, ema=True)
    prep = _time(eng.prepare_ema, reps)
    eng.set_meter(DeviceMeter("cuda"))

    def val(ema):
        for _ in range(n_batches):
            eng.eval_step(batch, ema=True) if ema else eng.eval_step(batch)
    raw_ms, ema_ms = _time(lambda: val(False), max(reps // 4, 3)), _time(lambda: val(True), max(reps // 4, 3))
    print(json.dumps(dict(card, what="eval", batches=n_batches, batch=batch.labels.shape[0],
                          prepare_ema_ms=round(prep, 3), val_raw_ms=round(raw_ms, 3), val_ema_ms=round(ema_ms, 3))),
          flush=True)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=32)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--eval-batches", type=int, default=20)
    args = ap.parse_args()
    ops.require()
    card = _card()
    batch = _batch(args.batch)
    engines = {"off": (_engine(args.batch, None), 0), "steps32": (_engine(args.batch, DECAY), 32),
               "steps1": (_engine(args.batch, DECAY), 1)}
    optimizer_launches(engines["steps1"][0], args.reps, card)
    step_times(engines, batch, args.steps, args.runs, card)
    evaluation(engines["steps1"][0], batch, args.eval_batches, args.reps, card)


if __name__ == "__main__":
    main()
