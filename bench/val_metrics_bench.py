"""What the per-class evaluation counts (--val-metrics) cost on the native engine, one GPU: an evaluation batch of 64 at
224^2, for VGG-F (C = 3, fused head) and VGG-16 (C = 1000, GEMM + cross-entropy head).

Prints one JSON line per (model, flag), with the card's name and power limit read in the same run: milliseconds per
evaluation batch with a plain meter (off) and with a confusion meter (on, one more launch per batch).  The two run in
alternating blocks of --steps batches; each figure is the median over --runs blocks.  Then one line per C with the
time of class_metrics_kernel alone on [64][C] logits (CUDA events around --kernel-iters back-to-back launches).  The
input is a validation FusedBatch of 256 x 256 images (Resize 256, crop 224).  With --out the lines are also written
to that file.
Usage: ``python bench/val_metrics_bench.py [--steps 10] [--runs 5] [--out bench/results/val_metrics_bench_h100.jsonl]``.
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
from distributed_vgg_f_b200.data import transforms as T  # noqa: E402
from distributed_vgg_f_b200.data.loader import FusedBatch  # noqa: E402
from distributed_vgg_f_b200.utils.metrics import DeviceMeter  # noqa: E402
from ema_bench import _card  # noqa: E402

MODELS = (("vggf", 3), ("vgg16", 1000))


def _val_batch(b: int, C: int) -> FusedBatch:
    g = torch.Generator().manual_seed(0)
    src = torch.randint(0, 256, (b, 256, 256, 3), dtype=torch.uint8, generator=g)
    return FusedBatch(src.pin_memory(), T.val_params(b, 256, 256).pin_memory(),
                      torch.randint(0, C, (b,), generator=g).pin_memory(), T.resized_dims(False, 256, 256), None)


def _block_ms(eng, batch, steps: int) -> float:
    a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        eng.eval_step(batch)
    e.record()
    e.synchronize()
    return a.elapsed_time(e) / steps


def _kernel_us(b: int, C: int, iters: int) -> float:
    g = torch.Generator().manual_seed(C)
    z = torch.randn(b, C, generator=g).cuda()
    y = torch.randint(0, C, (b,), generator=g).cuda()
    meter = DeviceMeter("cuda", C)
    for _ in range(10):
        ops.class_metrics(z, y, meter.confusion, meter.top5)
    a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        ops.class_metrics(z, y, meter.confusion, meter.top5)
    e.record()
    e.synchronize()
    return 1e3 * a.elapsed_time(e) / iters


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--kernel-iters", type=int, default=2000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    ops.require()
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine
    from distributed_vgg_f_b200.models.vggf import get_spec

    card = _card()
    b = args.batch
    lines = []
    for model, C in MODELS:
        batch = _val_batch(b, C)
        eng = NativeEngine(get_spec(model, C), device=torch.device("cuda"), batch=b, distributed=False)
        meters = {"off": DeviceMeter("cuda"), "on": DeviceMeter("cuda", C)}
        for m in meters.values():              # warm both paths
            eng.set_meter(m)
            for _ in range(3):
                eng.eval_step(batch)
        eng.sync()
        res = {k: [] for k in meters}
        for _ in range(args.runs):
            for k, m in meters.items():
                eng.set_meter(m)
                res[k].append(_block_ms(eng, batch, args.steps))
        eng.set_meter(None)
        off = statistics.median(res["off"])
        for k in meters:
            ms = statistics.median(res[k])
            rec = dict(card, model=model, classes=C, fused_head=bool(eng.fused_head), val_metrics=k, batch=b,
                       hw=eng.eval_hw, steps_per_block=args.steps, blocks=args.runs, ms_per_batch=round(ms, 4),
                       vs_off=round(ms / off, 4), all_blocks_ms=[round(t, 4) for t in res[k]])
            lines.append(json.dumps(rec))
            print(lines[-1], flush=True)
        del eng
        torch.cuda.empty_cache()
    for _, C in MODELS:
        us = _kernel_us(b, C, args.kernel_iters)
        rec = dict(card, kernel="class_metrics_kernel", batch=b, classes=C, launches=args.kernel_iters,
                   us_per_launch=round(us, 2), scores_bytes=b * C * 4)
        lines.append(json.dumps(rec))
        print(lines[-1], flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
