"""What test-time augmentation (--val-tta) costs on the native engine, one GPU: evaluation of a batch of 64 at 224^2.

Prints one JSON line per (model, mode), with the card's name and power limit read in the same run: milliseconds per
evaluation batch and images per second for none, flip, five-crop and ten-crop, for VGG-F and vggf11.  The modes run
in alternating blocks of --steps batches; each figure is the median over --runs blocks.  The input is a validation
FusedBatch of 256 x 256 images (Resize 256, crop 224), the fused input path every mode shares.  With --out the lines
are also written to that file.
Usage: ``python bench/tta_bench.py [--steps 10] [--runs 5] [--out bench/results/tta_bench_h100.jsonl]``.
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
from ema_bench import _card  # noqa: E402

MODES = ("none", "flip", "five-crop", "ten-crop")


def _val_batch(b: int) -> FusedBatch:
    g = torch.Generator().manual_seed(0)
    src = torch.randint(0, 256, (b, 256, 256, 3), dtype=torch.uint8, generator=g)
    return FusedBatch(src.pin_memory(), T.val_params(b, 256, 256).pin_memory(),
                      torch.randint(0, 3, (b,), generator=g).pin_memory(), T.resized_dims(False, 256, 256), None)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    ops.require()
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine
    from distributed_vgg_f_b200.models.vggf import get_spec

    card = _card()
    b = args.batch
    batch = _val_batch(b)
    lines = []
    for model in ("vggf", "vggf11"):
        eng = NativeEngine(get_spec(model, 3), device=torch.device("cuda"), batch=b, distributed=False)
        for mode in MODES:                     # warm every view shape
            eng.set_val_tta(mode)
            for _ in range(3):
                eng.eval_step(batch)
        eng.sync()
        res = {m: [] for m in MODES}
        for _ in range(args.runs):
            for mode in MODES:
                eng.set_val_tta(mode)
                a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(args.steps):
                    eng.eval_step(batch)
                e.record()
                e.synchronize()
                res[mode].append(a.elapsed_time(e) / args.steps)
        base = statistics.median(res["none"])
        for mode in MODES:
            ms = statistics.median(res[mode])
            rec = dict(card, model=model, mode=mode, views=len(T.tta_views(mode)), batch=b, hw=eng.eval_hw,
                       steps_per_block=args.steps, blocks=args.runs, ms_per_batch=round(ms, 3),
                       img_s=round(b / (ms * 1e-3), 1), vs_none=round(ms / base, 3),
                       all_blocks_ms=[round(t, 3) for t in res[mode]])
            lines.append(json.dumps(rec))
            print(lines[-1], flush=True)
        del eng
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
