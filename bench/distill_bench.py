"""What knowledge distillation costs on the native engine, one GPU, batch 64 at 224^2.

Prints one JSON line per case, each with the card's name and power limit read in the same run:
  * "step": training step time of VGG-F alone, VGG-F with a VGG-F teacher, vggf11 alone and vggf11 with a VGG-F
    teacher, in alternating blocks of --steps steps, median over --runs blocks, and images per second;
  * with a teacher, "teacher_ms" (its forward on the staged input: the convolutions, the FC stack and the fused head's
    evaluation pass) and "loss_ms" (the distillation-loss launch, head_ce_kd: forward, loss and the head's backward),
    against "ce_loss_ms" (the same launch without the teacher, head_ce); median device time of --reps launches each.
Usage: ``python bench/distill_bench.py [--steps 10] [--runs 5] [--reps 20]``.
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

ALPHA, TEMPERATURE = 0.5, 4.0


def _engine(model: str, b: int):
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine
    from distributed_vgg_f_b200.models.vggf import get_spec

    return NativeEngine(get_spec(model, 3), device=torch.device("cuda"), batch=b, distributed=False)


def _teacher(b: int):
    from distributed_vgg_f_b200.engine.native_engine import TeacherEngine
    from distributed_vgg_f_b200.models.vggf import build_oracle, get_spec

    spec = get_spec("vggf", 3)
    return TeacherEngine(spec, torch.device("cuda"), b, build_oracle(spec, seed=1).state_dict())


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    ops.require()
    card = _card()
    b = args.batch
    batch = _batch(b)
    engines = {}
    for model in ("vggf", "vggf11"):
        engines[model] = _engine(model, b)
        engines[model + "+vggf teacher"] = eng = _engine(model, b)
        eng.set_distillation(_teacher(b), ALPHA, TEMPERATURE)
    res = {k: [] for k in engines}
    for eng in engines.values():
        for _ in range(3):
            eng.train_step(batch)
        eng.sync()
    for _ in range(args.runs):
        for name, eng in engines.items():
            a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.steps):
                eng.train_step(batch)
            e.record()
            e.synchronize()
            res[name].append(a.elapsed_time(e) / args.steps)
    for name, eng in engines.items():
        ms = statistics.median(res[name])
        base = statistics.median(res[name.split("+")[0]])
        rec = dict(card, what="step", case=name, batch=b, hw=eng.HW, steps_per_block=args.steps, blocks=args.runs,
                   ms_per_step=round(ms, 3), img_s=round(b / (ms * 1e-3), 1), vs_alone=round(ms / base, 4),
                   all_blocks_ms=[round(t, 3) for t in res[name]])
        if eng.teacher is not None:
            eng.apply_updates = False              # the loss launches below only rewrite the head's gradient
            rec["teacher_ms"] = round(_time(lambda: eng.teacher.forward_teacher(eng.x_nhwc, eng.labels_dev, b),
                                            args.reps), 4)
            rec["loss_ms"] = round(_time(lambda: eng._loss(b, train=True), args.reps), 4)
            teacher, eng.teacher = eng.teacher, None
            rec["ce_loss_ms"] = round(_time(lambda: eng._loss(b, train=True), args.reps), 4)
            eng.teacher = teacher
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
