"""What label smoothing, MixUp and CutMix cost on the native engine.

For a uniform split (128 x 128 sources, the fused ``augment`` kernel) and a ragged split (images of
mixed sizes, the two-pass ``augment_ragged``), at the network's 224 x 224 input and batch 64, prints
one JSON line per case (off, label smoothing, MixUp, CutMix) with
  * augment_ms: device time of the input transform alone (CUDA events, median of --reps launches);
  * step_img_s: full VGG-F training steps per second x batch (median of --steps timed steps).
Usage: ``python bench/mix_bench.py [--model vggf] [--batch 64] [--steps 20] [--reps 50]``.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from distributed_vgg_f_b200 import ops  # noqa: E402
from distributed_vgg_f_b200.data import transforms as T  # noqa: E402
from distributed_vgg_f_b200.data.loader import FusedBatch, RaggedBatch  # noqa: E402

CASES = {"off": (0.0, None), "label_smoothing": (0.1, None),
         "mixup": (0.0, T.MixDraw("mixup", 0.37, (0, 0, 0, 0))),
         "cutmix": (0.0, T.MixDraw("cutmix", 1.0 - 112 * 112 / 224 ** 2, (56, 56, 168, 168)))}


def _batch(split: str, b: int):
    g = torch.Generator().manual_seed(0)
    y = torch.randint(0, 3, (b,), generator=g)
    if split == "uniform":
        src = torch.randint(0, 256, (b, 128, 128, 3), dtype=torch.uint8, generator=g)
        return FusedBatch(src.pin_memory(), T.sample_train_params(b, 128, 128, g).pin_memory(), y.pin_memory(),
                          T.resized_dims(True, 128, 128), None)
    sizes = [(480, 640), (375, 500), (256, 256), (600, 400), (333, 500)]
    hw = [sizes[i % len(sizes)] for i in range(b)]
    geom = T.ragged_geometry(hw, train=True)
    data = torch.randint(0, 256, (int(sum(h * w * 3 for h, w in hw)),), dtype=torch.uint8, generator=g)
    params = torch.cat([T.sample_train_params(1, h, w, g) for h, w in hw])
    return RaggedBatch(data.pin_memory(), geom.pin_memory(), params.pin_memory(), y.pin_memory(), None)


def _augment_ms(batch, mix, reps: int) -> float:
    dev = torch.device("cuda")
    out = torch.empty(len(batch.labels), 224, 224, 4, dtype=torch.bfloat16, device=dev)
    if isinstance(batch, FusedBatch):
        src, prm = batch.images_u8.to(dev), batch.params.to(dev)
        run = lambda: ops.augment(src, prm, out, batch.resized_hw, mode="nhwc", pad=4, mix=mix)  # noqa: E731
    else:
        data, geom, prm = batch.data_u8.to(dev), batch.geom.to(dev), batch.params.to(dev)
        inter = torch.empty(ops.ragged_inter_bytes(batch.geom), dtype=torch.uint8, device=dev)
        run = lambda: ops.augment_ragged(data, geom, prm, inter, out, batch.geom, batch.params, mix=mix)  # noqa: E731
    for _ in range(5):
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


def _step_img_s(model: str, batch, eps: float, mix, steps: int) -> float:
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine
    from distributed_vgg_f_b200.models.vggf import get_spec

    b = len(batch.labels)
    eng = NativeEngine(get_spec(model, 3), device=torch.device("cuda"), batch=b, label_smoothing=eps,
                       distributed=False)
    batch = batch._replace(mix=mix)
    for _ in range(5):
        eng.train_step(batch)
    eng.sync()
    times = []
    for _ in range(steps):
        a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        eng.train_step(batch)
        e.record()
        e.synchronize()
        times.append(a.elapsed_time(e))
    del eng
    torch.cuda.empty_cache()
    return b / (statistics.median(times) * 1e-3)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="vggf")
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    ops.require()
    gpu = torch.cuda.get_device_name()
    for split in ("uniform", "ragged"):
        batch = _batch(split, args.batch)
        for case, (eps, mix) in CASES.items():
            print(json.dumps({"split": split, "case": case, "batch": args.batch, "gpu": gpu,
                              "augment_ms": round(_augment_ms(batch, mix, args.reps), 4),
                              "step_img_s": round(_step_img_s(args.model, batch, eps, mix, args.steps), 1)}),
                  flush=True)


if __name__ == "__main__":
    main()
