"""Images/s of the fused input pipeline per source-size distribution, against the reference pipeline.

For each distribution a small ImageFolder split is written as JPEGs to a temporary directory, then:
  * ``input``  -- the fused pipeline alone: prefetch thread -> async H2D -> augment kernels
                  (``NativeEngine._stage_input``), with a device synchronise at the end;
  * ``train``  -- the same loader feeding the full VGG-F ``train_step``;
  * ``reference`` -- the per-sample PIL + torchvision loader (decode and transforms per image).
Distributions: uniform 128^2 (the ``FusedBatch`` path), uniform 480x640, and mixed sizes from 96 px to
1.5 MP (both ``RaggedBatch``).  The first pass over each split is a warm-up and is not timed.
Prints one JSON line per distribution, and the card's name and power limit read in the same run.

  python bench/input_bench.py [--images 256] [--mb 64] [--epochs 3]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from distributed_vgg_f_b200.data.loader import DataManager, _ReferenceLoader   # noqa: E402


def _sizes(kind: str, n: int, rng) -> list:
    if kind == "uniform-128":
        return [(128, 128)] * n
    if kind == "uniform-480x640":
        return [(480, 640)] * n
    out = []                      # mixed: area log-uniform in [96^2, 1.5 MP], aspect in [1/2, 2]
    for _ in range(n):
        area = float(np.exp(rng.uniform(np.log(96 * 96), np.log(1.5e6))))
        ar = float(np.exp(rng.uniform(np.log(0.5), np.log(2.0))))
        h = max(96, int(round((area / ar) ** 0.5)))
        w = max(96, int(round((area * ar) ** 0.5)))
        out.append((h, w))
    return out


def _write_split(root: str, sizes, rng) -> None:
    from PIL import Image

    for i, (h, w) in enumerate(sizes):
        d = os.path.join(root, "TrainData", "c%d" % (i % 3))
        os.makedirs(d, exist_ok=True)
        yy, xx = np.mgrid[0:h, 0:w]
        base = (127 + 90 * np.sin(xx * 0.05 + i) * np.cos(yy * 0.07))[..., None].repeat(3, 2)
        img = np.clip(base + rng.integers(-20, 20, (h, w, 3)), 0, 255).astype(np.uint8)
        Image.fromarray(img).save(os.path.join(d, "%04d.jpg" % i), quality=90)


def _card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"card": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def _rate(fn, loader, epochs: int) -> float:
    """Images/s over epochs 2..epochs (epoch 1 warms up), ending in a device synchronise."""
    n, t0 = 0, None
    for e in range(epochs):
        loader.set_epoch(e)
        if e == 1:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
        for b in loader:
            fn(b)
            if e >= 1:                      # FusedBatch / RaggedBatch, or the reference's (x, y)
                n += int((b[1] if isinstance(b, tuple) and len(b) == 2 else b.labels).numel())
    torch.cuda.synchronize()
    return n / (time.perf_counter() - t0)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=256)
    ap.add_argument("--mb", type=int, default=64)
    ap.add_argument("--epochs", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("input_bench needs a CUDA device")
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine
    from distributed_vgg_f_b200.models.vggf import vggf_spec

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    print(json.dumps(_card()), flush=True)
    eng = NativeEngine(vggf_spec(3), device=dev, batch=a.mb, lr=1e-4, seed=0)
    rng = np.random.default_rng(0)

    def stage(b):
        eng._stage_input(b)
        eng._release_input()

    for kind in ("uniform-128", "uniform-480x640", "mixed-96px-1.5MP"):
        with tempfile.TemporaryDirectory() as root:
            sizes = _sizes(kind, a.images, rng)
            _write_split(root, sizes, rng)
            dm = DataManager(root, a.mb, train=True, pipeline="fused")
            ld = dm.get_loader()
            res = {"dist": kind, "images": a.images, "mb": a.mb, "batch_type": type(next(iter(ld))).__name__,
                   "mean_mpix": round(float(np.mean([h * w for h, w in sizes])) / 1e6, 3),
                   "input_img_s": round(_rate(stage, ld, a.epochs), 1),
                   "train_step_img_s": round(_rate(lambda b: eng.train_step(b), ld, a.epochs), 1)}
            ref = _ReferenceLoader(dm.samples, a.mb, True, None, True, 0)
            res["reference_loader_img_s"] = round(_rate(lambda b: None, ref, 2), 1)
            print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
