"""Images/s of the streaming input pipeline (--pipeline stream) against the cached fused pipeline and the reference
loader, on seeded JPEG ImageFolders.

Distributions: ImageNet-like 500 x 375 JPEGs (quality 90, 4:2:0), and mixed sizes from 96 px to 1.5 MP (the
distribution of bench/input_bench.py, same encoder settings).  ``--images`` distinct files are written and each is
hard-linked ``--copies`` times, so an epoch of ``stream`` / ``fused`` is images x copies files (4096 by default, 64
batches: a timed block of several seconds, not a fraction of one).  For each distribution:
  * ``host_decode_img_s`` -- the stream loader alone at 1 / 4 / 8 / 16 decode threads: header layout, entropy
    decode into the pinned slots, nothing on the GPU (median of three epochs);
  * ``decode_kernels`` -- the two decode launches on one batch of 64 (CUDA events over 50 repetitions), and their
    share of the HBM bound: bytes moved, computed from the batch's shapes, over 3.35 TB/s;
  * ``input_img_s`` / ``train_img_s`` -- the loader feeding ``NativeEngine._stage_input`` alone, and the full VGG-F
    ``train_step``, at batch 64 through ``stream``, ``fused`` and ``reference``: the pipelines alternate in blocks
    of one epoch after a warm-up epoch each, and the median of five blocks is reported.  The reference loader's
    epoch is the ``--images`` distinct files (its per-image cost does not depend on the split's length).
The card's name and power limit and the host's CPU model and core count are read in the same run, with where the
model name came from (``cpu_source``) and the CPU identification fields /proc/cpuinfo has.

  python bench/stream_bench.py [--images 512] [--copies 8] [--mb 64] [--reps 5] [--out results.jsonl]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from distributed_vgg_f_b200 import ops                                                      # noqa: E402
from distributed_vgg_f_b200.data.loader import DataManager, _ReferenceLoader, _StreamLoader  # noqa: E402

HBM_BYTES_S = 3.35e12          # H100 SXM data sheet


def _sizes(kind: str, n: int, rng) -> list:
    if kind == "imagenet-500x375":
        return [(375, 500) if i % 4 else (500, 375) for i in range(n)]
    out = []                   # mixed: area log-uniform in [96^2, 1.5 MP], aspect in [1/2, 2] (input_bench.py)
    for _ in range(n):
        area = float(np.exp(rng.uniform(np.log(96 * 96), np.log(1.5e6))))
        ar = float(np.exp(rng.uniform(np.log(0.5), np.log(2.0))))
        out.append((max(96, int(round((area / ar) ** 0.5))), max(96, int(round((area * ar) ** 0.5)))))
    return out


def _write_split(root: str, sizes, rng, copies: int) -> None:
    from PIL import Image

    for i, (h, w) in enumerate(sizes):
        d = os.path.join(root, "TrainData", "c%d" % (i % 3))
        os.makedirs(d, exist_ok=True)
        yy, xx = np.mgrid[0:h, 0:w]
        base = (127 + 90 * np.sin(xx * 0.05 + i) * np.cos(yy * 0.07))[..., None].repeat(3, 2)
        img = np.clip(base + rng.integers(-20, 20, (h, w, 3)), 0, 255).astype(np.uint8)
        p = os.path.join(d, "%04d.jpg" % i)
        Image.fromarray(img).save(p, quality=90, subsampling="4:2:0")
        for c in range(1, copies):
            os.link(p, os.path.join(d, "%04d_%d.jpg" % (i, c)))


def _machine() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    cpu, source, fields = None, None, {}
    try:
        with open("/proc/cpuinfo") as f:
            for line in f:
                if not line.strip():
                    break                       # the first processor's block
                k, _, v = line.partition(":")
                if k.strip() in ("vendor_id", "cpu family", "model", "model name", "CPU implementer", "CPU part"):
                    fields[k.strip()] = v.strip()
    except OSError:
        pass
    if fields.get("model name"):
        cpu, source = fields["model name"], "/proc/cpuinfo"
    else:                   # e.g. hosts whose /proc/cpuinfo names no model
        try:
            out = subprocess.run(["lscpu"], capture_output=True, text=True).stdout
        except OSError:
            out = ""
        cpu = next((line.split(":", 1)[1].strip() for line in out.splitlines() if line.startswith("Model name")), None)
        source = "lscpu" if cpu else "none"
    return {"card": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1],
            "cpu": cpu, "cpu_source": source, "cpuinfo": fields, "cpu_count": os.cpu_count(),
            "cpus_usable": len(os.sched_getaffinity(0))}


def _epoch_rate(fn, loader, epoch: int) -> float:
    """Images/s of one epoch, ending in a device synchronise."""
    loader.set_epoch(epoch)
    torch.cuda.synchronize()
    n, t0 = 0, time.perf_counter()
    for b in loader:
        fn(b)
        n += int((b.labels if hasattr(b, "labels") else b[1]).numel())
    torch.cuda.synchronize()
    return n / (time.perf_counter() - t0)


def _decode_kernels(batch, reps: int = 50) -> dict:
    C = ops.require()
    dev = torch.device("cuda")
    coef, quant, desc, geom = (t.to(dev) for t in (batch.coef, batch.quant, batch.desc, batch.geom))
    raw = batch.raw.to(dev) if batch.raw.numel() else torch.zeros(1, dtype=torch.uint8, device=dev)
    planes = torch.empty(batch.coef.numel(), dtype=torch.uint8, device=dev)
    out = torch.empty(batch.nbytes, dtype=torch.uint8, device=dev)

    def run():
        C.jpeg_decode(coef, quant, desc, geom, raw, planes, out, batch.desc, batch.geom)

    for _ in range(5):
        run()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        run()
    b.record()
    torch.cuda.synchronize()
    ms = a.elapsed_time(b) / reps
    blocks = batch.coef.numel() // 64
    # coefficients read, planes written then read once, raw read, RGB written (tables and rows are negligible)
    moved = blocks * 64 * 2 + blocks * 64 * 2 + batch.raw.numel() + batch.nbytes
    return {"images": int(batch.labels.numel()), "blocks": blocks, "ms": round(ms, 4), "bytes": moved,
            "hbm_bound_ms": round(moved / HBM_BYTES_S * 1e3, 4),
            "share_of_hbm_bound": round(moved / HBM_BYTES_S * 1e3 / ms, 4)}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=512)
    ap.add_argument("--copies", type=int, default=8)
    ap.add_argument("--mb", type=int, default=64)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("stream_bench needs a CUDA device")
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine
    from distributed_vgg_f_b200.models.vggf import vggf_spec

    def emit(rec):
        line = json.dumps(rec)
        print(line, flush=True)
        if a.out:
            with open(a.out, "a") as f:
                f.write(line + "\n")

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    emit(_machine())
    eng = NativeEngine(vggf_spec(3), device=dev, batch=a.mb, lr=1e-4, seed=0)
    rng = np.random.default_rng(0)

    def stage(b):
        eng._stage_input(b)
        eng._release_input()

    for kind in ("imagenet-500x375", "mixed-96px-1.5MP"):
        with tempfile.TemporaryDirectory() as root:
            sizes = _sizes(kind, a.images, rng)
            _write_split(root, sizes, rng, a.copies)
            res = {"dist": kind, "images": a.images, "copies": a.copies, "mb": a.mb,
                   "mean_mpix": round(float(np.mean([h * w for h, w in sizes])) / 1e6, 3),
                   "jpeg_mb": round(sum(os.path.getsize(os.path.join(d, f)) for d, _, fs in os.walk(root)
                                        for f in fs) / 2**20, 1)}
            sdm = DataManager(root, a.mb, train=True, pipeline="stream")
            stream = sdm.get_loader()
            host = {}
            for t in (1, 4, 8, 16):
                ld = _StreamLoader(sdm.samples, a.mb, True, None, True, 0, threads=t)
                host[str(t)] = round(statistics.median(_epoch_rate(lambda b: None, ld, e) for e in range(3)), 1)
                del ld
            res["host_decode_img_s"] = host
            res["decode_kernels"] = _decode_kernels(next(iter(stream)))
            fused_dm = DataManager(root, a.mb, train=True, pipeline="fused")
            loaders = {"stream": stream, "fused": fused_dm.get_loader(),
                       "reference": _ReferenceLoader(fused_dm.samples[::a.copies], a.mb, True, None, True, 0)}
            for what, fn in (("input_img_s", stage), ("train_img_s", lambda b: eng.train_step(b))):
                for ld in loaders.values():            # warm-up epoch
                    _epoch_rate(fn, ld, 0)
                rates = {k: [] for k in loaders}
                for r in range(a.reps):
                    for k, ld in loaders.items():
                        rates[k].append(_epoch_rate(fn, ld, r + 1))
                res[what] = {k: round(statistics.median(v), 1) for k, v in rates.items()}
                res[what + "_blocks"] = {k: [round(x, 1) for x in v] for k, v in rates.items()}
            emit(res)


if __name__ == "__main__":
    main()
