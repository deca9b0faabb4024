"""What --freeze-layers saves: VGG-F, batch 64, 224^2, synthetic data, on one GPU.

One engine per frozen count N in {0, 7, 10, 13, 16} (0: everything trains; 13: all of features; 16: only the
last Linear).  Their training steps alternate in one process (device-timed blocks of steps, median of five
per N), so that every count sees the same clocks and neighbours.  Also reported per N: images per second,
launches per step and the memory of what freezing shrinks (fp32 gradient + Adam moments, and the bf16 wire a
multi-GPU run would allocate).  Then the same alternation for N in {0, 13} with the model EMA updated on every
step (--model-ema-steps 1, the most often it can run): what the EMA of the frozen range (ema_kernel) adds next to
the EMA the optimizer kernels keep.  Prints one JSON line; the card's name and power limit are read in the same run.

    python bench/freeze_bench.py [--batch 64] [--steps 10] [--repeats 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

COUNTS = (0, 7, 10, 13, 16)
EMA_COUNTS = (0, 13)


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out or torch.cuda.get_device_name(0) + ", power limit unknown"


def _timed(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=10, help="steps per timed block")
    ap.add_argument("--repeats", type=int, default=5)
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("freeze_bench measures on a GPU: none found")
    from distributed_vgg_f_b200 import ops
    from distributed_vgg_f_b200.data import transforms as T
    from distributed_vgg_f_b200.data.loader import FusedBatch
    from distributed_vgg_f_b200.data.synthetic import synthetic_uint8_batch
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine
    from distributed_vgg_f_b200.models.vggf import vggf_spec

    ops.require()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    B, spec = a.batch, vggf_spec(3)
    imgs, labels = synthetic_uint8_batch(B, 256, 3, seed=0)
    batch = FusedBatch(torch.from_numpy(imgs).pin_memory(), T.sample_train_params(B, 256, 256).pin_memory(),
                       torch.from_numpy(labels).pin_memory(), (256, 256), None)
    init = NativeEngine(spec, device=dev, batch=B, lr=1e-4, seed=0).export_state()     # one set of weights for all
    engines = {n: NativeEngine(spec, device=dev, batch=B, lr=1e-4, seed=0, init_state=init, freeze_layers=n)
               for n in COUNTS}
    times = {n: [] for n in COUNTS}
    launches = {}
    for n, eng in engines.items():
        _timed(lambda: eng.train_step(batch), 3)           # warm-up: every kernel of the step
        c0 = ops.launch_count()
        eng.train_step(batch)
        eng.sync()
        launches[n] = ops.launch_count() - c0
    for _ in range(a.repeats):
        for n, eng in engines.items():                      # alternating
            times[n].append(_timed(lambda: eng.train_step(batch), a.steps))
    rows = []
    for n, eng in engines.items():
        med = statistics.median(times[n])
        moments = eng.m32.numel() + (eng.v32.numel() if eng.v32 is not None else 0)
        rows.append(dict(freeze_layers=n, step_ms=round(med, 3), images_per_s=round(B / (med * 1e-3), 1),
                         speedup=round(statistics.median(times[0]) / med, 3), blocks_ms=[round(v, 3) for v in times[n]],
                         launches_per_step=launches[n], grad_elems=eng.n_grad,
                         grad_moments_wire_MB=round((eng.g32.numel() + moments) * 4 / 1e6 + eng.n_grad * 2 / 1e6, 1)))
    del engines
    torch.cuda.empty_cache()
    ema = {n: NativeEngine(spec, device=dev, batch=B, lr=1e-4, seed=0, init_state=init, freeze_layers=n, ema_decay=0.999)
           for n in EMA_COUNTS}
    ema_times = {n: [] for n in EMA_COUNTS}
    for n, eng in ema.items():
        _timed(lambda: eng.train_step(batch, ema=True), 3)
    for _ in range(a.repeats):
        for n, eng in ema.items():
            ema_times[n].append(_timed(lambda: eng.train_step(batch, ema=True), a.steps))
    ema_rows = [dict(freeze_layers=n, step_ms=round(statistics.median(ema_times[n]), 3),
                     without_ema_ms=next(r["step_ms"] for r in rows if r["freeze_layers"] == n),
                     blocks_ms=[round(v, 3) for v in ema_times[n]]) for n in EMA_COUNTS]
    res = dict(bench="freeze_bench", card=_card(), model="vggf", batch=B, input_hw=224, optimizer="adam",
               steps_per_block=a.steps, repeats=a.repeats, rows=rows, ema_every_step=ema_rows)
    print(json.dumps(res))
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
