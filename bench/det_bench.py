"""What --deterministic costs: VGG-F, batch 64, 224^2, synthetic data, on one GPU.

Default and deterministic training steps alternate in one process (device-timed blocks of steps, median
of five per mode), then every split-K launch of the deterministic step is timed alone: the PARTIAL kernel
and its splitk_reduce against the bytes of partial sums they write and read, next to the atomic kernel it
replaces.  Prints one JSON line; the card's name and power limit are read in the same run.

    python bench/det_bench.py [--batch 64] [--steps 10] [--repeats 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


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
        raise SystemExit("det_bench measures on a GPU: none found")
    from distributed_vgg_f_b200 import ops
    from distributed_vgg_f_b200.data import transforms as T
    from distributed_vgg_f_b200.data.loader import FusedBatch
    from distributed_vgg_f_b200.data.synthetic import synthetic_uint8_batch
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine, deterministic_plan
    from distributed_vgg_f_b200.models.vggf import vggf_spec

    C = ops.require()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    B, spec = a.batch, vggf_spec(3)
    imgs, labels = synthetic_uint8_batch(B, 256, 3, seed=0)
    batch = FusedBatch(torch.from_numpy(imgs).pin_memory(), T.sample_train_params(B, 256, 256).pin_memory(),
                       torch.from_numpy(labels).pin_memory(), (256, 256), None)
    engines = {det: NativeEngine(spec, device=dev, batch=B, lr=1e-4, seed=0, deterministic=det) for det in (False, True)}
    times = {False: [], True: []}
    for eng in engines.values():
        _timed(lambda: eng.train_step(batch), 3)           # warm-up: every kernel of the step
    for _ in range(a.repeats):
        for det, eng in engines.items():                      # alternating
            times[det].append(_timed(lambda: eng.train_step(batch), a.steps))
    med = {det: statistics.median(v) for det, v in times.items()}

    # ---- per launch: partial kernel + reduce, against the atomic kernel -------------------------------------
    ws = engines[True]._ws
    layers, h = [], 224
    for i, c in enumerate(spec.convs):
        if i > 0:
            dz = torch.randn(B, h, h, c.cout, device=dev).to(torch.bfloat16)
            x = torch.randn(B, h, h, c.cin, device=dev).to(torch.bfloat16)
            dw = torch.zeros(c.cout, 3, 3, c.cin, device=dev)
            splits = C.conv_wgrad_splits(B, h, h, c.cin, c.cout, C.sm_count())
            n = dw.numel()
            for f in (lambda: C.conv_wgrad(dz, x, dw, 1.0, 0, 0), lambda: C.conv_wgrad_partial(dz, x, ws, 1.0),
                      lambda: ops.splitk_reduce(ws, dw, n, splits)):
                f()
            t_atomic = _timed(lambda: C.conv_wgrad(dz, x, dw, 1.0, 0, 0), 10)
            t_part = _timed(lambda: C.conv_wgrad_partial(dz, x, ws, 1.0), 10)
            t_red = _timed(lambda: ops.splitk_reduce(ws, dw, n, splits), 10)
            moved = (splits + 1) * n * 4                      # reduce: reads the slices, writes dw
            layers.append(dict(layer=c.name, shape="%dx%d^2 %d->%d" % (B, h, c.cin, c.cout), splits=splits,
                               atomic_ms=round(t_atomic, 4), partial_ms=round(t_part, 4), reduce_ms=round(t_red, 4),
                               partial_MB=round(splits * n * 4 / 1e6, 2),
                               reduce_GBs=round(moved / (t_red * 1e-3) / 1e9, 1)))
            del dz, x, dw
        if c.pool_after:
            h //= 2
    plan = deterministic_plan(spec, B, 224, C.sm_count(), engines[True].fused_head)
    res = dict(bench="det_bench", card=_card(), sms=C.sm_count(), model="vggf", batch=B, input_hw=224,
               steps_per_block=a.steps, repeats=a.repeats,
               default_step_ms=round(med[False], 3), deterministic_step_ms=round(med[True], 3),
               slowdown=round(med[True] / med[False], 4),
               default_blocks_ms=[round(v, 3) for v in times[False]], deterministic_blocks_ms=[round(v, 3) for v in times[True]],
               workspace_MB=round(ws.numel() * 4 / 1e6, 1),
               partial_MB_per_step=round(sum(s * e for _, _, s, e in plan) * 4 / 1e6, 1), wgrad_layers=layers)
    print(json.dumps(res))
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
