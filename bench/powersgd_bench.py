"""What --powersgd-rank costs on one GPU: the compression kernels alone, and VGG-F's training step.

Kernels: psgd_project, psgd_backproject (with its split reduction), psgd_orthogonalize (of P and of Q) and
psgd_decompress at FC-1 (4096 x 25088), FC-2 (4096 x 4096) and a 512 x 4608 convolution, r = 1, 4 and 8, timed
with CUDA events over many launches, each as a share of the HBM bound of the bytes it must move (3.35 TB/s, the
H100 SXM data sheet): project reads g and e and writes e, back-project reads M, decompress reads M and writes g
and e (n m 4 bytes each), plus P, Q and the workspace.

Step: VGG-F, batch 64, 224^2, Adam, world 1, one engine per rank r in {0, 1, 4, 8} with --powersgd-start-iter 2
and every engine past its start iteration before timing, so r > 0 compresses on every timed step.  The engines'
steps alternate in one process (device-timed blocks, median of five per r).  At world 1 there is no wire: the
step time is what the compression adds to the GPU's own work; the bytes per update it would save on a network
are printed beside it (computed from the shapes).  Prints one JSON line; the card's name and power limit are
read in the same run.

    python bench/powersgd_bench.py [--batch 64] [--steps 10] [--repeats 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM = 3.35e12
RANKS = (0, 1, 4, 8)
SHAPES = (("fc1", 4096, 25088), ("fc2", 4096, 4096), ("conv512", 512, 4608))


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


def kernels(ops, reps: int = 20) -> list:
    rows = []
    for what, n, m in SHAPES:
        g = torch.randn(n, m, device="cuda") * 1e-3
        e = torch.zeros(n, m, device="cuda")
        for r in (1, 4, 8):
            q = torch.randn(m, r, device="cuda")
            p = torch.empty(n, r, device="cuda")
            ws = torch.empty(ops.psgd_workspace_elems(n, m, r), device="cuda")
            ops.psgd_orthogonalize(q, rows=m, rank=r)
            nm = n * m * 4
            pq = (n + m) * r * 4
            cases = {
                "project": (lambda: ops.psgd_project(g, e, q, p, n=n, m=m, rank=r, scale=1.0), 3 * nm + pq),
                "backproject": (lambda: ops.psgd_backproject(e, p, q, ws, n=n, m=m, rank=r), nm + pq + 2 * ws.numel() * 4),
                "orthogonalize_P": (lambda: ops.psgd_orthogonalize(p, rows=n, rank=r), 2 * n * r * 4),
                "orthogonalize_Q": (lambda: ops.psgd_orthogonalize(q, rows=m, rank=r), 2 * m * r * 4),
                "decompress": (lambda: ops.psgd_decompress(p, q, g, e, n=n, m=m, rank=r, alpha=1.0), 3 * nm + pq),
            }
            for k, (fn, nbytes) in cases.items():
                _timed(fn, 3)
                ms = _timed(fn, reps)
                rows.append(dict(shape=what, n=n, m=m, rank=r, kernel=k, us=round(ms * 1e3, 2), bytes=nbytes,
                                 hbm_bound_us=round(nbytes / HBM * 1e6, 2),
                                 share_of_hbm_bound=round(nbytes / HBM / (ms * 1e-3), 3)))
        del g, e
        torch.cuda.empty_cache()
    return rows


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=10, help="steps per timed block")
    ap.add_argument("--repeats", type=int, default=5)
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("powersgd_bench measures on a GPU: none found")
    from distributed_vgg_f_b200 import ops
    from distributed_vgg_f_b200.data import transforms as T
    from distributed_vgg_f_b200.data.loader import FusedBatch
    from distributed_vgg_f_b200.data.synthetic import synthetic_uint8_batch
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine
    from distributed_vgg_f_b200.models.vggf import vggf_spec
    from distributed_vgg_f_b200.parallel import powersgd

    ops.require()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    kernel_rows = kernels(ops)
    B, spec = a.batch, vggf_spec(3)
    imgs, labels = synthetic_uint8_batch(B, 256, 3, seed=0)
    batch = FusedBatch(torch.from_numpy(imgs).pin_memory(), T.sample_train_params(B, 256, 256).pin_memory(),
                       torch.from_numpy(labels).pin_memory(), (256, 256), None)
    init = NativeEngine(spec, device=dev, batch=B, lr=1e-4, seed=0).export_state()
    engines = {r: NativeEngine(spec, device=dev, batch=B, lr=1e-4, seed=0, init_state=init, powersgd_rank=r,
                               powersgd_start_iter=2) for r in RANKS}
    times = {r: [] for r in RANKS}
    launches = {}
    for r, eng in engines.items():
        _timed(lambda: eng.train_step(batch), 4)           # past the start iteration, every kernel warmed up
        c0 = ops.launch_count()
        eng.train_step(batch)
        eng.sync()
        launches[r] = ops.launch_count() - c0
    for _ in range(a.repeats):
        for r, eng in engines.items():                      # alternating
            times[r].append(_timed(lambda: eng.train_step(batch), a.steps))
    rows = []
    for r in RANKS:
        med = statistics.median(times[r])
        b = powersgd.exchange_bytes(powersgd.plan(spec, r)) if r else None
        rows.append(dict(rank=r, step_ms=round(med, 3), images_per_s=round(B / (med * 1e-3), 1),
                         vs_rank0=round(med / statistics.median(times[0]), 3), blocks_ms=[round(v, 3) for v in times[r]],
                         launches_per_step=launches[r],
                         exchange_MB_per_update=round((b["total"] if b else 2 * spec.num_params) / 1e6, 3)))
    res = dict(bench="powersgd_bench", card=_card(), model="vggf", batch=B, input_hw=224, optimizer="adam", world=1,
               steps_per_block=a.steps, repeats=a.repeats, step=rows, kernels=kernel_rows)
    print(json.dumps(res))
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
