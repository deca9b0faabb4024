"""Gradient accumulation on the native engine: what a micro-batch without an update costs, training
throughput at K = 1, 2, 4, 8, and the FC-1 weight-gradient GEMM with the storing and the red.add
epilogue (the latter is what the later micro-batches of a group use).

    python bench/accum_bench.py                      # one GPU: VGG-F, batch 64, synthetic data
    torchrun --nproc-per-node 2 bench/accum_bench.py # + all-reduce ms per update, fused and --allreduce nccl

All times are CUDA-event times around work that ends in a device synchronise; K runs alternate.  The
wire bytes per image are counted from the engine's bucket plan (no GPU needed for those: --plan-only).
Multi-host links cannot be measured on one machine: those rows say "not measured".
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def card(torch, index):
    """Card name and power limit, read in the same run as the measurement."""
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=name,power.limit",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = [s.strip() for s in out.split(",")[:2]]
        return name, limit
    except (OSError, ValueError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(index), "unknown (nvidia-smi unavailable)"


def wire_plan(spec, batch, world, K, bucket_mb=32.0):
    """Bytes on the wire per update and per image for the fused bf16 exchange and the fp32 NCCL one."""
    from distributed_vgg_f_b200.models import layout as L
    from distributed_vgg_f_b200.parallel.buckets import engine_bucket_plan

    plan = engine_bucket_plan(L.ready_order(spec), bucket_mb, 9.5, 2400.0)
    images = batch * K * world
    return {"arena_elements": plan.total, "buckets": len(plan.buckets),
            "fused_bf16_MB_per_update": round(plan.total * 2 / 1e6, 2),
            "nccl_fp32_MB_per_update": round(plan.total * 4 / 1e6, 2),
            "fused_bf16_MB_per_image": round(plan.total * 2 / images / 1e6, 4),
            "nccl_fp32_MB_per_image": round(plan.total * 4 / images / 1e6, 4)}


def timed(torch, device, body, n):
    torch.cuda.synchronize(device)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for k in range(n):
        body(k)
    e1.record()
    torch.cuda.synchronize(device)
    return e0.elapsed_time(e1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--micro", type=int, default=32, help="micro-batches per timed run (a multiple of 8)")
    ap.add_argument("--rounds", type=int, default=2, help="alternating rounds over K = 1, 2, 4, 8")
    ap.add_argument("--plan-only", action="store_true", help="print the wire-byte count and exit (no GPU)")
    args = ap.parse_args()

    import torch

    from distributed_vgg_f_b200.models.vggf import vggf_spec

    spec = vggf_spec(3)
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if args.plan_only:
        for K in (1, 2, 4, 8):
            print(json.dumps({"K": K, "world": max(world, 2), **wire_plan(spec, args.batch, max(world, 2), K)}))
        return
    if not torch.cuda.is_available():
        raise SystemExit("accum_bench: needs a CUDA device (use --plan-only for the byte count)")

    import torch.distributed as dist

    import bench as B                     # the flagship benchmark's synthetic batches
    from distributed_vgg_f_b200 import ops
    from distributed_vgg_f_b200.data.loader import FusedBatch
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine

    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    rank = dist.get_rank() if world > 1 else 0
    name, limit = card(torch, local)
    res = {"card": name, "power_limit": limit, "world": world, "batch": args.batch, "model": "vggf (3 classes)"}
    host = B.make_host_batches(torch, 4, args.batch, 3, seed=rank + 1)
    batches = [FusedBatch(b.images_u8.to(dev), b.params.to(dev), b.labels.to(dev), b.resized_hw, None) for b in host]

    def engine(allreduce="auto"):
        return NativeEngine(spec, device=dev, batch=args.batch, lr=1e-5, seed=0, allreduce=allreduce)

    eng = engine()
    for k in range(8):
        eng.train_step(batches[k % 4])

    # ---- one micro-batch with and without the update ---------------------------------------------
    n = 20
    ms = {"update": [], "no_update": []}
    for _ in range(2):
        for mode in ("no_update", "update"):
            upd = mode == "update"
            ms[mode].append(timed(torch, dev, lambda k: eng.train_step(batches[k % 4], update=upd), n) / n)
            if not upd:
                eng.train_step(batches[0])                  # close the group
    res["ms_per_micro_batch"] = {k: round(min(v), 3) for k, v in ms.items()}

    # ---- throughput at K = 1, 2, 4, 8, alternating -------------------------------------------------
    assert args.micro % 8 == 0
    ips = {K: [] for K in (1, 2, 4, 8)}
    for _ in range(args.rounds):
        for K in (1, 2, 4, 8):
            t = timed(torch, dev, lambda k: eng.train_step(batches[k % 4], update=(k + 1) % K == 0), args.micro)
            ips[K].append(args.micro * args.batch / (t / 1e3))
    res["images_per_s"] = {str(K): [round(v, 1) for v in ips[K]] for K in ips}

    # ---- FC-1 wgrad: store vs red.add epilogue -----------------------------------------------------
    f = spec.fcs[0]
    dz = torch.randn(args.batch, f.fout, device=dev).to(torch.bfloat16)
    x = torch.randn(args.batch, f.fin, device=dev).to(torch.bfloat16)
    out = torch.zeros(f.fout, f.fin, device=dev)
    wg = {"f32_store": [], "f32_atomic": []}
    reps = 30
    for epi in list(wg) * 3:
        wg[epi].append(timed(torch, dev, lambda k: ops.gemm(dz, x, out, M=f.fout, N=f.fin, K=args.batch, a_mn=True,
                                                              b_mn=True, epi=epi, ldo=f.fin), reps) / reps)
    res["fc1_wgrad_ms"] = {k: round(min(v), 4) for k, v in wg.items()}

    # ---- >= 2 ranks: the exchange per update ---------------------------------------------------------
    res["wire"] = {str(K): wire_plan(spec, args.batch, max(world, 2), K) for K in (1, 2, 4, 8)}
    if world > 1:
        eng.comm_timing(True)
        for k in range(8):
            eng.train_step(batches[k % 4], update=k % 2 == 1)
        rep = eng.comm_report(4)
        eng.comm_timing(False)
        res["fused_allreduce_ms_per_update"] = rep["ms_per_step"] if rep else None
        del eng
        nc = engine("nccl")
        per = {}
        for upd in (False, True, False, True):
            t = timed(torch, dev, lambda k: nc.train_step(batches[k % 4], update=upd), 10) / 10
            per.setdefault(upd, []).append(t)
            if not upd:
                nc.train_step(batches[0])
        # step with the NCCL exchange + optimizer minus the step without: what the update adds
        res["nccl_update_minus_no_update_ms"] = round(min(per[True]) - min(per[False]), 3)
    else:
        res["fused_allreduce_ms_per_update"] = "not measured (one GPU)"
        res["nccl_update_minus_no_update_ms"] = "not measured (one GPU)"
    res["multi_host_link"] = "not measured"
    if rank == 0:
        print(json.dumps(res))
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
