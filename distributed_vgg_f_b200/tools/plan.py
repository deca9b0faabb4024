"""Print the gradient-exchange plan of a model without touching a GPU: arena layout in gradient-ready order,
buckets, wire bytes, and which path each bucket takes at a given world size.

    python -m distributed_vgg_f_b200.tools.plan --model vggf --num-classes 3 --world 8

What DDP's Reducer decides at run time from autograd hooks (distributedVggf.py:225; rebuilt buckets of 1 / 25 MiB,
SURVEY N3), this framework fixes before the first step because it owns backward: the table below is exactly what
``NativeEngine`` executes (``parallel/buckets.py::engine_bucket_plan``, ``parallel/symm.py::pick_algo``)."""
from __future__ import annotations

import argparse

from ..models import layout as L
from ..models.vggf import get_spec
from ..parallel.buckets import engine_bucket_plan
from ..parallel.symm import ONESHOT_MAX_BYTES, ONESHOT_MAX_BYTES_NVLS


def describe(model: str = "vggf", num_classes: int = 3, world: int = 8, multicast: bool = True, zero1: str = "auto",
             bucket_mb: float = 32.0, conv_bucket_mb: float = 9.5, tail_bucket_kb: float = 2400.0,
             freeze_layers: int = 0):
    spec = get_spec(model, num_classes)
    ready = L.ready_order(spec)
    plan = engine_bucket_plan(ready, bucket_mb, conv_bucket_mb, tail_bucket_kb,
                              trainable=len(ready) - len(spec.frozen_param_names(freeze_layers)))
    fc_w = {f.name + ".weight" for f in spec.fcs}
    prepacked = set()
    for name in fc_w:
        ids = plan.bucket_of(name)
        if ids and all(plan.buckets[i].tensors == (name,) for i in ids):
            prepacked.update(ids)
    z1 = world >= 4 if zero1 == "auto" else zero1 == "on"
    rows = []
    for b in plan.buckets:
        wire = b.numel * 2
        if world == 1:
            path = "optimizer only"
        else:
            limit = ONESHOT_MAX_BYTES_NVLS if multicast else ONESHOT_MAX_BYTES
            algo = "oneshot" if wire <= limit else ("nvls" if multicast else "twoshot")
            if b.index in prepacked and algo == "oneshot":
                algo = "twoshot"
            fused = z1 and b.index in prepacked and algo != "oneshot"
            entry = "wire written by the wgrad GEMM" if b.index in prepacked else "pack fp32 -> bf16 * 1/ws"
            path = ("zero1: reduce-scatter + Adam + all-gather, " if fused else "all-reduce + Adam, ") + algo + ", " + entry
        rows.append((b.index, b.numel, wire, len(b.tensors), b.tensors[0], b.tensors[-1], path))
    return plan, rows


def frozen_lines(model: str, num_classes: int, plan, freeze_layers: int) -> list:
    """What --freeze-layers leaves out of the exchange: the frozen layers and where the gradient arena ends."""
    spec = get_spec(model, num_classes)
    names = spec.frozen_param_names(freeze_layers)
    if not names:
        return []
    layers = [l.name for l in list(spec.convs) + list(spec.fcs)][:freeze_layers]
    n = sum(plan.numels[t] for t in names)
    return ["frozen: %d layers, %s .. %s, %d parameters (native layouts); gradient arena, moments and wire end at "
            "T = %d of %d elements (%.1f MB of fp32 gradient instead of %.1f)"
            % (freeze_layers, layers[0], layers[-1], n, plan.grad_total, plan.total, plan.grad_total * 4 / 1e6,
               plan.total * 4 / 1e6)]


def deterministic(model: str, num_classes: int, batch: int, input_hw: int, sms: int, freeze_layers: int = 0) -> int:
    """Split count and partial-sum bytes of every split-K launch of a --deterministic step, from the
    launchers' own host arithmetic: needs the built extension, not a GPU."""
    from .. import ops
    if not ops.available():
        print("tools.plan --deterministic asks the native extension for its split counts: build it first "
              "(python build_native.py)")
        return 1
    from ..engine.native_engine import deterministic_plan, deterministic_workspace_elems
    spec = get_spec(model, num_classes)
    last = spec.fcs[-1]
    fused_head = len(spec.fcs) >= 2 and bool(ops.require().head_ce_supported(batch, last.fout, last.fin))
    rows = deterministic_plan(spec, batch, input_hw, sms, fused_head, freeze_layers)
    print("%s, %d classes, batch %d, %d x %d, %d SMs%s: workspace %.1f MB, %.1f MB of partial sums written and read "
          "per step" % (model, num_classes, batch, input_hw, input_hw, sms,
                        ", %d layers frozen" % freeze_layers if freeze_layers else "",
                        deterministic_workspace_elems(rows) * 4 / 1e6, sum(s * e for _, _, s, e in rows) * 4 / 1e6))
    print("%-16s %-6s %7s %12s %10s" % ("layer", "what", "splits", "slice elems", "MB"))
    for name, what, splits, elems in rows:
        print("%-16s %-6s %7d %12d %10.2f" % (name, what, splits, elems, splits * elems * 4 / 1e6))
    return 0


def powersgd_table(model: str, num_classes: int, rank: int, freeze_layers: int = 0) -> int:
    """Per trainable tensor (in DDP's bucket order): torch's n x m view, r' = min(n, m, r), whether
    PowerSGD compresses it, and the P + Q elements it exchanges; then the bytes of one update."""
    from ..parallel import powersgd
    spec = get_spec(model, num_classes)
    rows = powersgd.plan(spec, rank, freeze_layers)
    b = powersgd.exchange_bytes(rows)
    comp = [t for t in rows if t.compressed]
    print("%s, %d classes, PowerSGD rank %d: %d of %d tensors compressed (%d parameters), %d P + Q elements"
          % (model, num_classes, rank, len(comp), len(rows), sum(t.n * t.m for t in comp), sum(t.pq_elems for t in rows)))
    print("%3s %-24s %7s %8s %3s %-10s %9s" % ("#", "tensor", "n", "m", "r'", "exchange", "P + Q"))
    for j, t in enumerate(rows):
        print("%3d %-24s %7d %8d %3d %-10s %9d" % (j, t.name, t.n, t.m, t.rank,
                                                  "P, Q fp32" if t.compressed else "bf16 wire", t.pq_elems))
    print("bytes per update: %d of P + Q (fp32) + %d uncompressed (bf16) = %d (%.2f MB; %.2f MB without PowerSGD, "
          "%.0fx fewer)" % (b["compressed"], b["uncompressed"], b["total"], b["total"] / 1e6,
                            b["without_powersgd"] / 1e6, b["without_powersgd"] / b["total"]))
    return 0


def layerwise_table(model: str, num_classes: int, optimizer: str, sms: int, freeze_layers: int = 0,
                    powersgd_rank: int = 0, bucket_mb: float = 32.0) -> int:
    """The phase-1 / phase-2 launches of --optimizer lamb|lars over the buckets (parallel/layerwise.py)."""
    from ..parallel.layerwise import describe as lw_describe, engine_layerwise_plans
    spec = get_spec(model, num_classes)
    plans = engine_layerwise_plans(spec, sms, freeze_layers=freeze_layers, powersgd_rank=powersgd_rank,
                                   bucket_mb=bucket_mb)
    for compressed, lwp in plans.items():
        print("%s, %d classes, %d SMs%s%s:" % (model, num_classes, sms,
                                               ", %d layers frozen" % freeze_layers if freeze_layers else "",
                                               ", updates PowerSGD compresses" if compressed else ""))
        for line in lw_describe(lwp, optimizer):
            print(line)
    return 0


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--model", default="vggf")
    ap.add_argument("--num-classes", type=int, default=3)
    ap.add_argument("--world", type=int, default=8)
    ap.add_argument("--no-multicast", action="store_true", help="plan for a fabric without NVLS")
    ap.add_argument("--zero1", default="auto", choices=["auto", "on", "off"])
    ap.add_argument("--bucket-mb", type=float, default=32.0)
    ap.add_argument("--deterministic", action="store_true",
                    help="print the split-K launches of a --deterministic step and the workspace they need, instead")
    ap.add_argument("--batch", type=int, default=64, help="--deterministic: mini-batch per GPU")
    ap.add_argument("--input-hw", type=int, default=224, help="--deterministic: input side")
    ap.add_argument("--sms", type=int, default=132, help="--deterministic: SMs of the GPU planned for (H100 SXM: 132)")
    ap.add_argument("--freeze-layers", type=int, default=0,
                    help="plan for the first N layers frozen (the training option of the same name)")
    ap.add_argument("--powersgd-rank", type=int, default=0,
                    help="print which tensors PowerSGD at this rank compresses and the bytes per update, instead")
    ap.add_argument("--optimizer", default=None, choices=[None, "lamb", "lars"],
                    help="print the phase-1 / phase-2 launches of LAMB or LARS over the buckets (with --sms, "
                         "--freeze-layers and --powersgd-rank), instead")
    a = ap.parse_args(argv)
    try:
        get_spec(a.model, a.num_classes).check_freeze_layers(a.freeze_layers)
        if a.powersgd_rank:
            from ..parallel.powersgd import check_config
            check_config(a.powersgd_rank, 2)
    except ValueError as e:
        ap.error(str(e))
    if a.optimizer:
        return layerwise_table(a.model, a.num_classes, a.optimizer, a.sms, a.freeze_layers, a.powersgd_rank,
                               a.bucket_mb)
    if a.powersgd_rank:
        return powersgd_table(a.model, a.num_classes, a.powersgd_rank, a.freeze_layers)
    if a.deterministic:
        return deterministic(a.model, a.num_classes, a.batch, a.input_hw, a.sms, a.freeze_layers)
    plan, rows = describe(a.model, a.num_classes, a.world, not a.no_multicast, a.zero1, a.bucket_mb,
                          freeze_layers=a.freeze_layers)
    total = sum(r[2] for r in rows)
    print("%s, %d classes: %d elements (native layouts) in %d tensors, arena %d elements (tensors aligned to %d), %d buckets, %.1f MB of bf16 wire per step"
          % (a.model, a.num_classes, sum(plan.numels.values()), len(plan.order), plan.total, plan.align, len(rows), total / 1e6))
    for line in frozen_lines(a.model, a.num_classes, plan, a.freeze_layers):
        print(line)
    print("%3s %11s %9s %3s  %-24s %-24s %s" % ("#", "elements", "wire MB", "n", "first tensor", "last tensor (completes it)", "path at world=%d" % a.world))
    for i, n, wire, cnt, first, last, path in rows:
        print("%3d %11d %9.2f %3d  %-24s %-24s %s" % (i, n, wire / 1e6, cnt, first, last, path))
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
