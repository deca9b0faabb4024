"""NativeEngine: the whole training step on hand-written sm_90a kernels.

Where the reference's hot loop (distributedVggf.py:158-175) is ``model(inputs)`` ->
``cross_entropy`` -> ``zero_grad`` -> ``backward`` (DDP hooks all-reduce buckets) -> ``Adam.step``
-> two ``.item()`` syncs, all delegated to cuDNN / cuBLAS / c10d / ATen, this engine owns every
stage:

  input     fused augment kernel: uint8 HWC -> normalised bf16 im2col rows of the first conv
  forward   conv0 = wgmma GEMM on the im2col rows; conv1..12 = wgmma implicit GEMM (4-D TMA
            boxes, register accumulators, bias+ReLU epilogue); max-pool; FC stack = swap-AB split-K
            wgmma GEMMs + bias/ReLU/Philox-dropout epilogue; fused cross-entropy (+ metrics)
  backward  FC wgrad/dgrad GEMMs (MN-major operands, no transposed copies), conv dgrad with the
            ReLU mask fused in the epilogue, fused ReLU+pool backward, conv wgrad split-K with
            fp32 red.add straight into the flat gradient arena
  reduce    per bucket, as soon as its last gradient is enqueued: fused pack(fp32->bf16, 1/ws) +
            one-shot / two-shot / NVLS reduction over peer memory on a high-priority side stream
  update    fused Adam/SGD on the bucket right behind its reduction (reads the reduced bf16 wire,
            writes fp32 master + bf16 shadow, zeroes the gradient range)
Nothing synchronises with the host inside a step; loss / accuracy accumulate in a device meter.
"""
from __future__ import annotations

import contextlib
import math
import os

from typing import Dict, List, Optional, Tuple

import torch
import torch.distributed as dist

from .. import ops
from ..config import DATA, TRAIN
from ..data import transforms as T
from ..data.loader import FusedBatch, JpegBatch, RaggedBatch
from ..models import layout as L
from ..models.vggf import VGGSpec, build_oracle
from ..parallel import layerwise as lw
from ..parallel import powersgd as psgd
from ..parallel.buckets import Bucket, BucketPlan, engine_bucket_plan
from ..parallel.process_group import distributed_is_initialized
from ..utils.metrics import DeviceMeter
from ..utils.optim import LAYERWISE, check_layerwise_decay

BF16 = torch.bfloat16
F32 = torch.float32


def _round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


def _grown(buf: Optional[torch.Tensor], n: int, dtype: torch.dtype, device: torch.device) -> torch.Tensor:
    """``buf`` when it is a 1-D buffer of at least ``n`` elements, else a new one of ``n``: the input slots' buffers
    for batches of any image sizes grow to the largest batch the loader makes and then stay."""
    if buf is None or buf.dim() != 1 or buf.numel() < n:
        buf = torch.empty(n, dtype=dtype, device=device)
    return buf


def fc_ksplit(m_tiles: int, k_iters: int, target: int = 256) -> int:
    """Split-K factor the engine asks of a swap-AB FC GEMM (forward and dgrad)."""
    return max(1, min(k_iters, target // max(m_tiles, 1)))


def deterministic_plan(spec: VGGSpec, batch: int, input_hw: int, sms: int, fused_head: bool = True,
                       freeze_layers: int = 0) -> list:
    """The split-K launches of one deterministic training step, as [(layer, what, splits, elements per
    slice)]: what the workspace has to hold (``deterministic_workspace_elems``) and what ``tools.plan
    --deterministic`` prints.  The split counts are the launchers' own arithmetic (the extension's
    ``*_splits`` queries: pure host code), for ``sms`` SMs.  ``freeze_layers``: the frozen layers keep their
    forward launches only, and the first trainable layer has no dgrad."""
    C = ops.require()
    rows, fcs, convs = [], spec.fcs, spec.convs
    last = len(fcs) - 1
    k = spec.check_freeze_layers(freeze_layers)
    for i, f in enumerate(fcs):
        if i == last and fused_head:
            continue
        ks = fc_ksplit((f.fout + 127) // 128, (f.fin + 63) // 64)
        rows.append((f.name, "fprop", C.gemm_splits(f.fin, ks), C.workspace_slice(batch * f.fout)))
        if f.fout % 8 == 0 and len(convs) + i >= k:
            rows.append((f.name, "bias", C.colsum_partial_blocks(batch, f.fout, sms), f.fout))
        ks = fc_ksplit((f.fin + 127) // 128, (f.fout + 63) // 64)
        if ks > 1 and len(convs) + i > k:
            rows.append((f.name, "dgrad", C.gemm_splits(f.fout, ks), C.workspace_slice(batch * f.fin)))
    h = input_hw
    for i, c in enumerate(convs):
        if i < k:
            if c.pool_after:
                h //= 2
            continue
        rows.append((c.name, "bias", C.colsum_partial_blocks(batch * h * h, c.cout, sms), c.cout))
        if i == 0 and c.cout == 64:
            rows.append((c.name, "wgrad", C.conv0_wgrad_splits(batch, h, h, sms), 64 * 64))
        elif i == 0:
            M = batch * h * h
            rows.append((c.name, "wgrad", C.gemm_splits(M, max(1, min(M // 64, 296))),
                         C.workspace_slice(c.cout * L.CONV0_K)))
        else:
            rows.append((c.name, "wgrad", C.conv_wgrad_splits(batch, h, h, c.cin, c.cout, sms), c.cout * 9 * c.cin))
        if c.pool_after:
            h //= 2
    return rows


# Network input sizes the native engine runs: multiples of 8 keep every odd feature map (a crop that is not
# a multiple of 32, e.g. 176 -> 11 x 11 before the last pool) to the implicit-GEMM convolutions at <= 64 x 64,
# never the halo or first-layer kernels.
NATIVE_HW_MIN, NATIVE_HW_MAX, NATIVE_HW_STEP = 64, 512, 8


def check_native_hw(hw: int, what: str = "input_hw") -> int:
    """``hw`` if the native engine runs it, else ValueError naming the rule."""
    hw = int(hw)
    if not (NATIVE_HW_MIN <= hw <= NATIVE_HW_MAX and hw % NATIVE_HW_STEP == 0):
        raise ValueError("%s = %d: the native engine takes crops that are multiples of %d from %d to %d"
                         % (what, hw, NATIVE_HW_STEP, NATIVE_HW_MIN, NATIVE_HW_MAX))
    return hw


def deterministic_workspace_elems(plan: list) -> int:
    return max(splits * elems for _, _, splits, elems in plan)


class PhaseTimer:
    """CUDA-event timers around the phases of a step (``--profile events``)."""

    def __init__(self, enabled: bool, nvtx: bool = False) -> None:
        self.enabled = enabled
        self.nvtx = nvtx
        self.pending: List[Tuple[str, torch.cuda.Event, torch.cuda.Event]] = []
        self.totals: Dict[str, float] = {}
        self.counts: Dict[str, int] = {}
        self._open: Dict[str, torch.cuda.Event] = {}

    def start(self, name: str) -> None:
        if self.nvtx:
            torch.cuda.nvtx.range_push(name)
        if self.enabled:
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            self._open[name] = e

    def stop(self, name: str) -> None:
        if self.nvtx:
            torch.cuda.nvtx.range_pop()
        if self.enabled and name in self._open:
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            self.pending.append((name, self._open.pop(name), e))

    def collect(self) -> Dict[str, float]:
        for name, a, b in self.pending:
            b.synchronize()
            self.totals[name] = self.totals.get(name, 0.0) + a.elapsed_time(b)
            self.counts[name] = self.counts.get(name, 0) + 1
        self.pending.clear()
        return {k: self.totals[k] / max(self.counts[k], 1) for k in self.totals}


def check_native_spec(spec: VGGSpec) -> None:
    """ValueError unless the native kernels run every convolution of ``spec``."""
    for c in spec.convs[1:]:
        if c.cin % 64 or c.cout % 64:
            raise ValueError("native conv kernels need channel counts that are multiples of 64")
    if spec.convs[0].cout % 64 or spec.convs[0].cin != 3:
        raise ValueError("first conv must be 3 -> multiple of 64 channels")


class NativeEngine:
    # --val-tta (set_val_tta): the views of every evaluation pass, and their [B][C] fp32 probability accumulator
    val_tta, tta_acc = "none", None

    def __init__(self, spec: VGGSpec, device: torch.device, batch: int, lr: float = TRAIN.learning_rate,
                 optimizer: str = "adam", momentum: float = TRAIN.momentum, weight_decay: float = 0.0,
                 compute_dtype: str = "bf16", allreduce: str = "auto", wire_dtype: str = "bf16",
                 bucket_mb: float = 32.0, seed: int = 0, pretrained_state: Optional[dict] = None,
                 profile: Optional[str] = None, input_hw: int = DATA.crop, eval_hw: Optional[int] = None,
                 comm_ctas: int = 48,
                 init_state: Optional[Dict[str, torch.Tensor]] = None, unpack_fp32: bool = False,
                 distributed: bool = True, zero1="auto", conv_bucket_mb: float = 9.5,
                 tail_bucket_kb: float = 2400.0, same_dropout_all_ranks: bool = False,
                 label_smoothing: float = 0.0, ema_decay: Optional[float] = None,
                 bias_weight_decay: Optional[float] = None, deterministic: bool = False,
                 freeze_layers: int = 0, powersgd_rank: int = 0,
                 powersgd_start_iter: int = psgd.DEFAULT_START_ITER) -> None:
        ops.require()
        if compute_dtype != "bf16":
            raise NotImplementedError("the native engine computes in bf16 with fp32 master weights; "
                                      "use --engine oracle for fp32 numerics")
        check_native_spec(spec)
        self.spec, self.device, self.B = spec, torch.device(device), int(batch)
        if optimizer not in ("adam", "adamw", "sgd", "lamb", "lars"):
            raise ValueError("optimizer must be adam, adamw, sgd, lamb or lars (got %r)" % optimizer)
        for what, wd in (("weight_decay", weight_decay), ("bias_weight_decay", bias_weight_decay)):
            if wd is not None and not wd >= 0.0:
                raise ValueError("%s must be >= 0 (got %r)" % (what, wd))
        check_layerwise_decay(optimizer, weight_decay)
        self.lr, self.opt_name, self.momentum, self.weight_decay = lr, optimizer, momentum, weight_decay
        # torchvision's --bias-weight-decay: the biases' own decay (None: the biases take weight_decay)
        self.bias_weight_decay = bias_weight_decay
        self.beta1, self.beta2, self.eps = TRAIN.adam_beta1, TRAIN.adam_beta2, TRAIN.adam_eps
        # HW: the network input of training passes; eval_hw: of eval_step / forward_logits (FixRes: train at
        # a smaller crop than the one evaluated).  AdaptiveAvgPool2d((7, 7)) makes every weight size-free.
        self.seed, self.HW = int(seed), check_native_hw(input_hw, "input_hw")
        self.eval_hw = self.HW if eval_hw is None else check_native_hw(eval_hw, "eval_hw")
        if not 0.0 <= label_smoothing < 1.0:
            raise ValueError("label_smoothing must lie in [0, 1) (got %r)" % label_smoothing)
        # training loss only: F.cross_entropy(label_smoothing=); the evaluation loss stays plain
        self.label_smoothing = float(label_smoothing)
        self._mix = None                 # MixUp / CutMix draw of the staged batch (data.transforms.MixDraw)
        if ema_decay is not None and not 0.0 <= ema_decay <= 1.0:
            raise ValueError("ema_decay must lie in [0, 1] (got %r)" % ema_decay)
        # moving average of the weights (torchvision's --model-ema): ema = d * ema + (1 - d) * p, updated by
        # the optimizer kernels of the steps that ask for it (train_step(ema=True)); None: no EMA at all
        self.ema_decay = None if ema_decay is None else float(ema_decay)
        self.ema_updates = 0             # AveragedModel's n_averaged
        self._ema_step = False           # per train_step: this step's optimizer launches update the EMA
        self.same_dropout_all_ranks = bool(same_dropout_all_ranks)
        self.step_count = 0              # optimizer updates (Adam / SGD step, LR schedule, checkpoint "step")
        self.micro_count = 0             # training micro-batches: the Philox dropout offset
        self._accum = 0                  # micro-batches whose gradients sit in g32 awaiting an update
        self._update = self._wire_direct = True      # per train_step: see train_step
        self.train_dropout = True        # tests switch dropout off to compare gradients exactly
        self.apply_updates = True        # False: leave raw gradients in g32 (gradient inspection)
        self.meter: Optional[DeviceMeter] = None
        self.class_weights: Optional[torch.Tensor] = None
        self.teacher: Optional["TeacherEngine"] = None       # knowledge distillation (set_distillation)
        self.timer = PhaseTimer(profile == "events", nvtx=(profile == "nvtx"))
        self._comm_events: Optional[list] = None     # [(start, end, wire bytes)] while comm timing is on
        self._tl: Optional[list] = None              # step timeline marks (timeline())
        self.nvtx = profile == "nvtx"
        self.world = dist.get_world_size() if (distributed and distributed_is_initialized()) else 1
        self.rank = dist.get_rank() if (distributed and distributed_is_initialized()) else 0
        # Same inputs, same bits: every split-K and column sum stores per-split partials into one workspace
        # and adds them in split order (DESIGN 2.9) instead of letting fp32 atomics arrive in any order.
        self.deterministic = bool(deterministic)
        self._ws: Optional[torch.Tensor] = None      # the split-K workspace, allocated by _build_buffers
        if self.deterministic and allreduce == "nvls":
            raise ValueError("--deterministic: --allreduce nvls leaves the summation order to the NVLink switch; "
                             "use auto, oneshot or twoshot (they add the ranks in a fixed order)")
        # --powersgd-rank: from update powersgd_start_iter + 1 on, the tensors torch's powerSGD_hook compresses
        # are exchanged as rank-r factors P and Q (DESIGN 3.1); 0: off, and nothing below changes
        psgd.check_config(powersgd_rank, powersgd_start_iter)
        self.powersgd_rank, self.powersgd_start_iter = int(powersgd_rank), int(powersgd_start_iter)
        psgd.check_deterministic(self.powersgd_rank, self.deterministic, self.world)
        zero1 = psgd.resolve_zero1(zero1, self.powersgd_rank)
        self.ar_algo, self.comm_ctas, self.unpack_fp32 = allreduce, comm_ctas, unpack_fp32
        self.use_nccl = allreduce == "nccl"
        dev = self.device

        # --freeze-layers: the first ``freeze_layers`` entries of the layer table (convs, then fcs) keep
        # their weights, as torch with requires_grad_(False): forward as usual, no gradient, no exchange,
        # no optimizer state; the EMA still averages them (_frozen_ema)
        self.freeze_layers = spec.check_freeze_layers(freeze_layers)
        self._frozen = set(spec.frozen_param_names(self.freeze_layers))

        # ---- flat arenas (gradient-ready order) --------------------------------------------------
        # FC weights (ready first, 88 % of the bytes): ``bucket_mb`` messages.  Convolution gradients
        # (ready one layer at a time over the rest of backward): one bucket per big layer, and a small
        # final bucket -- its reduction and update are the only exposed part of the exchange.
        # Frozen layers come last in ready order: the buckets, g32, the moments and the wire cover the
        # trainable prefix [0, n_grad) alone; p32, w16 and the EMA span every tensor.
        ready = L.ready_order(spec)
        self.plan: BucketPlan = engine_bucket_plan(ready, bucket_mb, conv_bucket_mb, tail_bucket_kb,
                                                   trainable=len(ready) - len(self._frozen))
        n, ng = self.plan.total, self.plan.grad_total
        self.n_grad = ng
        self.p32 = torch.zeros(n, dtype=F32, device=dev)
        self.g32 = torch.zeros(ng, dtype=F32, device=dev)
        self.m32 = torch.zeros(ng, dtype=F32, device=dev)
        self.v32 = torch.zeros(ng, dtype=F32, device=dev) if optimizer in ("adam", "adamw", "lamb") else None
        # each bucket's weight-decay segments [(start within the bucket, decay), ...], one entry when the
        # decay is uniform: biases and weights share buckets, and one launch per bucket stays one launch
        self._wd_segments = {bk.start: self.decay_segments(bk) for bk in self.plan.buckets}
        self.w16 = torch.zeros(n, dtype=BF16, device=dev)

        if init_state is None:
            init_state = build_oracle(spec, seed=seed, pretrained_state=pretrained_state).state_dict()
        self.import_state(init_state, sync=False)

        # ---- cross-GPU plumbing ------------------------------------------------------------------
        self.arena = None
        self.cross_group = None          # inter-node stage of the hierarchical reduction
        self.comm_mode = "single" if self.world == 1 else ("nccl" if self.use_nccl else "flat")
        # high priority by default: a ready bucket should start reducing at once.  B200_COMM_PRIORITY=0
        # lets the comm / optimizer CTAs yield to the conv kernels instead (DESIGN 2.3 item 6).
        self.comm_stream = torch.cuda.Stream(device=dev, priority=int(os.environ.get("B200_COMM_PRIORITY", "-1")))
        # Second side stream for the optimizer: the reduction of bucket k+1 (NVLink-bound) runs while
        # bucket k is being updated (HBM-bound).  On ONE stream the two add up, and 24 x
        # (all-reduce + Adam) of serial work can outlast backward, so that the comm stream, not the
        # convolutions, ends the step.
        self.opt_stream = torch.cuda.Stream(device=dev, priority=int(os.environ.get("B200_COMM_PRIORITY", "-1"))) \
            if os.environ.get("B200_SPLIT_COMM", "1") == "1" else self.comm_stream
        if self.world > 1 and not self.use_nccl:
            from ..parallel import topology
            from ..parallel.symm import SymmetricArena

            layout = topology.detect_layout()
            self.comm_mode = layout.mode()
            if self.comm_mode == "flat" and os.environ.get("B200_FORCE_HIERARCHICAL", "0") == "1":
                self.comm_mode = "hierarchical"          # test hook: one node, both stages exercised
            node_group = None
            if self.comm_mode == "hierarchical":
                node_group, self.cross_group = topology.make_hierarchy_groups(layout)
            if self.comm_mode == "nccl":
                # one GPU per host (the reference's deployment) or uneven hosts: no peer memory to fuse over
                self.use_nccl = True
                if self.rank == 0:
                    print(f"[b200] {layout.n_nodes} hosts x {layout.local_size} GPU: gradient all-reduce "
                          f"falls back to NCCL (--allreduce {allreduce} needs an NVLink domain)", flush=True)
            else:
                wdt = BF16 if wire_dtype == "bf16" else F32
                self.arena = SymmetricArena(ng, dev, wire_dtype=wdt, group=node_group)
        if self.world > 1:
            self._broadcast_params()
        # buckets holding only FC weight gradients are written with plain stores by the wgrad GEMM:
        # the optimizer does not need to re-zero them (conv / bias gradients accumulate with red.add)
        fc_w = {f.name + ".weight" for f in spec.fcs}
        self._bucket_store_only = [all(t in fc_w for t in bk.tensors) for bk in self.plan.buckets]
        # FC weights that span whole buckets by themselves can be produced directly as bf16 on the wire
        # (when the updating micro-batch is also the first of its accumulation group: see _wire_direct);
        # those buckets are also the ones ZeRO-1 may shard
        self._prepacked = set()
        self._bucket_prepacked = [False] * len(self.plan.buckets)
        if self.arena is not None and self.arena.wire_dtype == BF16:
            for f in spec.fcs:
                name = f.name + ".weight"
                ids = self.plan.bucket_of(name)
                if ids and all(self.plan.buckets[i].tensors == (name,) for i in ids):
                    self._prepacked.add(name)
                    for i in ids:
                        self._bucket_prepacked[i] = True

        # EXPERIMENTAL (--zero1): buckets that take a reduce-scatter algorithm run reduce-scatter +
        # Adam on the owned cells + all-gather of the new bf16 weights as ONE kernel; the fp32 master
        # and moments of a cell are then only current on its owner (prepare_export gathers them).
        # zero1: True / False, or "auto" = on from 4 ranks up (at 8 ranks it shortened the step on the
        # GPU this was first tuned on; at 2 ranks every rank still owns half of the optimizer
        # state and the fused kernel's thin CTAs are slower than all-reduce + replicated Adam).
        z1_ok = self.arena is not None and self.arena.wire_dtype == BF16 and self.cross_group is None \
            and optimizer in ("adam", "adamw")
        if zero1 == "auto":
            zero1 = z1_ok and self.world >= 4
        self.zero1 = bool(zero1) and z1_ok
        if zero1 and not self.zero1 and self.world > 1:
            raise ValueError("--zero1 needs Adam or AdamW, the bf16 wire and all ranks in one NVLink domain")
        self._zero1_buckets: set = set()
        # the fused ZeRO-1 kernel keeps less in flight per CTA (128 threads, one switch reduction +
        # 96 bytes of optimizer state each): more, equally thin, CTAs
        self.zero1_ctas = int(os.environ.get("B200_ZERO1_CTAS", "128"))

        # EMA arenas: fp32 at p32's offsets (kept by the optimizer kernels) and its bf16 cast, made by
        # prepare_ema() for an evaluation pass (w16 cannot hold it: under ZeRO-1 w16 is rebuilt only by
        # the all-gather of the training step).  The average starts as the weights, like AveragedModel.
        self.ema32 = self.p32.clone() if self.ema_decay is not None else None
        self.ema16 = torch.zeros(n, dtype=BF16, device=dev) if self.ema_decay is not None else None
        self._ema16_current = False
        # arenas the forward pass reads weights (bf16) and biases (fp32) from; eval passes over the EMA swap them
        self._wsrc, self._bsrc = self.w16, self.p32

        self._build_buffers()
        self._psgd_now = False           # per train_step: this update compresses (update index > start iter)
        if self.powersgd_rank:
            self._powersgd_setup(ready, bucket_mb, conv_bucket_mb, tail_bucket_kb, wire_dtype)
        self._layerwise_setup()

    # ============================================================================ LAMB / LARS
    def layerwise_plans(self) -> Dict[bool, "lw.LayerwisePlan"]:
        """The phase-1 / phase-2 launch plans of --optimizer lamb|lars (parallel/layerwise.py), keyed by whether
        the update compresses with PowerSGD: the plain buckets, and the buckets without the compressed tensors
        plus one unit per compressed tensor."""
        sms = ops.require().sm_count()
        plans = {False: lw.layerwise_plan(self.plan, self.decay_of, sms)}
        if self.powersgd_rank:
            plan2 = self._psgd_tables[1][0]
            plans[True] = lw.layerwise_plan(plan2, self.decay_of, sms, lw.update_units(plan2, list(self._psgd)))
        return plans

    def _layerwise_setup(self) -> None:
        """LAMB / LARS only: the launch plans, the partial-sum workspace (a pair of fp32 per slot, one slot per
        phase-1 CTA) and the per-tensor trust ratios of the last update."""
        self.layerwise = self.opt_name in LAYERWISE
        if not self.layerwise:
            return
        self._lw_plans = self.layerwise_plans()
        self._lw_ws = torch.zeros(max(p.workspace_elems() for p in self._lw_plans.values()), dtype=F32,
                                  device=self.device)
        self.trust_ratio = torch.ones(len(self._lw_plans[False].tensors), dtype=F32, device=self.device)

    def _layerwise_update(self, s: int, e: int, g16: Optional[torch.Tensor], zero: bool, grad_scale: float) -> None:
        """The update of unit [s, e) under LAMB / LARS: its phase-1 launches, then the phase-2 launches of the
        tensors whose last piece it holds.  Both on the caller's stream, after the unit's reduction."""
        plan = self._lw_plans[self._psgd_now]
        lamb, kind = self.opt_name == "lamb", self.opt_name
        if lamb:
            hyper = dict(beta1=TRAIN.lamb_beta1, beta2=TRAIN.lamb_beta2, eps=TRAIN.lamb_eps, step=self.step_count)
        else:
            hyper = dict(momentum=self.momentum, first=self.step_count == 1, trust_coeff=TRAIN.lars_trust_coeff,
                         trust_eps=TRAIN.lars_eps)
        for L in plan.phase1[s]:
            a, b = L.start, L.end
            grad = dict(g16=g16[a - s:b - s]) if g16 is not None else dict(g32=self.g32[a:b])
            ops.layerwise_step(1, kind, self.p32[a:b], self.m32[a:b], self.v32[a:b] if lamb else None,
                               zero=self.g32[a:b] if (zero and lamb) else None, ws=self._lw_ws, lr=self.lr,
                               grad_scale=grad_scale, segments=L.segments, **grad, **hyper)
        for L in plan.phase2[s]:
            a, b = L.start, L.end
            # LARS reads the reduced gradient again (always fp32 in g32: see _reduce_and_update) and clears it
            grad = {} if lamb else dict(g32=self.g32[a:b], zero=self.g32[a:b])
            ops.layerwise_step(2, kind, self.p32[a:b], self.m32[a:b], self.v32[a:b] if lamb else None,
                               shadow=self.w16[a:b], ws=self._lw_ws, ratio=self.trust_ratio, lr=self.lr,
                               grad_scale=grad_scale, segments=L.segments, **grad, **hyper, **self._ema_kw(a, b))

    # ============================================================================== PowerSGD
    def _plan_tables(self) -> tuple:
        return (self.plan, self._wd_segments, self._bucket_store_only, self._bucket_prepacked, self._prepacked,
                self._tensor_buckets)

    def _set_plan_tables(self, tables: tuple) -> None:
        (self.plan, self._wd_segments, self._bucket_store_only, self._bucket_prepacked, self._prepacked,
         self._tensor_buckets) = tables

    def _powersgd_setup(self, ready, bucket_mb: float, conv_bucket_mb: float, tail_bucket_kb: float,
                        wire_dtype: str) -> None:
        """The second bucket plan (the compressed tensors in no bucket, every offset kept), the error arena over
        the compressed tensors, P and Q, and the back-projection workspace."""
        spec, dev = self.spec, self.device
        rows = psgd.plan(spec, self.powersgd_rank, self.freeze_layers)
        self._psgd_rows = rows
        comp = [t for t in rows if t.compressed]
        self._psgd: Dict[str, tuple] = {}
        eo = po = qo = 0
        for t in comp:
            n, m = psgd.native_nm(spec, t.name)
            if m % 4:
                raise ValueError("--powersgd-rank: %s has %d columns; the compression kernels need a multiple of 4"
                                 % (t.name, m))
            self._psgd[t.name] = (n, m, t.rank, eo, po, qo)
            eo += _round_up(n * m, 4)
            po += _round_up(n * t.rank, 4)
            qo += _round_up(m * t.rank, 4)
        self._psgd_e = torch.zeros(max(eo, 4), dtype=F32, device=dev)        # local error, M while compressing
        self._psgd_p = torch.zeros(max(po, 4), dtype=F32, device=dev)
        self._psgd_q = torch.zeros(max(qo, 4), dtype=F32, device=dev)
        self._psgd_ws = torch.empty(psgd.workspace_elems(rows, spec, ops.require().sm_count(), ops.require()),
                                    dtype=F32, device=dev)
        self._psgd_started = False       # e and Q start afresh at the first compressed update of this process
        # tables of the plain plan, then the same for the plan without the compressed tensors
        self._tensor_buckets = {n: self.plan.bucket_of(n) for n in self.plan.order}
        plain = self._plan_tables()
        plan2 = engine_bucket_plan(ready, bucket_mb, conv_bucket_mb, tail_bucket_kb,
                                   trainable=len(ready) - len(self._frozen), exclude=list(self._psgd))
        self.plan = plan2
        self._wd_segments = {bk.start: self.decay_segments(bk) for bk in plan2.buckets}
        for name in self._psgd:          # one optimizer launch per compressed tensor, over its aligned range
            s0 = plan2.offsets[name]
            bk = Bucket(-1, s0, s0 + _round_up(plan2.numels[name], plan2.align), (name,))
            self._wd_segments[s0] = self.decay_segments(bk)
        fc_w = {f.name + ".weight" for f in spec.fcs}
        self._bucket_store_only = [all(t in fc_w for t in bk.tensors) for bk in plan2.buckets]
        self._psgd_store_only = {name: name in fc_w for name in self._psgd}
        # the compressed FC wgrads go to g32 in fp32; the other FC weights that own whole buckets stay on the wire
        self._bucket_prepacked = [False] * len(plan2.buckets)
        self._prepacked = {n for n in self._prepacked if n not in self._psgd and
                           all(plan2.buckets[i].tensors == (n,) for i in plan2.bucket_of(n))}
        for name in self._prepacked:
            for i in plan2.bucket_of(name):
                self._bucket_prepacked[i] = True
        self._tensor_buckets = {n: plan2.bucket_of(n) for n in plan2.order}
        self._psgd_tables = (plain, self._plan_tables())
        self._set_plan_tables(plain)
        if self.rank == 0:
            print(psgd.summary_line(rows, self.powersgd_rank, 2 if wire_dtype == "bf16" else 4), flush=True)

    def _powersgd_begin(self, update_index: int) -> None:
        """Pick the bucket plan of this micro-batch's update; at the first compressed update, zero the error
        and load the hook's initial Q draws (permuted into the native column order)."""
        if not self.powersgd_rank:
            return
        self._psgd_now = update_index > self.powersgd_start_iter
        self._set_plan_tables(self._psgd_tables[1 if self._psgd_now else 0])
        if self._psgd_now and not self._psgd_started:
            self._psgd_e.zero_()
            for name, q in psgd.initial_q_torch(self._psgd_rows, self.seed).items():
                _, m, r, _, _, qo = self._psgd[name]
                self._psgd_q[qo:qo + m * r].copy_(psgd.q_to_native(self.spec, name, q).reshape(-1))
            self._psgd_started = True

    def _powersgd_update(self, name: str) -> None:
        """One compressed tensor, on the comm stream as soon as its gradient is final: project, all-reduce P,
        orthogonalise, back-project, all-reduce Q, decompress; then its optimizer launch."""
        n, m, r, eo, po, qo = self._psgd[name]
        s0 = self.plan.offsets[name]
        s1 = s0 + _round_up(self.plan.numels[name], self.plan.align)
        g, e = self.g32[s0:s0 + n * m], self._psgd_e[eo:eo + n * m]
        p, q = self._psgd_p[po:po + n * r], self._psgd_q[qo:qo + m * r]
        ev = torch.cuda.Event()
        ev.record()
        self.comm_stream.wait_event(ev)
        with torch.cuda.stream(self.comm_stream):
            self._mark("psgd %s start" % name, "comm")
            ops.psgd_orthogonalize(q, rows=m, rank=r)
            # g32 holds the sum of the group's k' micro-batch means: the hook sees their mean
            ops.psgd_project(g, e, q, p, n=n, m=m, rank=r, scale=1.0 / (self._accum + 1))
            if self.world > 1:
                dist.all_reduce(p)
            ops.psgd_orthogonalize(p, rows=n, rank=r)
            ops.psgd_backproject(e, p, q, self._psgd_ws, n=n, m=m, rank=r)
            if self.world > 1:
                dist.all_reduce(q)
            # q keeps the sum over ranks; torch's Q is q / W, and the next orthogonalisation removes the scale
            ops.psgd_decompress(p, q, g, e, n=n, m=m, rank=r, alpha=1.0 / self.world)
            self._mark("psgd %s end" % name, "comm")
        if not self.apply_updates:
            return
        if self.opt_stream is not self.comm_stream:
            done = torch.cuda.Event()
            done.record(self.comm_stream)
            self.opt_stream.wait_event(done)
        with torch.cuda.stream(self.opt_stream):
            self._apply_update(s0, s1, None, zero=not self._psgd_store_only[name])

    # ============================================================================ parameters
    def _view(self, arena: torch.Tensor, name: str) -> torch.Tensor:
        off = self.plan.offsets[name]
        return arena[off:off + self.plan.numels[name]].view(L.native_shape(self.spec, name))

    def import_state(self, state: Dict[str, torch.Tensor], sync: bool = True) -> None:
        """Load torch-layout tensors (checkpoint / oracle state dict) into the arenas."""
        with torch.no_grad():
            for name in self.spec.param_names:
                t = state[name].detach().to(self.device, F32)
                self._view(self.p32, name).copy_(L.to_native(self.spec, name, t))
            ops.require().cast_to_bf16(self.p32, self.w16)
        if sync and self.world > 1:
            self._broadcast_params()

    def prepare_export(self) -> None:
        """Collective.  Under --zero1 every rank holds the current fp32 master / moments (and EMA) only
        for the cells it owns: sum the owned pieces over ranks so that every rank has the full state again."""
        self._refuse_pending("prepare_export")
        self._gather_owned((self.p32, self.m32, self.v32) + ((self.ema32,) if self.ema32 is not None else ()))

    def _gather_owned(self, arenas) -> None:
        if not self._zero1_buckets:
            return
        self.sync()
        for arena in arenas:
            for bi in sorted(self._zero1_buckets):
                bk = self.plan.buckets[bi]
                tmp = torch.zeros(bk.end - bk.start, dtype=F32, device=self.device)
                for a, b in self.arena.owned_ranges(bk.start, bk.end - bk.start, self.zero1_ctas):
                    tmp[a - bk.start:b - bk.start] = arena[a:b]
                dist.all_reduce(tmp)
                arena[bk.start:bk.end] = tmp
        torch.cuda.synchronize(self.device)

    def prepare_ema(self) -> None:
        """Collective under --zero1.  Make the EMA readable by an evaluation pass: gather the owned EMA
        cells of the sharded buckets (as prepare_export does), then cast ema32 -> ema16."""
        self._require_ema("prepare_ema")
        self._refuse_pending("prepare_ema")
        self._gather_owned((self.ema32,))
        ops.require().cast_to_bf16(self.ema32, self.ema16)
        self._ema16_current = True

    def export_ema_state(self) -> Dict[str, torch.Tensor]:
        """The EMA in torch layout ({name: fp32 tensor}); under --zero1 call prepare_export first."""
        self._require_ema("export_ema_state")
        self._refuse_pending("export_ema_state")
        return {name: L.to_torch(self.spec, name, self._view(self.ema32, name)).detach().cpu()
                for name in self.spec.param_names}

    def import_ema_state(self, state: Dict[str, torch.Tensor], n_averaged: int) -> None:
        """Load a torch-layout EMA and its update count (AveragedModel's n_averaged)."""
        self._require_ema("import_ema_state")
        with torch.no_grad():
            for name in self.spec.param_names:
                t = state[name].detach().to(self.device, F32)
                self._view(self.ema32, name).copy_(L.to_native(self.spec, name, t))
        self.ema_updates = int(n_averaged)
        self._ema16_current = False

    def _require_ema(self, what: str) -> None:
        if self.ema32 is None:
            raise RuntimeError("%s: this engine keeps no EMA (construct it with ema_decay=)" % what)

    def _refuse_pending(self, what: str) -> None:
        if self._accum:
            raise RuntimeError("%s: %d accumulated micro-batch(es) await an update; finish the group with "
                               "train_step(batch, update=True) first" % (what, self._accum))

    def export_state(self) -> Dict[str, torch.Tensor]:
        self._refuse_pending("export_state")
        return {name: L.to_torch(self.spec, name, self._view(self.p32, name)).detach().cpu()
                for name in self.spec.param_names}

    def export_optimizer_state(self) -> dict:
        st = {"name": self.opt_name, "step": self.step_count, "micro_step": self.micro_count, "lr": self.lr}
        if getattr(self, "deterministic", False):     # key absent without the flag: the parent's checkpoint
            st["deterministic"] = True
        frozen = getattr(self, "freeze_layers", 0)
        if frozen:
            st["frozen_layers"] = frozen
        if getattr(self, "powersgd_rank", 0):      # the error and Q are per rank and not saved (as DDP's hook)
            st["powersgd"] = {"rank": self.powersgd_rank, "start_iter": self.powersgd_start_iter}
        # state for the trainable tensors only: torch keeps none for parameters without a gradient
        names = self.trainable_names()
        if self.opt_name in ("adam", "adamw", "lamb"):
            st["exp_avg"] = {n: L.to_torch(self.spec, n, self._view(self.m32, n)).cpu() for n in names}
            st["exp_avg_sq"] = {n: L.to_torch(self.spec, n, self._view(self.v32, n)).cpu() for n in names}
        else:
            st["momentum_buffer"] = {n: L.to_torch(self.spec, n, self._view(self.m32, n)).cpu() for n in names}
        return st

    def trainable_names(self) -> List[str]:
        """The parameters that train, in layer-table order (all of them without --freeze-layers)."""
        frozen = getattr(self, "_frozen", ())
        return [n for n in self.spec.param_names if n not in frozen]

    def import_optimizer_state(self, st: dict) -> None:
        # Per-parameter Adam step counts make "unfreeze and continue" a different optimizer: refuse it
        mine, theirs = getattr(self, "freeze_layers", 0), int(st.get("frozen_layers", 0))
        if "name" in st and theirs != mine:
            raise ValueError("the checkpoint's optimizer state was written with --freeze-layers %d, this run has "
                             "--freeze-layers %d: resume with %d (or evaluate it with --eval-only)"
                             % (theirs, mine, theirs))
        self.step_count = int(st.get("step", 0))
        if "name" in st and bool(st.get("deterministic", False)) != getattr(self, "deterministic", False):
            print("[Warn] the checkpoint was written %s --deterministic, this run is %s it: the run continues, "
                  "but not bit for bit as the one that wrote it would have" %
                  (("with", "without") if st.get("deterministic") else ("without", "with")), flush=True)
        self.micro_count = int(st.get("micro_step", self.step_count))    # one micro-batch per update before
        if "lr" in st:                       # a run resumed behind an LR-step boundary keeps the decayed rate
            self.lr = float(st["lr"])
        with torch.no_grad():
            for key, arena in (("exp_avg", self.m32), ("exp_avg_sq", self.v32), ("momentum_buffer", self.m32)):
                if key in st and arena is not None:
                    for n, t in st[key].items():
                        self._view(arena, n).copy_(L.to_native(self.spec, n, t.to(self.device, F32)))

    def set_lr(self, lr: float) -> None:
        self.lr = lr

    def decay_of(self, name: str) -> float:
        """The weight decay of parameter ``name``: bias_weight_decay for ``*.bias`` when it is set."""
        if name.endswith(".bias") and self.bias_weight_decay is not None:
            return float(self.bias_weight_decay)
        return float(self.weight_decay)

    def decay_segments(self, bk) -> list:
        """[(start within bucket ``bk``, weight decay), ...] with neighbours of equal decay merged.  Every
        tensor starts on an ``align``-element boundary of the arena, so the starts are whole float4s; the
        padding behind a tensor takes its decay (its weights and gradients stay zero)."""
        segs = []
        for name in sorted(bk.tensors, key=lambda t: self.plan.offsets[t]):
            start, wd = max(self.plan.offsets[name] - bk.start, 0), self.decay_of(name)
            if not segs or segs[-1][1] != wd:
                segs.append((start, wd))
        segs[0] = (0, segs[0][1])
        return segs

    def _update_ranges(self, s: int, e: int) -> list:
        """The optimizer launches of bucket [s, e): [(start, end, segment table relative to start)].  One
        launch unless the bucket has more decay segments than a launch takes (the test-sized models pack
        all their layers into a few buckets); VGG-F's buckets have at most ten."""
        segs, cap = self._wd_segments[s], ops.wd_max_segments()
        out = []
        for k in range(0, len(segs), cap):
            part = segs[k:k + cap]
            lo = part[0][0]
            hi = segs[k + cap][0] if k + cap < len(segs) else e - s
            out.append((s + lo, s + hi, [(a - lo, w) for a, w in part]))
        return out

    def _broadcast_params(self) -> None:
        """DDP's constructor sync (distributedVggf.py:225): everybody adopts rank 0's weights."""
        if self.arena is not None and self.cross_group is None:
            # the wire spans the trainable prefix only: the frozen range (up to all of VGG-F's 136 M weights for
            # a linear probe) goes as one collective instead of thousands of wire-sized chunks
            self.arena.broadcast_(self.p32[:self.n_grad], root=0)
            if self.n_grad < self.plan.total:
                dist.broadcast(self.p32[self.n_grad:], src=0)
        else:
            dist.broadcast(self.p32, src=0)
        ops.require().cast_to_bf16(self.p32, self.w16)
        torch.cuda.synchronize(self.device)

    # ============================================================================== buffers
    def _build_buffers(self, backward: bool = True) -> None:
        """Input staging, activations and the FC stack's buffers; with ``backward`` also the gradient buffers and,
        under --deterministic, a workspace for every split-K launch of a training step (else for the forward's)."""
        spec, B, dev, HW = self.spec, self.B, self.device, self.HW
        # double-buffered device-side input staging, filled by a copy stream
        self.copy_stream = torch.cuda.Stream(device=dev)
        self._in_slot = 0
        self._src_u8 = [None, None]
        self._params_dev = [torch.zeros(B, 8, dtype=F32, device=dev) for _ in range(2)]
        self._labels_dev = [torch.zeros(B, dtype=torch.int64, device=dev) for _ in range(2)]
        self._geom_dev = [torch.zeros(B, 5, dtype=torch.int64, device=dev) for _ in range(2)]   # RaggedBatch rows
        self._inter_u8 = None        # RaggedBatch: horizontally filtered rows, written and read on one stream
        # JpegBatch: coef, quant, raw and desc copied per slot on the copy stream (grown to the loader's slot
        # capacity, as _src_u8); the IDCT's sample planes are written and read on one stream
        self._jpeg_dev = [{} for _ in range(2)]
        self._planes_u8 = None
        self._in_free = [None, None]           # event: the step that used this slot is done with it
        self.labels_dev = self._labels_dev[0]
        # first conv: fused kernels build the im2col operand in shared memory from NHWC4 pixels
        # (csrc/include/conv0.cuh); the explicit im2col matrix only exists for other widths
        self.fused_conv0 = spec.convs[0].cout == 64
        # On by default (B200_FUSE_POOL=0 turns it off): the pooled layers' conv epilogue pools in
        # registers and records argmax / ReLU bit masks; the un-pooled activation is never written
        # (acts[i] of such a layer then holds stale data) and backward is an "unpool" kernel.
        want_fused_pool = os.environ.get("B200_FUSE_POOL", "1") == "1"
        cl = spec.convs[-1].cout
        ph = spec.pooled_hw
        assert spec.fcs[0].fin == cl * ph * ph, "classifier.0 must consume the pooled feature map"
        # The buffers of every size-dependent tensor hold the larger of the training and evaluation sizes;
        # each pass takes views at its own size (_set_hw).  An evaluation pass runs between training
        # steps, never between a step's forward and backward, so it may reuse them.
        shapes = {}
        for hw in sorted({self.HW, self.eval_hw}):
            g = dict(x_nhwc=(B, hw, hw, 4), acts=[], pools=[], masks=[])
            if not self.fused_conv0:
                g["col0"] = (B * hw * hw, L.CONV0_K)
            h = hw
            for i, c in enumerate(spec.convs):
                g["acts"].append((B, h, h, c.cout))
                fused = (want_fused_pool and c.pool_after and i > 0 and c.cout % 32 == 0
                         and bool(ops.require().conv_pool_fusable(B, h, h)))
                g["masks"].append(tuple(ops.pool_mask_like(B, h, h, c.cout, "meta").shape) if fused else None)
                if c.pool_after:
                    h //= 2
                g["pools"].append((B, h, h, c.cout) if c.pool_after else None)
            g["feat_hw"] = h
            shapes[hw] = g

        def arena(key, dtype, zero=False, i=None):
            """One buffer for slot ``key`` (layer ``i``), large enough for every size; {hw: view}."""
            want = {hw: (g[key] if i is None else g[key][i]) for hw, g in shapes.items()}
            n = max((math.prod(v) for v in want.values() if v is not None), default=0)
            if not n:
                return {hw: None for hw in want}
            buf = (torch.zeros if zero else torch.empty)(n, dtype=dtype, device=dev)
            return {hw: None if v is None else buf[:math.prod(v)].view(v) for hw, v in want.items()}

        col0 = arena("col0", BF16) if not self.fused_conv0 else {hw: None for hw in shapes}
        x_nhwc = arena("x_nhwc", BF16)
        acts, pools, masks = [], [], []
        for i in range(len(spec.convs)):
            acts.append(arena("acts", BF16, i=i))
            masks.append(arena("masks", torch.int32, zero=True, i=i))
            pools.append(arena("pools", BF16, i=i))
        avg = None
        if any(g["feat_hw"] != ph for g in shapes.values()):
            avg = torch.empty(B, ph, ph, cl, dtype=BF16, device=dev)
        self._geo = {hw: dict(x_nhwc=x_nhwc[hw], col0=col0[hw], acts=[a[hw] for a in acts],
                              pools=[p[hw] for p in pools], pool_masks=[m[hw] for m in masks],
                              feat_hw=g["feat_hw"], avg=None if g["feat_hw"] == ph else avg)
                     for hw, g in shapes.items()}
        self._hw = None
        self._set_hw(self.HW)
        # FC stack
        self.fc_acc = [torch.zeros(B, f.fout, dtype=F32, device=dev) for f in spec.fcs]
        self.fc_y = [torch.empty(B, f.fout, dtype=BF16, device=dev) if i < len(spec.fcs) - 1 else None
                     for i, f in enumerate(spec.fcs)]
        if backward:
            self.fc_dacc = [torch.zeros(B, f.fin, dtype=F32, device=dev) for f in spec.fcs]
            self.fc_dz = [torch.zeros(B, _round_up(f.fout, 8), dtype=BF16, device=dev) for f in spec.fcs]
        self.logits = torch.zeros(B, spec.num_classes, dtype=F32, device=dev)
        self.loss_buf = torch.zeros(1, dtype=F32, device=dev)
        self.scratch_meter = torch.zeros(4, dtype=F32, device=dev)
        # K-FUN2+CE: last Linear + cross-entropy + metrics + that layer's backward as ONE launch when the
        # head is small (the funnel: 512 -> C <= 8); VGG-16/1000 keeps the GEMM path.  B200_FUSED_HEAD=0: off.
        lastf = spec.fcs[-1]
        self.fused_head = (os.environ.get("B200_FUSED_HEAD", "1") == "1" and len(spec.fcs) >= 2
                           and bool(ops.require().head_ce_supported(B, lastf.fout, lastf.fin)))
        self._head_in = None
        if backward:
            # backward activations-gradients: two ping-pong buffers big enough for the largest map
            biggest = max(a.numel() for g in self._geo.values() for a in g["acts"])
            self.dbuf = [torch.empty(biggest, dtype=BF16, device=dev) for _ in range(2)]
            self.dfeat = torch.empty(B, ph, ph, cl, dtype=BF16, device=dev)
        if self.deterministic:
            # one workspace for every split-K launch of the step: they all run on the compute stream
            plan = deterministic_plan(spec, B, HW, ops.require().sm_count(), self.fused_head, self.freeze_layers)
            if not backward:
                plan = [row for row in plan if row[1] == "fprop"] or [(None, "fprop", 1, 4)]
            self._ws = torch.empty(deterministic_workspace_elems(plan), dtype=F32, device=dev)

    def _set_hw(self, hw: int) -> None:
        """Point the size-dependent buffers (input, activations, pools, pool masks, feature map) at the
        views of a pass at network input ``hw``."""
        if hw == self._hw:
            return
        g = self._geo[hw]
        self.x_nhwc, self.col0, self.acts, self.pools = g["x_nhwc"], g["col0"], g["acts"], g["pools"]
        self.pool_masks, self.feat_hw, self.avg = g["pool_masks"], g["feat_hw"], g["avg"]
        self._hw = hw

    # ================================================================================ inputs
    def _stage_input(self, batch, views=None) -> int:
        """Copy a batch to the device and produce the network input.  Returns b.  ``views`` (TTA view codes): the
        input of the first view; ``_view_input`` makes the others from the same staged copy."""
        j, HW = self._in_slot, self._hw
        self._in_slot ^= 1
        self.labels_dev = self._labels_dev[j]
        if isinstance(batch, (FusedBatch, RaggedBatch, JpegBatch)):
            b, mix = self._copy_to_slot(batch, j), batch.mix
        else:                            # the reference pipeline's (float batch, labels[, MixUp / CutMix draw])
            b, mix = int(batch[1].shape[0]), batch[2] if len(batch) > 2 else None
            x = self._staged_x = batch[0].to(self.device, F32, non_blocking=True).contiguous()
            if views is not None:        # the reference pipeline's views: [b][V][3][HW][HW]
                assert x.dim() == 5 and x.shape[1] == len(views), "the batch does not carry the evaluation's views"
                assert x.shape[3] == HW and x.shape[4] == HW, "input size differs from the evaluation size (eval_hw)"
            else:
                assert x.shape[2] == HW and x.shape[3] == HW, \
                    "input size differs from the pass's size (input_hw / eval_hw)"
            self.labels_dev[:b].copy_(batch[1], non_blocking=True)
        self._staged, self._mix = j, mix
        return self._view_input(batch, b, 0, views)

    def _copy_to_slot(self, batch, j: int) -> int:
        """Copy a loader batch to input slot ``j`` (and decode a JpegBatch into the slot's image buffer).  Returns b."""
        b, dev = int(batch.labels.shape[0]), self.device
        if isinstance(batch, FusedBatch):
            if self._src_u8[j] is None or self._src_u8[j].shape[1:] != batch.images_u8.shape[1:]:
                self._src_u8[j] = torch.empty((self.B, *batch.images_u8.shape[1:]), dtype=torch.uint8, device=dev)
            copies = [(self._src_u8[j][:b], batch.images_u8)]
        else:
            nbytes = batch.nbytes
            self._src_u8[j] = _grown(self._src_u8[j], nbytes, torch.uint8, dev)
            self._inter_u8 = _grown(self._inter_u8, ops.ragged_inter_bytes(batch.geom), torch.uint8, dev)
            if isinstance(batch, JpegBatch):
                jd, copies = self._jpeg_dev[j], []
                for name in ("coef", "quant", "raw", "desc"):
                    t = getattr(batch, name)
                    jd[name] = _grown(jd.get(name), max(t.numel(), 1), t.dtype, dev)
                    copies.append((jd[name][:t.numel()], t.view(-1)))
                self._planes_u8 = _grown(self._planes_u8, max(batch.coef.numel(), 1), torch.uint8, dev)
            else:
                copies = [(self._src_u8[j][:nbytes], batch.data_u8)]
            copies.append((self._geom_dev[j][:b], batch.geom))
        copies += [(self._params_dev[j][:b], batch.params), (self._labels_dev[j][:b], batch.labels)]
        with torch.cuda.stream(self.copy_stream):
            if self._in_free[j] is not None:
                self.copy_stream.wait_event(self._in_free[j])
            for dst, src in copies:
                dst.copy_(src, non_blocking=True)
            h2d = self.copy_stream.record_event()
        if batch.state is not None:
            batch.state["event"] = h2d          # the loader may refill the pinned slot after this
        torch.cuda.current_stream(dev).wait_event(h2d)
        if isinstance(batch, JpegBatch):
            ops.require().jpeg_decode(jd["coef"], jd["quant"][:batch.quant.numel()].view(-1, 64),
                                      jd["desc"][:batch.desc.numel()].view(b, -1), self._geom_dev[j][:b], jd["raw"],
                                      self._planes_u8, self._src_u8[j][:nbytes], batch.desc, batch.geom)
        return b

    def _view_input(self, batch, b: int, i: int, views) -> int:
        """The network input of the staged batch (with ``views``: of its view ``i``), and conv0's im2col rows if any."""
        C, HW, j, x = ops.require(), self._hw, self._staged, self.x_nhwc[:b]
        if isinstance(batch, FusedBatch):
            args = (self._src_u8[j][:b], self._params_dev[j][:b], x, batch.resized_hw)
            if views is None:        # MixUp / CutMix in the same pass (sample i with i-1 mod b)
                ops.augment(*args, out_hw=HW, mode="nhwc", pad=4, mix=self._mix)
            else:
                ops.augment_view(*args, views[i], out_hw=HW)
        elif isinstance(batch, (RaggedBatch, JpegBatch)):     # view 0 also runs the horizontal pass of every view
            args = (self._src_u8[j][:batch.nbytes], self._geom_dev[j][:b], self._params_dev[j][:b], self._inter_u8, x,
                    batch.geom, batch.params)
            if views is None:
                ops.augment_ragged(*args, out_hw=HW, mix=self._mix)
            else:
                ops.augment_ragged_view(*args, views[i], out_hw=HW, pass1=views if i == 0 else ())
        else:                            # the reference pipeline's float batch, or its view i
            C.nchw_to_nhwc(self._staged_x if views is None else self._staged_x[:, i].contiguous(), x)
        if not self.fused_conv0:         # a second pass expands the L2-resident NHWC4 pixels with 16-byte stores
            C.im2col_c3(x, self.col0[:b * HW * HW], L.CONV0_K)
        return b

    def _release_input(self) -> None:
        """The augment kernel and the loss have consumed the staged batch: its slot may be refilled."""
        ev = torch.cuda.Event()
        ev.record()
        self._in_free[self._in_slot ^ 1] = ev

    # =============================================================================== forward
    def _w(self, name: str) -> torch.Tensor:
        return self._view(self._wsrc, name + ".weight")

    def _b(self, name: str) -> torch.Tensor:
        return self._view(self._bsrc, name + ".bias")

    def _drop_key(self, layer: int) -> int:
        """Philox key of a dropout layer.  Every replica draws its OWN mask, like the reference's
        per-process RNG (distributedVggf.py:55; one process per rank) -- identical masks on all ranks
        would correlate the replicas' gradient noise.  ``same_dropout_all_ranks`` is for parity tests."""
        r = 0 if self.same_dropout_all_ranks else self.rank
        return self.seed * 1000003 + layer + 7919 * r

    _ksplit = staticmethod(fc_ksplit)

    def _forward(self, b: int, train: bool) -> None:
        C = ops.require()
        spec, HW = self.spec, self._hw
        c0 = spec.convs[0]
        M0 = b * HW * HW
        # conv0 (K = 27): im2col GEMM with fused bias + ReLU -> bf16 NHWC
        if self.fused_conv0:
            C.conv0_fprop(self.x_nhwc[:b], self._w(c0.name), self._b(c0.name), self.acts[0][:b])
        else:
            ops.gemm(self.col0[:M0], self._w(c0.name), self.acts[0][:b].view(M0, c0.cout), M=M0, N=c0.cout,
                     K=L.CONV0_K, epi="bf16_bias_relu", bias=self._b(c0.name))
        x = self.acts[0][:b]
        if c0.pool_after:
            x = ops.maxpool2x2(x, out=self.pools[0][:b])
        for i, c in enumerate(spec.convs[1:], start=1):
            if self.pool_masks[i] is not None:           # fused conv + ReLU + pool
                x, _ = ops.conv3x3_fprop_pool(x, self._w(c.name), self._b(c.name), out=self.pools[i][:b],
                                              mask=self.pool_masks[i][:b])
                self._mark("fwd " + c.name)
                continue
            y = self.acts[i][:b]
            C.conv_fprop(x, self._w(c.name), self._b(c.name), y, True, 0)
            x = y
            if c.pool_after:
                x = ops.maxpool2x2(y, out=self.pools[i][:b])
            self._mark("fwd " + c.name)
        if self.avg is not None:
            x = ops.adaptive_avgpool(x, spec.pooled_hw, spec.pooled_hw, out=self.avg[:b])
        self.feat = x
        h = x.reshape(b, -1)
        last = len(spec.fcs) - 1
        for i, f in enumerate(spec.fcs):
            if i == last and self.fused_head:
                self._head_in = h            # logits, loss and this layer's backward: _head()
                break
            m_tiles = (f.fout + 127) // 128
            ks = self._ksplit(m_tiles, (f.fin + 63) // 64)
            acc = self.fc_acc[i][:b]
            if self.deterministic:
                ops.gemm_det(self._w(f.name), h, acc, self._ws, M=f.fout, N=b, K=f.fin, transposed=True, ksplit=ks)
            else:
                ops.gemm(self._w(f.name), h, acc, M=f.fout, N=b, K=f.fin, epi="f32_atomic_t", ksplit=ks, ldo=f.fout)
            if i == last:
                ops.fc_bias_act(acc, self._b(f.name), None, self.logits[:b], B=b, N=f.fout, relu=False)
            else:
                p = f.dropout if (train and self.train_dropout) else 0.0
                ops.fc_bias_act(acc, self._b(f.name), self.fc_y[i][:b], None, B=b, N=f.fout, relu=f.relu,
                                drop_p=p, seed=self._drop_key(i), offset=self.micro_count)
                h = self.fc_y[i][:b]

    def _loss(self, b: int, train: bool) -> None:
        """Loss + metrics (+ dlogits when training) from the forward state."""
        meter = self.meter.buf if self.meter is not None else self.scratch_meter
        # soft targets (label smoothing, MixUp / CutMix) shape the training loss only
        eps, mix = (self.label_smoothing, self._mix) if train else (0.0, None)
        kd = train and self.teacher is not None
        if not self.fused_head:
            ld = self.fc_dz[-1].shape[1] if train else 0
            if kd:
                ops.cross_entropy_kd(self.logits[:b], self.labels_dev[:b], self._teacher_logits, alpha=self.distill_alpha,
                                     temperature=self.distill_temperature, dlogits=self.fc_dz[-1][:b], ldd=ld,
                                     meter=meter, loss_out=self.loss_buf, class_weights=self.class_weights,
                                     label_smoothing=eps, mix=mix)
                return
            ops.cross_entropy(self.logits[:b], self.labels_dev[:b], self.fc_dz[-1][:b] if train else None,
                              ld, meter, self.loss_buf,
                              class_weights=self.class_weights if train else None,   # like the reference's loops
                              label_smoothing=eps, mix=mix)
            return
        f, prev = self.spec.fcs[-1], self.spec.fcs[-2]
        C = ops.require()
        if train:
            p = prev.dropout if self.train_dropout else 0.0
            # linear probe (every layer before the head frozen): no gradient for the head's input
            dh = None if self.freeze_layers == self.spec.num_layers - 1 else self.fc_dz[-2][:b]
            args = (self._head_in, self._w(f.name), self._b(f.name), self.labels_dev[:b], self.logits[:b],
                    self.fc_dz[-1][:b], self.fc_dz[-1].shape[1], self._grad(f.name + ".weight"),
                    self._grad(f.name + ".bias"), dh, 1.0 / (1.0 - p), bool(prev.relu), meter,
                    self.loss_buf, self.class_weights)
            soft = ops.soft_targets(eps, mix)
            if kd:
                C.head_ce_kd(*args, bool(self._accum), soft, self._teacher_logits, self.distill_alpha,
                             self.distill_temperature)
            elif soft is not None:
                C.head_ce(*args, bool(self._accum), soft)
            elif self._accum:                # a later micro-batch of the group: dW += (db always accumulates)
                C.head_ce(*args, True)
            else:
                C.head_ce(*args)
        else:
            C.head_ce(self._head_in, self._w(f.name), self._b(f.name), self.labels_dev[:b], self.logits[:b],
                      None, 0, None, None, None, 1.0, False, meter, self.loss_buf, None)

    # ============================================================================== backward
    def _grad(self, name: str) -> torch.Tensor:
        return self._view(self.g32, name)

    def _bias_grad(self, dz2d: torch.Tensor, name: str, rows: int, C: int, ld: Optional[int] = None) -> None:
        """Bias gradient of layer ``name`` from its dz.  Deterministic: per-block column sums added in block
        order; a width the vector kernel does not take goes to the one-thread-per-channel kernel, which
        adds each element once per launch in row order (reproducible as it is)."""
        db = self._grad(name + ".bias")
        if self.deterministic and C % 8 == 0 and ld in (None, C):
            ops.colsum_det(dz2d, db, self._ws, rows, C, accumulate=True)     # db: zeroed by the optimizer
        else:
            ops.bias_grad(dz2d, db, rows, C, ld=ld)

    def _backward(self, b: int) -> None:
        C = ops.require()
        det, acc_g = self.deterministic, bool(self._accum)
        spec = self.spec
        fcs, convs = spec.fcs, spec.convs
        last = len(fcs) - 1
        # backward stops at the first trainable layer k (layer-table index): its bias gradient and wgrad
        # run, its dgrad does not, and nothing below it is launched
        k = self.freeze_layers
        # ---- FC stack ----------------------------------------------------------------------
        for i in range(last, -1, -1):
            f = fcs[i]
            if i == last and self.fused_head:     # produced by _loss(): gradients are already in the arena
                self._bucket_done(f.name + ".bias")
                self._bucket_done(f.name + ".weight")
                self._mark("bwd " + f.name)
                if k == len(convs) + i:
                    return
                continue
            ld = self.fc_dz[i].shape[1]
            dz = self.fc_dz[i][:b]                                   # [b][ld] bf16, cols >= fout are 0
            x_in = self.fc_y[i - 1][:b] if i > 0 else self.feat.reshape(b, -1)
            self._bias_grad(dz, f.name, b, f.fout, ld=ld)
            self._bucket_done(f.name + ".bias")
            # wgrad: dW[fout][fin] = dz^T x_in   (both operands MN-major: stored [K=b][*])
            if self._wire_direct and (f.name + ".weight") in self._prepacked:
                # big FC weights own whole buckets: write bf16(dW / ws) straight into the symmetric
                # wire buffer -- no fp32 gradient, no pack pass before the reduction
                off = self.plan.offsets[f.name + ".weight"]
                wire_w = self.arena.wire[off:off + f.fout * f.fin].view(f.fout, f.fin)
                ops.gemm(dz, x_in, wire_w, M=f.fout, N=f.fin, K=b, a_mn=True, b_mn=True, epi="bf16_store",
                         ldo=f.fin, alpha=1.0 / self.world)
            else:
                # the first micro-batch of a group stores, later ones add (ksplit 1: each tile owns its
                # elements, so the red.add epilogue adds every element exactly once -- which is why the FC
                # wgrads, this one and the bf16 one above, are the same launches under `deterministic`)
                ops.gemm(dz, x_in, self._grad(f.name + ".weight"), M=f.fout, N=f.fin, K=b, a_mn=True,
                         b_mn=True, epi="f32_atomic" if self._accum else "f32_store", ldo=f.fin)
            if k == len(convs) + i:              # the first trainable layer: its input needs no gradient
                self._bucket_done(f.name + ".weight")
                self._mark("bwd " + f.name)
                return
            # dgrad: dX[b][fin] = dz W ; swap-AB with W read MN-major (stored [K=fout][M=fin])
            m_tiles = (f.fin + 127) // 128
            ks = self._ksplit(m_tiles, (f.fout + 63) // 64)
            dacc = self.fc_dacc[i][:b]
            if det and ks > 1:
                ops.gemm_det(self._w(f.name), dz, dacc, self._ws, M=f.fin, N=b, K=f.fout, a_mn=True, transposed=True,
                             ksplit=ks)
            else:
                ops.gemm(self._w(f.name), dz, dacc, M=f.fin, N=b, K=f.fout, a_mn=True,
                         epi="f32_atomic_t" if ks > 1 else "f32_store_t", ksplit=ks, ldo=f.fin)
            # only now may the optimizer touch W_i: the dgrad above still reads the old weights
            self._bucket_done(f.name + ".weight")
            if i > 0:
                prev = fcs[i - 1]
                ops.fc_grad_act(dacc, self.fc_y[i - 1][:b], self.fc_dz[i - 1][:b], B=b, N=f.fin,
                                relu=prev.relu, drop_p=prev.dropout if self.train_dropout else 0.0)
            else:
                ops.fc_grad_act(dacc, None, self.dfeat[:b].view(b, -1), B=b, N=f.fin, relu=False)
            self._mark("bwd " + f.name)
        # ---- feature map gradient ------------------------------------------------------------
        g = self.dfeat[:b]
        if self.avg is not None:
            g = ops.adaptive_avgpool_bwd(g, self.feat_hw, self.feat_hw,
                                         out=self.dbuf[1][:b * self.feat_hw ** 2 * convs[-1].cout]
                                         .view(b, self.feat_hw, self.feat_hw, convs[-1].cout))
        # ---- conv stack ----------------------------------------------------------------------
        # invariant at loop entry: if layer i pools, `g` is dP_i (grad wrt pooled output);
        # otherwise `g` is dZ_i (grad wrt the pre-ReLU output, mask already applied).
        pp = 0
        bias_fused = False      # was this layer's bias gradient already produced by the kernel that made dz?
        for i in range(len(convs) - 1, -1, -1):
            c = convs[i]
            y = self.acts[i][:b]
            if c.pool_after:
                dz = self.dbuf[pp][:y.numel()].view_as(y)
                # ReLU + pool backward, bias gradient (column sum of dz) fused
                # (deterministic: no fused column sum, its atomics arrive in any order; _bias_grad below)
                colsum = None if det else self._grad(c.name + ".bias")
                if self.pool_masks[i] is not None:
                    ops.unpool2x2(g, self.pool_masks[i][:b], out=dz, colsum=colsum)
                else:
                    ops.maxpool2x2_relu_bwd(y, g, out=dz, colsum=colsum)
                pp ^= 1
                bias_fused = not det
            else:
                dz = g
            M = y.numel() // c.cout
            if not bias_fused:
                self._bias_grad(dz.view(M, c.cout), c.name, M, c.cout)
            self._bucket_done(c.name + ".bias")
            if i == 0:
                if self.fused_conv0 and det:
                    ops.conv0_wgrad_det(dz, self.x_nhwc[:b], self._grad(c.name + ".weight"), self._ws, accumulate=acc_g)
                elif self.fused_conv0:
                    C.conv0_wgrad(dz, self.x_nhwc[:b], self._grad(c.name + ".weight"))
                elif det:
                    ops.gemm_det(dz.view(M, c.cout), self.col0[:M], self._grad(c.name + ".weight"), self._ws, M=c.cout,
                                 N=L.CONV0_K, K=M, a_mn=True, b_mn=True, ksplit=max(1, min(M // 64, 296)),
                                 accumulate=acc_g)
                else:
                    ks = max(1, min(M // 64, 296))
                    ops.gemm(dz.view(M, c.cout), self.col0[:M], self._grad(c.name + ".weight"), M=c.cout,
                             N=L.CONV0_K, K=M, a_mn=True, b_mn=True, epi="f32_atomic", ksplit=ks, ldo=L.CONV0_K)
                self._bucket_done(c.name + ".weight")
                self._mark("bwd " + c.name)
                break
            prev = convs[i - 1]
            x_in = self.pools[i - 1][:b] if prev.pool_after else self.acts[i - 1][:b]
            if det:
                ops.conv3x3_wgrad_det(dz, x_in, self._grad(c.name + ".weight"), self._ws, accumulate=acc_g)
            else:
                C.conv_wgrad(dz, x_in, self._grad(c.name + ".weight"), 1.0, 0, 0)
            if i == k:                            # the first trainable layer: no dgrad, layer i-1 is frozen
                self._bucket_done(c.name + ".weight")
                self._mark("bwd " + c.name)
                break
            dx = self.dbuf[pp][:x_in.numel()].view_as(x_in)
            # ReLU backward of layer i-1 is fused here unless a pool sits in between; when it is,
            # dx IS dZ_{i-1} and its column sum (layer i-1's bias gradient) comes for free
            fuse = not prev.pool_after
            C.conv_dgrad(dz, self._w(c.name), x_in if fuse else None, dx,
                         self._grad(prev.name + ".bias") if fuse and not det else None, 0)
            bias_fused = fuse and not det
            self._bucket_done(c.name + ".weight")      # after dgrad: it reads the pre-update weights
            self._mark("bwd " + c.name)
            pp ^= 1
            g = dx

    # ================================================================= all-reduce + optimizer
    def _begin_step(self) -> None:
        self._missing = [len(bk.tensors) for bk in self.plan.buckets]
        self._tensor_buckets = getattr(self, "_tensor_buckets", None) or \
            {n: self.plan.bucket_of(n) for n in self.plan.order}

    def _bucket_done(self, name: str) -> None:
        """Called right after the kernels producing ``name``'s gradient were enqueued."""
        if self._psgd_now and self._update and name in self._psgd:
            self._powersgd_update(name)
            return
        for bi in self._tensor_buckets[name]:
            self._missing[bi] -= 1
            if self._missing[bi] == 0 and self._update:
                self._reduce_and_update(bi)

    def _frozen_ema(self) -> None:
        """On an EMA step, the moving average of the frozen range [n_grad, total), which no optimizer launch
        covers (AveragedModel averages every parameter): one launch on the optimizer's side stream, under
        backward.  The frozen weights never change, so it may run anywhere in the step."""
        if not self._ema_step or self.n_grad == self.plan.total:
            return
        ev = torch.cuda.Event()
        ev.record()                      # an evaluation pass may still read the EMA biases
        self.opt_stream.wait_event(ev)
        with torch.cuda.stream(self.opt_stream):
            ops.ema_update(self.p32[self.n_grad:], self.ema32[self.n_grad:], decay=self.ema_decay,
                           first=self.ema_updates == 0)

    def _ema_kw(self, s: int, e: int) -> dict:
        """The EMA arguments of an optimizer launch over [s, e): none unless this step updates the EMA."""
        if not self._ema_step:
            return {}
        return dict(ema=self.ema32[s:e], ema_decay=self.ema_decay, ema_first=self.ema_updates == 0)

    def _apply_update(self, s: int, e: int, g16: Optional[torch.Tensor], zero: bool = True,
                      grad_scale: float = 1.0) -> None:
        if getattr(self, "layerwise", False):
            self._layerwise_update(s, e, g16, zero, grad_scale)
            return
        ranges = self._update_ranges(s, e)
        if len(ranges) == 1:
            self._launch_update(s, e, g16, zero, grad_scale, ranges[0][2])
            return
        for a, b, segs in ranges:
            self._launch_update(a, b, None if g16 is None else g16[a - s:b - s], zero, grad_scale, segs)

    def _launch_update(self, s: int, e: int, g16: Optional[torch.Tensor], zero: bool, grad_scale: float,
                       segs: list) -> None:
        g32 = None if g16 is not None else self.g32[s:e]
        z = self.g32[s:e] if zero else None      # ranges written with plain stores need no re-zeroing
        # a uniform decay goes as the scalar: the launch is the one made before segment tables existed
        wd_kw = dict(weight_decay=segs[0][1]) if len(segs) == 1 else dict(weight_decay=segs[0][1], wd_segments=segs)
        if self.opt_name in ("adam", "adamw"):
            if self.opt_name == "adamw":
                wd_kw["decoupled"] = True
            ops.adam_step(self.p32[s:e], self.m32[s:e], self.v32[s:e], g32=g32, g16=g16, shadow=self.w16[s:e],
                          lr=self.lr, beta1=self.beta1, beta2=self.beta2, eps=self.eps,
                          step=self.step_count, grad_scale=grad_scale, zero=z, **wd_kw, **self._ema_kw(s, e))
        else:
            ops.sgd_step(self.p32[s:e], self.m32[s:e], g32=g32, g16=g16, shadow=self.w16[s:e], lr=self.lr,
                         momentum=self.momentum, first=(self.step_count == 1), grad_scale=grad_scale, zero=z,
                         **wd_kw, **self._ema_kw(s, e))

    def _reduce_and_update(self, bi: int) -> None:
        bk = self.plan.buckets[bi]
        s, e = bk.start, bk.end
        # g32 holds the sum of the group's k' micro-batch means: the update uses their mean (1/k' where
        # 1/world is applied, on the optimizer's grad_scale at world 1)
        k = self._accum + 1
        if self.world == 1:
            if self.apply_updates:
                # The optimizer is HBM-bound, the convolutions still to come are tensor-bound: run the
                # update of a finished bucket on the side stream so it hides under the rest of backward
                # (FC-1/FC-2 are 88 % of the parameters and finish first).
                ev = torch.cuda.Event()
                ev.record()
                self.comm_stream.wait_event(ev)
                with torch.cuda.stream(self.comm_stream):
                    self._mark("opt%d start" % bi, "comm")
                    self._apply_update(s, e, None, zero=not self._bucket_store_only[bi], grad_scale=1.0 / k)
                    self._mark("opt%d end" % bi, "comm")
            return
        ev = torch.cuda.Event()
        ev.record()
        self.comm_stream.wait_event(ev)
        with torch.cuda.stream(self.comm_stream):
            if self.use_nccl:                    # library baseline (comparison only)
                self.g32[s:e].mul_(1.0 / (self.world * k))
                dist.all_reduce(self.g32[s:e])
                if self.apply_updates:
                    self._apply_update(s, e, None)
                return
            algo = self.arena.pick_algo(e - s, self.ar_algo)
            if self.deterministic and algo == "nvls":        # auto may pick it: the two-shot adds in rank order
                algo = "twoshot"
            prepacked = self._wire_direct and self._bucket_prepacked[bi]
            if self._bucket_prepacked[bi] and algo == "oneshot":
                algo = "twoshot"                 # one-shot cannot leave its result on the wire
            # ZeRO-1 only for buckets that hold nothing but one big FC weight (88 % of the parameters):
            # the forward pass reads those through the all-gathered bf16 shadow.  Buckets with biases
            # stay replicated -- biases are read from the fp32 master, which under ZeRO-1 is current on
            # the owner rank only.
            if self.zero1 and self.apply_updates and self._bucket_prepacked[bi] and algo != "oneshot":
                self._mark("z1_%d start" % bi, "comm")
                zev0 = None
                if self._comm_events is not None:
                    zev0 = torch.cuda.Event(enable_timing=True)
                    zev0.record()
                self.arena.zero1_step(None if prepacked else self.g32, self.p32, self.m32, self.v32, self.w16,
                                      s, e - s, algo=algo, slot=bi % self.arena.slots, max_ctas=self.zero1_ctas,
                                      inv_world=1.0 / (self.world * k), lr=self.lr, beta1=self.beta1,
                                      beta2=self.beta2, eps=self.eps, weight_decay=self._wd_segments[s][0][1],
                                      step=self.step_count, decoupled=self.opt_name == "adamw",
                                      **self._ema_kw(s, e))
                self._zero1_buckets.add(bi)
                if zev0 is not None:             # reduce-scatter + optimizer + all-gather: same wire bytes
                    zev1 = torch.cuda.Event(enable_timing=True)
                    zev1.record()
                    self._comm_events.append((zev0, zev1, (e - s) * self.arena.wire.element_size()))
                self._mark("z1_%d end" % bi, "comm")
                return
            # LARS reads a tensor's gradient again in its phase 2, after later buckets reduced: in g32, whatever
            # algorithm each bucket took
            to_f32 = (algo == "oneshot" or self.unpack_fp32 or self.arena.wire_dtype == F32
                      or not self.apply_updates or self.opt_name == "lars")
            self._mark("ar%d start" % bi, "comm")
            ev0 = None
            if self._comm_events is not None:    # observability: device time of every reduction
                ev0 = torch.cuda.Event(enable_timing=True)
                ev0.record()
            self.arena.allreduce(None if prepacked else self.g32, self.g32 if to_f32 else None, s, e - s,
                                 algo=algo, slot=bi % self.arena.slots, max_ctas=self.comm_ctas,
                                 inv_world=1.0 / (self.world * k))
            if ev0 is not None:
                ev1 = torch.cuda.Event(enable_timing=True)
                ev1.record()
                self._comm_events.append((ev0, ev1, (e - s) * self.arena.wire.element_size()))
            if self.cross_group is not None:     # node sums (already x 1/(world k')) -> job sum, over NCCL
                dist.all_reduce(self.g32[s:e] if to_f32 else self.arena.wire[s:e], group=self.cross_group)
            self._mark("ar%d end" % bi, "comm")
            if self.apply_updates:
                if self.opt_stream is not self.comm_stream:
                    red = torch.cuda.Event()
                    red.record()                      # on the comm stream: bucket bi is reduced
                    self.opt_stream.wait_event(red)
                with torch.cuda.stream(self.opt_stream):
                    self._apply_update(s, e, None if to_f32 else self.arena.wire[s:e],
                                       zero=not (prepacked or self._bucket_store_only[bi]))
                    self._mark("opt%d end" % bi, "opt")

    def _end_step(self) -> None:
        cur = torch.cuda.current_stream(self.device)
        cur.wait_stream(self.comm_stream)
        if self.opt_stream is not self.comm_stream:
            cur.wait_stream(self.opt_stream)

    # ================================================================================ public
    def set_meter(self, meter: Optional[DeviceMeter]) -> None:
        self.meter = meter

    def set_distillation(self, teacher: Optional["TeacherEngine"], alpha: float = 0.5,
                         temperature: float = 4.0) -> None:
        """Train against ``teacher``'s logits as well as the labels (knowledge distillation): every train_step runs
        the teacher's forward on the staged input, and the loss is (1 - alpha) CE + alpha T^2 KL(teacher || student)
        at temperature T (ops.cross_entropy_kd).  None: plain cross-entropy again."""
        if teacher is not None:
            if not 0.0 < alpha <= 1.0:
                raise ValueError("distillation alpha must lie in (0, 1] (got %r)" % alpha)
            if not (math.isfinite(temperature) and temperature > 0.0):
                raise ValueError("distillation temperature must be finite and > 0 (got %r)" % temperature)
            if teacher.spec.num_classes != self.spec.num_classes:
                raise ValueError("the teacher has %d classes, the student %d" % (teacher.spec.num_classes,
                                                                                  self.spec.num_classes))
            if (teacher.B, teacher.HW, teacher.device) != (self.B, self.HW, self.device):
                raise ValueError("the teacher engine must be built for the student's batch, training crop and device")
            if teacher.deterministic != self.deterministic:
                raise ValueError("the teacher engine must follow the student's deterministic flag")
        self.teacher = teacher
        self.distill_alpha, self.distill_temperature = float(alpha), float(temperature)

    def set_class_weights(self, weights: Optional[torch.Tensor]) -> None:
        """Per-class loss weights (the reference's optional weighted cross-entropy)."""
        self.class_weights = None if weights is None else weights.to(self.device, F32).contiguous()

    def train_step(self, batch, update: bool = True, ema: bool = False) -> torch.Tensor:
        """One micro-batch: forward, loss and backward into the gradient arena, and with ``update`` the
        reduction and optimizer step over the group of micro-batches accumulated since the last update
        (mean of their gradients).  With ``ema`` (and ``update``) the optimizer launches also update the
        moving average of the weights from the new weights.  Returns the device scalar holding this
        batch's mean loss."""
        if ema:
            self._require_ema("train_step(ema=True)")
        self._ema_step = bool(ema and update and self.apply_updates)
        self._powersgd_begin(self.step_count + 1)
        self.micro_count += 1
        if update:
            self.step_count += 1
        self._update = bool(update)
        # FC-1 / FC-2 gradients go straight to the wire as bf16 only when nothing else is to be added
        self._wire_direct = self._update and self._accum == 0
        t = self.timer
        if self.nvtx:
            torch.cuda.nvtx.range_push("step")
        self._mark("step start")
        t.start("input")
        self._set_hw(self.HW)
        b = self._stage_input(batch)
        t.stop("input")
        self._mark("input")
        if self.teacher is not None:
            t.start("teacher")
            self._teacher_logits = self.teacher.forward_teacher(self.x_nhwc, self.labels_dev, b)
            t.stop("teacher")
            self._mark("teacher")
        t.start("forward")
        self._forward(b, train=True)
        self._loss(b, train=True)
        self._release_input()
        self._mark("loss")
        t.stop("forward")
        t.start("backward+reduce+update")
        self._begin_step()
        self._frozen_ema()
        self._backward(b)
        self._end_step()
        self._accum = 0 if update else self._accum + 1
        if self._ema_step:
            self.ema_updates += 1
            self._ema16_current = False
            self._ema_step = False
        self._mark("step end (joined comm)")
        t.stop("backward+reduce+update")
        if self.nvtx:
            torch.cuda.nvtx.range_pop()
        return self.loss_buf

    def set_val_tta(self, mode: str) -> None:
        """Evaluate with test-time augmentation (``data.transforms.TTA_VIEWS``): every eval_step runs each view of
        the batch through the network and scores the mean of their softmaxes; forward_logits returns every view's
        logits.  "none": the single centre crop, as without this call."""
        T.tta_views(mode)
        self.val_tta = mode
        self.tta_acc = None if mode == "none" else torch.empty(self.B, self.spec.num_classes, dtype=F32,
                                                               device=self.device)

    def _view_logits(self, b: int) -> None:
        """The evaluation forward of the network input into self.logits[:b] (the fused head's evaluation pass writes
        them with its metrics in the scratch meter)."""
        self._forward(b, train=False)
        if self.fused_head:
            keep = self.meter
            self.meter = None
            self._loss(b, train=False)
            self.meter = keep

    def _tta_pass(self, batch, keep: Optional[list] = None) -> int:
        """Stage the batch once, then per view: its augment launch, the forward at batch b and, without ``keep``,
        the view's step of the reduction (into the meter at the last view).  ``keep``: collect each view's logits
        instead of reducing them.  Views are looped rather than stacked into a larger batch, so every launch keeps
        a shape the single-crop pass already makes."""
        views = T.tta_views(self.val_tta)
        meter = self.meter.buf if self.meter is not None else self.scratch_meter
        b = self._stage_input(batch, views)
        for i in range(len(views)):
            if i:
                self._view_input(batch, b, i, views)
            self._view_logits(b)
            if keep is not None:
                keep.append(self.logits[:b].clone())
            else:
                ops.tta_accumulate(self.logits[:b], self.labels_dev[:b], self.tta_acc, view=i, views=len(views),
                                   meter=meter, loss_out=self.loss_buf)
        return b

    def eval_step(self, batch, ema: bool = False) -> torch.Tensor:
        """Evaluation forward, loss and metrics; ``ema``: with the moving average of the weights
        (after prepare_ema()).  With a TTA mode (set_val_tta) the loss and metrics are those of the view mean.
        A meter with a confusion matrix (DeviceMeter(num_classes=)) also gets the batch's per-class counts: one
        class_metrics launch on the logits, or on the view sums after the last view."""
        counts = self.meter is not None and self.meter.confusion is not None
        with self._eval_pass(ema):
            if self.val_tta != "none":
                b = self._tta_pass(batch)
                if counts:
                    ops.class_metrics(self.tta_acc[:b], self.labels_dev[:b], self.meter.confusion, self.meter.top5,
                                      views=len(T.tta_views(self.val_tta)))
                self._release_input()
                return self.loss_buf
            b = self._stage_input(batch)
            self._forward(b, train=False)
            self._loss(b, train=False)
            if counts:
                ops.class_metrics(self.logits[:b], self.labels_dev[:b], self.meter.confusion, self.meter.top5)
            self._release_input()
        return self.loss_buf

    def forward_logits(self, batch, ema: bool = False) -> torch.Tensor:
        """Logits [b][C] fp32 of an evaluation pass; with a TTA mode (set_val_tta) every view's, [b][V][C]."""
        with self._eval_pass(ema):
            if self.val_tta != "none":
                keep = []
                self._tta_pass(batch, keep)
                self._release_input()
                return torch.stack(keep, 1)
            b = self._stage_input(batch)
            self._view_logits(b)
            self._release_input()
        return self.logits[:b].clone()

    @contextlib.contextmanager
    def _eval_pass(self, ema: bool):
        """An evaluation pass: the weights of ``_use_weights(ema)`` at the evaluation size, then the training
        weights and size again."""
        self._use_weights(ema)
        self._set_hw(self.eval_hw)
        try:
            yield
        finally:
            self._use_weights(False)
            self._set_hw(self.HW)

    def _use_weights(self, ema: bool) -> None:
        """Point the forward pass at the EMA arenas (ema16 weights, ema32 biases) or back at w16 / p32."""
        if ema:
            self._require_ema("an EMA evaluation pass")
            if not self._ema16_current:
                raise RuntimeError("the EMA changed since its last cast: call prepare_ema() before an EMA pass")
            self._wsrc, self._bsrc = self.ema16, self.ema32
        else:
            self._wsrc, self._bsrc = self.w16, self.p32

    def sync(self) -> None:
        torch.cuda.synchronize(self.device)

    # ---- step timeline (SURVEY 5.1 tracing; there is no nsys on the box) ----------------------------
    def timeline(self, on: bool) -> None:
        """Record a CUDA event after every layer's kernels on the compute stream and around every
        all-reduce / optimizer launch on the comm stream.  ``timeline_report()`` turns them into
        milliseconds since the start of the step: which bucket's reduction ran under which layer's
        backward, and what (if anything) is exposed after the last wgrad."""
        self._tl = [] if on else None

    def _mark(self, name: str, lane: str = "compute") -> None:
        if self._tl is not None:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()                      # on the current stream
            self._tl.append((name, lane, ev))

    def timeline_report(self) -> list:
        """[(name, lane, ms since the step's first mark)] for everything recorded since timeline(True)."""
        if not self._tl:
            return []
        self.sync()
        t0 = self._tl[0][2]
        out = [(n, lane, round(t0.elapsed_time(ev), 4)) for n, lane, ev in self._tl]
        self._tl = []
        return out

    # ---- gradient all-reduce observability (SURVEY 5.5: GB/s and roofline fraction) -----------------
    def comm_timing(self, on: bool) -> None:
        """Record CUDA events around every fused all-reduce launch (comm stream).  The times include
        whatever the kernel waits for (peers arriving late) and run under backward's kernels -- it is
        the rate the training step actually sees, not an isolated micro-benchmark."""
        self._comm_events = [] if on else None

    def comm_report(self, steps: int) -> Optional[dict]:
        """Device time and bus bandwidth of the gradient all-reduces of the last ``steps`` steps:
        bus GB/s = 2(ws-1)/ws * wire bytes / time (NCCL's convention), against H100 NVLink 4's
        nominal 450 GB/s per direction."""
        if not self._comm_events or self.world == 1:
            return None
        self.sync()
        ms = sum(a.elapsed_time(b) for a, b, _ in self._comm_events)
        nbytes = sum(n for _, _, n in self._comm_events)
        self._comm_events = []
        bus = 2.0 * (self.world - 1) / self.world * nbytes / (ms * 1e-3) / 1e9 if ms > 0 else 0.0
        return {"wire_MB_per_step": round(nbytes / steps / 1e6, 2), "ms_per_step": round(ms / steps, 4),
                "launches_per_step": len(self.plan.buckets), "bus_GBs": round(bus, 1),
                "frac_of_450_nominal": round(bus / 450.0, 3),
                "comm_ctas": self.comm_ctas, "overlapped_with_backward": True,
                "includes_fused_optimizer": bool(self._zero1_buckets)}

    def phase_times(self) -> Dict[str, float]:
        return self.timer.collect()

    # torch-module-like conveniences used by Trainer / checkpoint
    def train(self) -> None:
        pass

    def eval(self) -> None:
        pass


class TeacherEngine(NativeEngine):
    """A NativeEngine that only runs forward, in evaluation mode (no dropout): the teacher of knowledge distillation.
    It holds the weights (fp32 master for the biases, bf16 for the GEMMs), the input staging of an evaluation pass,
    the activations at the training crop and the evaluation crop, and the logits.  No gradient, moment, EMA or wire
    arena, no backward buffer and no comm or optimizer stream.  ``forward_teacher`` runs _forward and the fused
    head's evaluation pass on the student's staged input; ``eval_step`` scores it like any engine."""

    def __init__(self, spec: VGGSpec, device: torch.device, batch: int, state: Dict[str, torch.Tensor],
                 input_hw: int = DATA.crop, eval_hw: Optional[int] = None, deterministic: bool = False) -> None:
        ops.require()
        check_native_spec(spec)
        self.spec, self.device, self.B = spec, torch.device(device), int(batch)
        self.HW = check_native_hw(input_hw, "input_hw")
        self.eval_hw = self.HW if eval_hw is None else check_native_hw(eval_hw, "eval_hw")
        self.deterministic, self._ws = bool(deterministic), None
        self.world, self.rank, self.seed = 1, 0, 0            # each rank loads the same file: nothing to broadcast
        self.freeze_layers, self._frozen = 0, set()
        self.train_dropout, self.same_dropout_all_ranks, self.micro_count = False, False, 0
        self.label_smoothing, self._mix, self._accum = 0.0, None, 0
        self.meter, self.class_weights, self.teacher, self.ema32 = None, None, None, None
        self.timer, self.nvtx, self._tl = PhaseTimer(False), False, None
        self.plan = engine_bucket_plan(L.ready_order(spec), 32.0, 9.5, 2400.0)     # the arena offsets only
        self.p32 = torch.zeros(self.plan.total, dtype=F32, device=self.device)
        self.w16 = torch.zeros(self.plan.total, dtype=BF16, device=self.device)
        self.import_state(state, sync=False)
        self._wsrc, self._bsrc = self.w16, self.p32
        self._build_buffers(backward=False)

    def forward_teacher(self, x_nhwc: torch.Tensor, labels: torch.Tensor, b: int) -> torch.Tensor:
        """Logits [b][C] fp32 of the network input ``x_nhwc`` staged by the student at the training crop (read in
        place); ``labels`` only feed the fused head's metrics, which land in a scratch meter."""
        self._set_hw(self.HW)
        own = self.x_nhwc
        self.x_nhwc, self.labels_dev = x_nhwc, labels
        try:
            self._view_logits(b)
        finally:
            self.x_nhwc = own
        return self.logits[:b]

    def device_bytes(self) -> int:
        """Bytes of device memory the teacher's tensors take, from their shapes (views of one buffer counted once)."""
        seen, total = set(), 0

        def add(t) -> None:
            nonlocal total
            if isinstance(t, torch.Tensor):
                st = t.untyped_storage()
                if st.data_ptr() not in seen:
                    seen.add(st.data_ptr())
                    total += st.nbytes()
            elif isinstance(t, (list, tuple)):
                for u in t:
                    add(u)
            elif isinstance(t, dict):
                for u in t.values():
                    add(u)

        for v in vars(self).values():
            add(v)
        return total
