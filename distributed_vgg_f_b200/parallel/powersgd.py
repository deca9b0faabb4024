"""PowerSGD gradient compression (``--powersgd-rank r``): torch's ``powerSGD_hook`` with each parameter in a
DDP bucket of its own, the buckets in DDP's order (``hook_order``).

What both engines share lives here: which tensors are compressed (torch's ``_should_compress``), the bytes an
update puts on the wire, the initial Q draws (reproduced on the host exactly as the hook draws them) and their
permutation into the native column order.  The native engine runs the compression with the kernels of
``csrc/powersgd.cu``; the torch-op engine (``FlatDDP(powersgd=...)``) calls the hook itself.
"""
from __future__ import annotations

import dataclasses
import math
from typing import Dict, List, Sequence

import numpy as np
import torch

from ..models import layout as L
from ..models.vggf import VGGSpec

MAX_RANK = 8                   # the kernels keep r fp32 accumulators per thread in a 40-register budget
MIN_COMPRESSION_RATE = 2       # torch's PowerSGDState default
DEFAULT_START_ITER = 1000      # torch's PowerSGDState default


def check_config(rank: int, start_iter: int) -> None:
    """The rank and start iteration a run may use (rank 0: PowerSGD off)."""
    if not 0 <= int(rank) <= MAX_RANK:
        raise ValueError("--powersgd-rank must lie in [0, %d] (got %d): the compression kernels keep r fp32 "
                         "accumulators per thread, and more than %d do not fit their register budget"
                         % (MAX_RANK, rank, MAX_RANK))
    if rank and int(start_iter) < 2:
        raise ValueError("--powersgd-start-iter must be >= 2 (got %d): torch's PowerSGD with error feedback and "
                         "warm start refuses a start before DDP's buckets are rebuilt after the first iteration"
                         % start_iter)


@dataclasses.dataclass(frozen=True)
class TensorPlan:
    name: str
    n: int                     # rows: torch shape[0]
    m: int                     # columns in torch's layout: prod(shape[1:])
    rank: int                  # r' = min(n, m, r)
    compressed: bool

    @property
    def pq_elems(self) -> int:
        """P + Q elements a compressed update exchanges (0 when uncompressed)."""
        return (self.n + self.m) * self.rank if self.compressed else 0


def should_compress(n: int, m: int, rank: int) -> bool:
    """torch's _should_compress with min_compression_rate = 2."""
    return (n + m) * rank * MIN_COMPRESSION_RATE < n * m


def tensor_plan(spec: VGGSpec, name: str, rank: int) -> TensorPlan:
    shape = spec.param_shape(name)
    n = int(shape[0])
    m = int(math.prod(shape[1:])) if len(shape) > 1 else 1
    r = min(n, m, int(rank))
    return TensorPlan(name, n, m, r, should_compress(n, m, r))


def hook_order(spec: VGGSpec, freeze_layers: int = 0) -> List[str]:
    """The trainable tensors in DDP's bucket order once it has rebuilt its buckets after the first iteration:
    the order autograd finishes the gradients, which is ``models.layout.ready_order`` except that a convolution's
    weight gradient is final before its bias gradient (a Linear's bias comes first).  Bucket j takes the j-th
    initial-Q draw."""
    frozen = set(spec.frozen_param_names(freeze_layers))
    convs = {c.name for c in spec.convs}
    out: List[str] = []
    for name, _ in L.ready_order(spec):
        if name in frozen:
            continue
        base, kind = name.rsplit(".", 1)
        if kind == "weight" and base in convs and out and out[-1] == base + ".bias":
            out.insert(len(out) - 1, name)
        else:
            out.append(name)
    return out


def plan(spec: VGGSpec, rank: int, freeze_layers: int = 0) -> List[TensorPlan]:
    """Every trainable tensor in DDP's bucket order (``hook_order``), with its compression decision."""
    return [tensor_plan(spec, n, rank) for n in hook_order(spec, freeze_layers)]


def exchange_bytes(rows: Sequence[TensorPlan], wire_bytes: int = 2) -> Dict[str, int]:
    """Bytes one update puts on the wire: fp32 P and Q of the compressed tensors, the rest at ``wire_bytes``
    per element (2: the bf16 wire), and the same model without compression."""
    comp = sum(4 * t.pq_elems for t in rows)
    unc = sum(wire_bytes * t.n * t.m for t in rows if not t.compressed)
    full = sum(wire_bytes * t.n * t.m for t in rows)
    return {"compressed": comp, "uncompressed": unc, "total": comp + unc, "without_powersgd": full}


def summary_line(rows: Sequence[TensorPlan], rank: int, wire_bytes: int = 2) -> str:
    b = exchange_bytes(rows, wire_bytes)
    return ("[powersgd] rank %d: %d of %d tensors compressed; per update %.2f MB of P + Q (fp32) and %.2f MB of "
            "uncompressed tensors, %.2f MB in all (%.1f MB without compression)"
            % (rank, sum(t.compressed for t in rows), len(rows), b["compressed"] / 1e6, b["uncompressed"] / 1e6,
               b["total"] / 1e6, b["without_powersgd"] / 1e6))


def initial_q_torch(rows: Sequence[TensorPlan], seed: int) -> Dict[str, torch.Tensor]:
    """The hook's first Q of every compressed tensor, [m][r'] in torch's column order: bucket j (``hook_order``)
    seeds torch's CPU generator with the j-th draw of ``RandomState(seed).randint(1_000_000_000)`` and takes
    ``torch.randn(1, m, r')``.  Every bucket consumes a draw, compressed or not."""
    rng = np.random.RandomState(seed)
    out: Dict[str, torch.Tensor] = {}
    with torch.random.fork_rng(devices=[]):
        for t in rows:
            torch.manual_seed(rng.randint(1_000_000_000))
            if t.compressed:
                out[t.name] = torch.randn(1, t.m, t.rank, device="cpu", dtype=torch.float32)[0]
    return out


def native_columns(spec: VGGSpec, name: str) -> torch.Tensor:
    """For each column of the native [n][m_native] gradient, its column in torch's layout (-1: padding).
    OHWI convolutions, conv0 padded to CONV0_K columns, classifier.0 in NHWC-flatten order."""
    base = name.rsplit(".", 1)[0]
    for i, c in enumerate(spec.convs):
        if c.name == base:
            # native (kh, kw, c) <- torch c * 9 + kh * 3 + kw
            idx = torch.arange(c.cin * 9).view(c.cin, 3, 3).permute(1, 2, 0).reshape(-1)
            if i == 0:
                idx = torch.cat([idx, torch.full((L.CONV0_K - idx.numel(),), -1, dtype=idx.dtype)])
            return idx
    shape = spec.param_shape(name)
    m = int(math.prod(shape[1:]))
    if base == spec.fcs[0].name:
        ph = spec.pooled_hw
        return torch.arange(m).view(m // (ph * ph), ph, ph).permute(1, 2, 0).reshape(-1)
    return torch.arange(m)


def q_to_native(spec: VGGSpec, name: str, q: torch.Tensor) -> torch.Tensor:
    """Torch-order Q [m][r'] -> native order [m_native][r'], zero rows at the padding."""
    cols = native_columns(spec, name)
    out = torch.zeros(cols.numel(), q.shape[1], dtype=q.dtype, device=q.device)
    keep = cols >= 0
    out[keep] = q[cols[keep].to(q.device)]
    return out


def q_to_torch(spec: VGGSpec, name: str, q: torch.Tensor) -> torch.Tensor:
    """Native-order Q [m_native][r'] -> torch order [m][r']."""
    cols = native_columns(spec, name)
    keep = cols >= 0
    out = torch.empty(int(keep.sum()), q.shape[1], dtype=q.dtype, device=q.device)
    out[cols[keep].to(q.device)] = q[keep.to(q.device)]
    return out


class HookBucket:
    """The part of ``dist.GradBucket`` that ``powerSGD_hook`` reads: one parameter's flat gradient."""

    def __init__(self, index: int, flat: torch.Tensor, shape, last: bool) -> None:
        self._index, self._flat, self._shape, self._last = index, flat, tuple(shape), last

    def buffer(self) -> torch.Tensor:
        return self._flat

    def index(self) -> int:
        return self._index

    def gradients(self) -> List[torch.Tensor]:
        return [self._flat.view(self._shape)]

    def is_last(self) -> bool:
        return self._last


def make_state(rank: int, start_iter: int, seed: int, process_group=None):
    """The torch PowerSGDState this project's --powersgd-rank / --powersgd-start-iter / --seed stand for."""
    from torch.distributed.algorithms.ddp_comm_hooks.powerSGD_hook import PowerSGDState

    return PowerSGDState(process_group=process_group, matrix_approximation_rank=int(rank),
                         start_powerSGD_iter=int(start_iter), min_compression_rate=MIN_COMPRESSION_RATE,
                         use_error_feedback=True, warm_start=True, orthogonalization_epsilon=0,
                         random_seed=int(seed))


def resolve_zero1(zero1, rank: int):
    """--zero1 under PowerSGD: ``auto`` turns ZeRO-1 off, ``on`` is refused (it shards the compressed tensors)."""
    if not rank:
        return zero1
    if zero1 is True:
        raise ValueError("--powersgd-rank with --zero1 on: ZeRO-1 shards the FC weights across ranks, and those are "
                         "the very tensors PowerSGD compresses; use --zero1 off (or auto)")
    return False


def check_deterministic(rank: int, deterministic: bool, world: int) -> None:
    if rank and deterministic and world > 1:
        raise ValueError("--powersgd-rank with --deterministic at world > 1: P and Q are summed with "
                         "dist.all_reduce, whose summation order NCCL does not promise")


def workspace_elems(rows: Sequence[TensorPlan], spec: VGGSpec, sms: int, C) -> int:
    """Back-projection workspace (floats) for the largest compressed tensor, native shapes."""
    best = 4
    for t in rows:
        if t.compressed:
            n, m = native_nm(spec, t.name)
            best = max(best, int(C.psgd_workspace_elems(n, m, t.rank, sms)))
    return best


def native_nm(spec: VGGSpec, name: str):
    shape = L.native_shape(spec, name)
    return int(shape[0]), int(math.prod(shape[1:]))


