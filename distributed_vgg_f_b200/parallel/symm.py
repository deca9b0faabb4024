"""Symmetric (peer-mapped) memory for the gradient wire buffer and the cross-GPU signal pads.

The reference moves gradients with gloo over TCP, staged through host memory (SURVEY N4).  Here
every rank owns a *wire* buffer and a *signal pad* that are mapped into every peer's address space
over NVLink (and, when the fabric supports it, bound to an NVSwitch multicast object so that
``multimem.ld_reduce`` / ``multimem.st`` work on it).  ``torch.distributed._symmetric_memory`` is
used strictly as the allocator + handle-exchange helper (CUDA VMM allocation, fd/fabric-handle
exchange through the rendezvous store); none of its collectives are called -- the raw device
pointer tables it returns are handed to our own kernels (csrc/allreduce.cu).
"""
from __future__ import annotations

from typing import Dict, Optional

import torch
import torch.distributed as dist

from .. import ops

ONESHOT_MAX_BYTES = 512 * 1024      # wire bytes below which the latency-optimal one-shot wins (no multicast)
ONESHOT_MAX_BYTES_NVLS = 0          # with NVLS the switch does the ws-way sum in one pass, which beat one-shot at
                                    # every size from 1 KB up where it was tuned (not yet measured on the H100)


def owned_cells(start: int, n: int, G: int, world: int, rank: int):
    """The cell decomposition of csrc/allreduce.cu in Python: the bucket is cut into G chunks of
    ``world`` cells of ``cell`` 8-element vectors; cell (b, r) is reduced (and, under ZeRO-1, owned)
    by rank r.  Returns [(first element, one past the last element)] for ``rank``."""
    nvec = n // 8
    cell = (nvec + G * world - 1) // (G * world)
    out = []
    for b in range(G):
        chunk0, chunk1 = min(nvec, b * world * cell), min(nvec, (b + 1) * world * cell)
        c0 = min(chunk1, chunk0 + rank * cell)
        c1 = min(chunk1, c0 + cell)
        if c1 > c0:
            out.append((start + 8 * c0, start + 8 * c1))
    return out


class SymmetricArena:
    def __init__(self, wire_elems: int, device: torch.device, wire_dtype: torch.dtype = torch.bfloat16,
                 slots: int = 32, group=None) -> None:
        import torch.distributed._symmetric_memory as symm_mem

        C = ops.require()
        self.group = group if group is not None else dist.group.WORLD
        self.rank = dist.get_rank(self.group)
        self.world = dist.get_world_size(self.group)
        self.device = device
        self.wire_dtype = wire_dtype
        try:
            symm_mem.set_backend("CUDA")
        except Exception:       # backend already fixed by an earlier allocation
            pass
        self.wire = symm_mem.empty(wire_elems, dtype=wire_dtype, device=device)
        self.wire.zero_()
        self.wire_hdl = symm_mem.rendezvous(self.wire, self.group)
        words = int(C.allreduce_signal_words(slots))
        self.flags = symm_mem.empty(words, dtype=torch.int32, device=device)
        self.flags.zero_()
        self.flags_hdl = symm_mem.rendezvous(self.flags, self.group)
        torch.cuda.synchronize(device)
        dist.barrier(self.group)        # every pad is zero before anybody signals
        self.has_multicast = bool(getattr(self.wire_hdl, "has_multicast_support", False)) and \
            int(getattr(self.wire_hdl, "multicast_ptr", 0) or 0) != 0
        mc = int(self.wire_hdl.multicast_ptr) if self.has_multicast else 0
        self.comm = C.make_comm(self.rank, self.world, int(self.wire_hdl.buffer_ptrs_dev),
                                int(self.flags_hdl.buffer_ptrs_dev), mc, 0,
                                self.wire.numel() * self.wire.element_size(), slots)
        self.slots = slots
        self._epoch: Dict[int, int] = {}
        self._algo = {"oneshot": C.AR_ONESHOT, "twoshot": C.AR_TWOSHOT, "nvls": C.AR_NVLS}

    def next_epoch(self, slot: int) -> int:
        e = self._epoch.get(slot, 0) + 1
        self._epoch[slot] = e
        return e

    def pick_algo(self, n_elems: int, requested: str = "auto") -> str:
        if requested != "auto":
            if requested == "nvls" and not self.has_multicast:
                raise RuntimeError("NVLS requested but the wire buffer has no multicast mapping")
            return requested
        nbytes = n_elems * self.wire.element_size()
        if nbytes <= (ONESHOT_MAX_BYTES_NVLS if self.has_multicast else ONESHOT_MAX_BYTES):
            return "oneshot"
        return "nvls" if self.has_multicast else "twoshot"

    def allreduce(self, grad_f32: Optional[torch.Tensor], grad_out_f32: Optional[torch.Tensor],
                  start: int, n: int, algo: str = "auto", slot: int = 0, max_ctas: int = 48,
                  inv_world: Optional[float] = None) -> str:
        """Fused pack + reduce (+ unpack) of arena range [start, start+n) on the current stream."""
        algo = self.pick_algo(n, algo)
        if algo == "oneshot" and grad_out_f32 is None:
            raise ValueError("one-shot writes its result to the fp32 arena: pass grad_out_f32")
        ops.require().allreduce(self.comm, grad_f32, grad_out_f32, start, n,
                                (1.0 / self.world) if inv_world is None else inv_world,
                                self._algo[algo], self.wire_dtype == torch.float32, slot,
                                self.next_epoch(slot), max_ctas)
        return algo

    def zero1_step(self, grad_f32: Optional[torch.Tensor], p32: torch.Tensor, m32: torch.Tensor,
                   v32: torch.Tensor, w16: torch.Tensor, start: int, n: int, *, algo: str, slot: int,
                   max_ctas: int, inv_world: float, lr: float, beta1: float, beta2: float, eps: float,
                   weight_decay: float, step: int, ema: Optional[torch.Tensor] = None, ema_decay: float = 0.0,
                   ema_first: bool = False, decoupled: bool = False) -> None:
        """EXPERIMENTAL: reduce-scatter + Adam on the cells this rank owns + all-gather of the new
        bf16 weights, one kernel (csrc/allreduce.cu::zero1_kernel).  bf16 wire, two-shot or NVLS.
        ``ema``: the owner also updates the weights' moving average of its cells (ops.adam_step).
        ``decoupled``: AdamW, as ops.adam_step."""
        if self.wire_dtype != torch.bfloat16 or algo not in ("twoshot", "nvls"):
            raise ValueError("zero1_step needs the bf16 wire and a reduce-scatter algorithm")
        tail = ops._ema_args(ema, ema_decay, ema_first) if not decoupled else \
            (ema, float(ema_decay), bool(ema_first), True)
        ops.require().zero1_step(self.comm, grad_f32, p32, m32, v32, w16, start, n, inv_world,
                                 self._algo[algo], slot, self.next_epoch(slot), max_ctas, lr, beta1, beta2,
                                 eps, weight_decay, step, *tail)

    def owned_ranges(self, start: int, n: int, max_ctas: int):
        """Element ranges of [start, start+n) whose fp32 master this rank owns under zero1_step
        (cell (b, r) of the kernel's decomposition belongs to rank r)."""
        G = int(ops.require().allreduce_grid(n, self.world, max_ctas, False))
        return owned_cells(start, n, G, self.world, self.rank)

    def broadcast_(self, data_f32: torch.Tensor, root: int = 0, slot: int = 0) -> None:
        """Rank ``root``'s fp32 ``data`` -> every rank, pulled through the wire buffer in chunks."""
        cap = (self.wire.numel() * self.wire.element_size()) // 4
        cap -= cap % 4
        flat = data_f32.view(-1)
        pos = 0
        while pos < flat.numel():
            n = min(cap, flat.numel() - pos)
            n4 = n - n % 4
            if n4:
                ops.require().broadcast(self.comm, flat[pos:pos + n4], root, slot, self.next_epoch(slot))
            if n4 != n:       # tail shorter than a vector: go through the control plane
                tail = flat[pos + n4:pos + n].clone()
                dist.broadcast(tail, src=root, group=self.group)
                flat[pos + n4:pos + n].copy_(tail)
            pos += n

    def barrier(self, slot: int = 0) -> None:
        ops.require().barrier(self.comm, slot, self.next_epoch(slot))
