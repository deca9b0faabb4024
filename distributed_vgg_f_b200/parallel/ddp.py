"""Data-parallel wrapper for the torch-op (oracle / CPU) path.

Reference: ``nn.parallel.DistributedDataParallel(model)`` (distributedVggf.py:225) -- constructor
broadcast of rank-0 parameters, autograd hooks feeding a bucketed all-reduce that overlaps with the
rest of backward, gradients averaged (divided by world size before the sum).

``FlatDDP`` gives the same semantics with our own plumbing:
  * every ``param.grad`` is a *view* into one flat arena laid out in gradient-ready order
    (``parallel.buckets``), so a bucket is a contiguous range and nothing is copied;
  * ``register_post_accumulate_grad_hook`` marks tensors ready; when the last tensor of a bucket
    lands the bucket is pre-scaled by 1/ws and handed to a ``Collective`` asynchronously;
  * ``finish_backward()`` drains outstanding work before the optimizer step.
With ``powersgd=`` (a torch ``PowerSGDState``) the buckets are not all-reduced as they land: on the
synchronising backward, ``finish_backward()`` forms the accumulation group's mean and calls torch's own
``powerSGD_hook`` once per tensor, each tensor a bucket of its own, in the order autograd finished the
gradients of the first backward pass (DDP's rebuilt bucket order); the oracle of the native engine's
``--powersgd-rank``.
The ``Collective`` is ``TorchCollective`` (gloo on CPU -- BASELINE config #1) or
``parallel.fused.FusedCollective`` (our sm_90a P2P/NVLS kernels on the symmetric arena).
``state_dict()`` emits ``module.``-prefixed keys like the reference's wrapped model would.
"""
from __future__ import annotations

from typing import Dict, List

import torch
import torch.distributed as dist
from torch import nn

from .buckets import BucketPlan, make_bucket_plan
from .process_group import distributed_is_initialized


class TorchCollective:
    """All-reduce through torch.distributed (gloo / nccl).  The *baseline*, and the CPU path."""

    def __init__(self, group=None) -> None:
        self.group = group
        self.world_size = dist.get_world_size(group)

    def allocate(self, numel: int, dtype, device) -> torch.Tensor:
        return torch.zeros(numel, dtype=dtype, device=device)

    def broadcast_(self, flat: torch.Tensor, src: int = 0) -> None:
        dist.broadcast(flat, src=src, group=self.group)

    def allreduce_range_async(self, flat: torch.Tensor, start: int, end: int):
        view = flat[start:end]
        view.mul_(1.0 / self.world_size)          # DDP divides before summing
        return dist.all_reduce(view, op=dist.ReduceOp.SUM, group=self.group, async_op=True)


class FlatDDP(nn.Module):
    def __init__(self, module: nn.Module, collective=None, bucket_cap_mb: float = 64.0,
                 broadcast_from_rank0: bool = True, powersgd=None) -> None:
        super().__init__()
        self.module = module
        if collective is None and distributed_is_initialized():
            collective = TorchCollective()
        self.collective = collective
        params = [(n, p) for n, p in module.named_parameters() if p.requires_grad]
        ready = [(n, p.numel()) for n, p in reversed(params)]
        dtype, device = params[0][1].dtype, params[0][1].device
        cap = int(bucket_cap_mb * 1024 * 1024 / params[0][1].element_size())
        self.plan: BucketPlan = make_bucket_plan(ready, cap_elems=cap)
        alloc = collective.allocate if collective is not None else \
            (lambda n, dt, dev: torch.zeros(n, dtype=dt, device=dev))
        self.grad_arena = alloc(self.plan.total, dtype, device)
        self._params: Dict[str, nn.Parameter] = dict(params)
        self._pending: List[int] = []
        self._works: list = []
        self._require_sync = True
        self.powersgd = powersgd
        # the order autograd finished the gradients in the first backward pass: DDP rebuilds its buckets in this order
        # after the first iteration, and the hook's bucket indices (its initial Q draws) follow it
        self._ready_order: List[str] = []
        self._backwards = 0              # backward passes since zero_grad (the accumulation group)
        for name, p in params:
            off = self.plan.offsets[name]
            p.grad = self.grad_arena[off:off + p.numel()].view_as(p)
            p.register_post_accumulate_grad_hook(self._make_hook(name))
        self._bucket_missing = [len(b.tensors) for b in self.plan.buckets]
        if collective is not None and broadcast_from_rank0:
            self._sync_parameters()

    # -- construction-time sync (DDP's _sync_module_states) -------------------------------------
    def _sync_parameters(self) -> None:
        # every parameter, frozen ones (requires_grad off) included, as DDP's _sync_module_states does
        params = list(self.module.parameters())
        with torch.no_grad():
            flat = torch.cat([p.detach().reshape(-1) for p in params])
            self.collective.broadcast_(flat, 0)
            pos = 0
            for p in params:
                p.copy_(flat[pos:pos + p.numel()].view_as(p))
                pos += p.numel()

    # -- backward-time hooks -------------------------------------------------------------------
    def _make_hook(self, name: str):
        bucket_ids = None

        def hook(_param) -> None:
            nonlocal bucket_ids
            if self.powersgd is not None and len(self._ready_order) < len(self._params) \
                    and name not in self._ready_order:
                self._ready_order.append(name)
            if self.collective is None or not self._require_sync or self.powersgd is not None:
                return
            if bucket_ids is None:
                bucket_ids = self.plan.bucket_of(name)
            for bi in bucket_ids:
                self._bucket_missing[bi] -= 1
                if self._bucket_missing[bi] == 0:
                    b = self.plan.buckets[bi]
                    self._works.append(
                        self.collective.allreduce_range_async(self.grad_arena, b.start, b.end))
        return hook

    def forward(self, *args, **kwargs):
        return self.module(*args, **kwargs)

    def zero_grad(self, set_to_none: bool = False) -> None:   # grads are arena views: never None
        self.grad_arena.zero_()
        self._bucket_missing = [len(b.tensors) for b in self.plan.buckets]
        self._backwards = 0

    @property
    def averages_group(self) -> bool:
        """True when finish_backward already leaves the mean of the accumulation group in the gradients."""
        return self.powersgd is not None

    def _powersgd_exchange(self) -> None:
        from torch.distributed.algorithms.ddp_comm_hooks.powerSGD_hook import powerSGD_hook

        from .powersgd import HookBucket

        if self._backwards > 1:          # the hook sees the group's mean, as under DDP with a loss / K
            self.grad_arena.mul_(1.0 / self._backwards)
        names = self._ready_order
        for j, name in enumerate(names):
            off, p = self.plan.offsets[name], self._params[name]
            flat = self.grad_arena[off:off + p.numel()]
            out = powerSGD_hook(self.powersgd, HookBucket(j, flat, p.shape, j == len(names) - 1)).wait()
            if out.data_ptr() != flat.data_ptr():
                flat.copy_(out)

    def finish_backward(self) -> None:
        self._backwards += 1
        if self.powersgd is not None and self.collective is not None and self._require_sync:
            self._powersgd_exchange()
        for w in self._works:
            if w is not None:
                w.wait()
        self._works.clear()

    def state_dict(self, *args, **kwargs):
        return {"module." + k: v for k, v in self.module.state_dict(*args, **kwargs).items()}

    def load_state_dict(self, state, strict: bool = True):
        stripped = {(k[len("module."):] if k.startswith("module.") else k): v
                    for k, v in state.items()}
        return self.module.load_state_dict(stripped, strict=strict)
