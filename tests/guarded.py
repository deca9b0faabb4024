"""Guarded operands: the footprint half of the kernel checks.

``Guarded`` places a tensor of a given shape, strides, dtype and storage offset mod 16 elements
inside a larger buffer (so the kernel takes the same alignment paths as with the engine's tensor):

* a guard of at least 64 KiB before it;
* a guard of min(operand extent, 64 MiB), and at least 64 KiB, after it -- room for a whole extra
  pixel box of an activation (32 images at 14^2, 8 at 28^2), so that a kernel which rounds a
  ragged batch up to its batch block writes into the guard rather than past it;
* the gaps of a strided view (``ldo > M``, ``[:, :K]`` of a ``[M, Kp]`` buffer).

Guards and gaps hold a poison value; ``seal()`` snapshots the whole buffer after the operand has
been filled and ``check()`` requires every byte outside the regions the kernel is allowed to write
to be bit-identical (integer views, so NaN compares like any other pattern).  A read-only operand
allows no region at all: it must come back bitwise unchanged, guards, gaps and contents alike.

The poison is chosen per operand so that reading a guard element changes a checked output:

* float operands that are summed or multiplied (wgmma operands, biases, gradients, optimizer state,
  casts): NaN, which survives a multiplication by zero;
* float operands reduced by a maximum (max-pool inputs, cross-entropy logits): the largest finite
  value, because fmaxf and ``v > max`` drop a NaN;
* stored outputs are pre-filled with NaN over their whole extent, so an element the kernel should
  have written but skipped fails the value check;
* index and parameter operands hold values the kernel can consume without leaving its operands: a
  valid class index for int64 targets, an in-range crop box for augment parameters, all bits set
  (argmax 3, maximum > 0) for int32 pool-mask words.  An invalid index would turn a stray read into
  a memory fault instead of a wrong value.
"""
from __future__ import annotations

import torch

GUARD_BEFORE = 64 * 1024          # bytes
GUARD_AFTER_MIN = 64 * 1024
GUARD_AFTER_MAX = 64 * 1024 * 1024
_INT = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}


def extent(shape, stride) -> int:
    """Elements from the first to one past the last element of a strided view."""
    if any(n == 0 for n in shape):
        return 0
    return 1 + sum((n - 1) * st for n, st in zip(shape, stride))


NAN = float("nan")


def fmax(dtype):
    """The largest finite value of a float dtype: the poison of max-reduced operands."""
    return torch.finfo(dtype).max


class Guarded:
    """One operand inside its guarded buffer.  ``t`` is the operand; ``poison`` is a scalar or a 1-D
    pattern tiled over the buffer from its start."""

    def __init__(self, shape, stride, dtype, offset, poison, device):
        shape, stride = tuple(shape), tuple(stride)
        isz = torch.empty((), dtype=dtype).element_size()
        n = extent(shape, stride)
        before = (-(-GUARD_BEFORE // isz) + 15) // 16 * 16 + offset % 16
        after = -(-max(GUARD_AFTER_MIN, min(n * isz, GUARD_AFTER_MAX)) // isz)
        total = before + n + after
        if isinstance(poison, torch.Tensor):
            reps = -(-total // poison.numel())
            self.base = poison.to(device=device, dtype=dtype).repeat(reps)[:total].clone()
        else:
            self.base = torch.full((total,), poison, dtype=dtype, device=device)
        self.t = self.base.as_strided(shape, stride, before)
        self.lo, self.hi = before, before + n
        self._snap = None

    def bits(self) -> torch.Tensor:
        return self.base.view(_INT[self.base.element_size()])

    def seal(self) -> None:
        self._snap = self.bits().clone()

    def check(self, written=(), what: str = "") -> None:
        """Every element outside the views in ``written`` (views of ``t``) is bit-identical to the
        snapshot of ``seal()``."""
        assert self._snap is not None, "seal() before the launch"
        diff = self.bits() != self._snap
        for w in written:
            assert w.untyped_storage().data_ptr() == self.base.untyped_storage().data_ptr(), "not a view of t"
            diff.as_strided(tuple(w.shape), tuple(w.stride()), w.storage_offset()).fill_(False)
        n = int(diff.sum())
        if not n:
            return
        first = int(diff.nonzero()[0, 0])
        last = int(diff.nonzero()[-1, 0])
        inside = torch.zeros_like(diff)
        inside.as_strided(tuple(self.t.shape), tuple(self.t.stride()), self.t.storage_offset()).fill_(True)

        def where(i):
            if i < self.lo:
                return "%d elements before the start" % (self.lo - i)
            if i >= self.hi:
                return "%d elements past the end" % (i - self.hi + 1)
            return "inside the operand (offset %d)" % (i - self.lo) if bool(inside[i]) else \
                "in a stride gap (offset %d)" % (i - self.lo)

        raise AssertionError("%s: %d elements changed outside what the kernel may write; first %s, last %s" %
                             (what, n, where(first), where(last)))


def guarded(shape, stride, dtype, offset, poison, device, values=None) -> Guarded:
    """A guarded operand; ``values`` (a tensor of ``shape``, or None to leave it poisoned) fills it."""
    g = Guarded(shape, stride, dtype, offset, poison, device)
    if values is not None:
        g.t.copy_(values.reshape(g.t.shape))
    return g
