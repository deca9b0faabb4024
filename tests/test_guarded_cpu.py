"""Evidence, without a GPU, that the guarded operands of guarded.py catch footprint defects.

A fake kernel on CPU tensors (out = 2 a + 1 over a strided view; acc += a) passes the guard
check and the value check; each planted defect fails one of them: a write one element past the
end, one before the start, one into a stride gap, an output element never written, an
accumulation target overwritten, and a read of one poisoned element before, after or in a gap,
summed or reduced by a maximum.
"""
import pytest
import torch

import guarded as G
import kernel_check as KC
from launch_replay import ACCUM, CONTRACT, READ, RECORDED, STORE, UPDATE

CPU = "cpu"
F64 = torch.float64
SHAPE, STRIDE, OFF = (4, 6), (8, 1), 3          # [:, :6] of a [4, 8] buffer at element offset 3


def _operands(dtype=torch.float32):
    g = torch.Generator().manual_seed(0)
    a = G.guarded(SHAPE, STRIDE, dtype, OFF, G.NAN, CPU, torch.randint(-4, 5, SHAPE, generator=g).to(dtype))
    out = G.guarded(SHAPE, STRIDE, dtype, OFF, G.NAN, CPU)                               # stored: left poisoned
    acc = G.guarded(SHAPE, STRIDE, dtype, OFF, G.NAN, CPU, torch.randint(-8, 9, SHAPE, generator=g).to(dtype))
    pre = acc.t.clone()
    for op in (a, out, acc):
        op.seal()
    return a, out, acc, pre


def _check(a, out, acc, pre):
    ref = a.t.to(F64) * 2 + 1
    KC.check(out.t, ref, ref.abs(), chain=0, exact=True, what="out")
    KC.check(acc.t, pre.to(F64) + a.t.to(F64), pre.to(F64).abs() + a.t.to(F64).abs(), chain=0, exact=True,
             what="acc")
    a.check((), what="a")
    out.check((out.t,), what="out")
    acc.check((acc.t,), what="acc")


def _kernel(a, out, acc):
    out.t.copy_(a.t * 2 + 1)
    acc.t.add_(a.t)


def _at(op, offset, shape=(1,), stride=(1,)):
    """A view of the buffer at an element offset relative to the operand's first element."""
    return op.base.as_strided(shape, stride, op.lo + offset)


def test_guards_have_the_promised_layout():
    op = G.Guarded((37, 14, 14, 512), (14 * 14 * 512, 14 * 512, 512, 1), torch.bfloat16, 5, G.NAN, CPU)
    n = G.extent(op.t.shape, op.t.stride())
    assert op.lo * 2 >= 64 * 1024 and op.lo % 16 == 5 and op.t.storage_offset() == op.lo
    assert (op.base.numel() - op.hi) * 2 >= min(n * 2, 64 << 20) and op.base.numel() - op.hi >= 32 * 14 * 14 * 512
    small = G.Guarded((3,), (1,), torch.float32, 0, 0.0, CPU)
    assert (small.base.numel() - small.hi) * 4 >= 64 * 1024
    gaps = G.guarded(SHAPE, STRIDE, torch.float32, OFF, G.NAN, CPU, torch.zeros(SHAPE))
    assert bool(gaps.base[gaps.lo + 6:gaps.lo + 8].isnan().all())          # the gap keeps the poison


def test_a_correct_kernel_passes():
    a, out, acc, pre = _operands()
    _kernel(a, out, acc)
    _check(a, out, acc, pre)


@pytest.mark.parametrize("where", ["past the end", "before the start", "in a stride gap"])
def test_a_stray_write_fails(where):
    a, out, acc, pre = _operands()
    _kernel(a, out, acc)
    offset = {"past the end": G.extent(SHAPE, STRIDE), "before the start": -1, "in a stride gap": 6}[where]
    _at(out, offset).fill_(1.0)
    with pytest.raises(AssertionError, match=where):
        _check(a, out, acc, pre)


def test_a_write_into_a_read_only_operand_fails():
    a, out, acc, pre = _operands()
    _kernel(a, out, acc)
    a.t[1, 2] += 1
    with pytest.raises(AssertionError, match="inside the operand"):
        a.check((), what="a")


def test_an_element_never_written_fails():
    a, out, acc, pre = _operands()
    saved = out.t[3, 5].clone()
    _kernel(a, out, acc)
    out.t[3, 5] = saved                                  # still the poison
    with pytest.raises(AssertionError, match="out"):
        _check(a, out, acc, pre)


def test_an_overwritten_accumulation_target_fails():
    a, out, acc, pre = _operands()
    out.t.copy_(a.t * 2 + 1)
    acc.t.copy_(a.t)                                     # a store instead of an add
    with pytest.raises(AssertionError, match="acc"):
        _check(a, out, acc, pre)


@pytest.mark.parametrize("where", ["before", "after", "gap"])
@pytest.mark.parametrize("reduce", ["sum", "max"])
def test_reading_one_poisoned_element_changes_a_checked_output(where, reduce):
    """A row reduction that reads one element too many: the sum picks up a NaN poison, the maximum
    the largest-finite poison (a NaN would vanish in fmaxf, shown last)."""
    poison = G.NAN if reduce == "sum" else G.fmax(torch.float32)
    g = torch.Generator().manual_seed(1)
    a = G.guarded(SHAPE, STRIDE, torch.float32, OFF, poison, CPU, torch.randint(-4, 5, SHAPE, generator=g).float())
    out = G.guarded((4,), (1,), torch.float32, 0, G.NAN, CPU)
    a.seal()
    out.seal()
    rows = a.t.clone()
    stray = {"before": _at(a, -1), "after": _at(a, G.extent(SHAPE, STRIDE)), "gap": _at(a, 6)}[where]
    row = 0 if where != "after" else 3
    if reduce == "sum":
        ref = rows.to(F64).sum(1)
        got = rows.sum(1)
        got[row] = got[row] + stray[0]
    else:
        ref = rows.to(F64).amax(1)
        got = rows.amax(1)
        got[row] = torch.fmax(got[row], stray[0])
    out.t.copy_(got)
    a.check((), what="a")                                # reading leaves no trace in the guards ...
    with pytest.raises(AssertionError):                  # ... but the output shows it
        KC.check(out.t, ref, ref.abs(), chain=0, exact=True, what=reduce)
    if reduce == "max":
        assert torch.fmax(got[row].new_tensor(float("nan")), rows[row].amax()) == rows[row].amax()


def test_the_write_contract_covers_the_recorded_kernels():
    assert set(CONTRACT) == set(RECORDED) and len(RECORDED) == len(set(RECORDED))
    for name, row in CONTRACT.items():
        for key, role in row.items():
            if callable(role):
                roles = {role({"atomic": t, "clear": t}) for t in (False, True)}
            else:
                roles = {role}
            assert roles <= {READ, STORE, ACCUM, UPDATE}, (name, key)
    assert CONTRACT["cross_entropy"]["dlogits"] == STORE and CONTRACT["adam"]["zero"] == UPDATE
    assert CONTRACT["fc_bias_act"]["acc"]({"clear": True}) == UPDATE
    assert CONTRACT["fc_bias_act"]["acc"]({"clear": False}) == READ
    assert CONTRACT["gemm"]["out"]({"atomic": True}) == ACCUM
