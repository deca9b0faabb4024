"""The collective kernels of allreduce.cu (all-reduce one-shot and two-shot, bf16 and fp32 wire, pack
and wire-only entries; the fused ZeRO-1 step; broadcast; barrier) on ONE GPU, against bitwise fp32
emulations of their documented arithmetic and float64 references, with emulated ranks.

The kernels take raw pointer tables, so one process can hand a kernel W wire buffers and W signal pads
on the same device and run it as any rank of any world size: peer loads and stores become local ones,
and the arithmetic, the cell decomposition and the footprint are those of a real run.

Emulated ranks are launched one at a time on one stream and never wait: before each launch the rank's
whole own signal pad holds the launch's epoch, so every `(int)(flag - epoch) >= 0` poll passes at
once, whatever the pad layout.  (Several emulated ranks launched concurrently on one GPU would rely on
their CTAs being co-scheduled, which nothing guarantees.)  Sequential emulation is exact:

* two-shot: cell (b, r) is read and written by rank r only, so running ranks 0 .. W-1 one after
  another on the wire-only entry (grad=None) leaves every wire in its final all-reduced state;
* with the pack entry a rank overwrites its whole own wire range first: those launches are checked
  one rank at a time, with the peers' wires prefilled with what their own pack would have written.

Each case checks the exact bits of every reduced cell, packed vector, fp32 output, Adam state and
shadow weight, that nothing outside [start, start+n) of any wire, arena, gradient or output changes
(tests/guarded.py), and that a launch writes its epoch into exactly the words
[slot, phase, cta < G, src = rank] of every peer's signal pad.  Not covered here: the concurrent
handshake across real peers, NVLS (multimem needs a multicast object across GPUs) and NVLink timing;
test_multigpu.py covers those on a multi-GPU host."""
import itertools

import pytest
import torch

import kernel_check as KC
from guarded import NAN, Guarded
from distributed_vgg_f_b200.ops import ref as R
from distributed_vgg_f_b200.parallel.symm import owned_cells

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
MAX_WORLD = 16              # AR_MAX_WORLD
MAX_CTAS = 128              # AR_MAX_CTAS
THREADS = 256               # AR_THREADS
SLOTS = 4
PAD_POISON = 0x5A5A5A5A     # signal-pad guards
# NaN payloads of their own for the wires and the shadows: a kernel that copied a guard of one into the
# other (an unpack or shadow copy that starts a vector early) changes the bits it lands on
WIRE_POISON = {torch.bfloat16: 0x7FA1, torch.float32: 0x7FC0A1A1}
SHADOW_POISON = 0x7FB2
TAIL = 24                   # elements of every tensor past start + n: inside the tensor, outside the range


def _C():
    from distributed_vgg_f_b200 import ops
    return ops.require()


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


_EPOCHS = itertools.count(0x7FFFFFF0)       # crosses the int32 sign boundary early


def _next_epoch():
    return next(_EPOCHS) % 0xFFFFFFFF + 1     # never 0: a peer pad starts at 0


def _i32(epoch):
    return epoch - (1 << 32) if epoch >= (1 << 31) else epoch


def _grid(n, world, max_ctas, wire_fp32):
    """allreduce_grid of allreduce.cu, restated."""
    nvec = n // (4 if wire_fp32 else 8)
    G = min(48 if max_ctas <= 0 else max_ctas, MAX_CTAS)
    return max(1, min(G, nvec // (THREADS * world) + 1))


def _owner_map(n, G, world, epv):
    """Owning rank of every element of [0, n) under the kernels' decomposition: G chunks of ``world``
    cells of ``cell`` vectors of ``epv`` elements; cell (b, r) belongs to rank r."""
    nvec = n // epv
    cell = -(-nvec // (G * world))
    own = torch.full((n,), -1, dtype=torch.int8)
    for b in range(G):
        chunk0, chunk1 = min(nvec, b * world * cell), min(nvec, (b + 1) * world * cell)
        for r in range(world):
            c0 = min(chunk1, chunk0 + r * cell)
            c1 = min(chunk1, c0 + cell)
            own[c0 * epv:c1 * epv] = r
    assert int(own.min()) >= 0, "the cells do not cover the range"
    return own.to(DEV)


def _values(mode, n, gen):
    if mode == "exact":                       # integers: on the bf16 wire every sum of packed values is exact in fp32
        return torch.randint(-8, 9, (n,), generator=gen, device=DEV).float()
    x = torch.randn(n, generator=gen, device=DEV)
    if mode == "spread":                      # magnitudes over 2^-30 .. 2^30: bf16 rounding everywhere
        x = x * torch.exp2(torch.randint(-30, 31, (n,), generator=gen, device=DEV).float())
    return x


def _inv(kind, world):
    """inv_world as the engine passes it: 1/W, 1/(W k') under accumulation of k' = 3 micro-batches,
    1/(2W) for a node group of W ranks in a job of two nodes (hierarchical reduction)."""
    return {"1/W": 1.0 / world, "1/3W": 1.0 / (3 * world), "1/2W": 1.0 / (2 * world)}[kind]


def _bits(t):
    return t.view({2: torch.int16, 4: torch.int32}[t.element_size()])


def _poison(dtype, bits):
    """A one-element poison pattern of ``dtype`` with the given bits."""
    return torch.tensor([bits], dtype={2: torch.int16, 4: torch.int32}[torch.empty((), dtype=dtype).element_size()]) \
        .view(dtype)


def _same_bits(got, want, what):
    assert got.dtype == want.dtype and got.shape == want.shape, (what, got.dtype, want.dtype, got.shape, want.shape)
    bad = _bits(got) != _bits(want)
    n = int(bad.sum())
    if n:
        i = int(bad.nonzero()[0, 0])
        raise AssertionError("%s: %d of %d elements differ; first at %d: got %r, expected %r" %
                             (what, n, got.numel(), i, float(got[i]), float(want[i])))


def _half_ulp(x, fmt):
    """Half a unit in the last place of |x| in ``fmt`` (bf16 or fp32); 0 where x == 0."""
    _, e = torch.frexp(x.double())
    h = torch.exp2((e - (9 if fmt == BF16 else 25)).double())
    return torch.where(x == 0, torch.zeros_like(h), h)


def _some_ranks(world):
    return sorted({0, world // 2, world - 1})


class Group:
    """W emulated ranks on one device: a guarded wire and a guarded signal pad per rank, the pointer
    tables, and one make_comm per rank.  The tables have MAX_WORLD entries (the unused ones repeat
    rank 0), so that no index a kernel could form from a valid comm leaves them."""

    def __init__(self, world, wire_elems, wire_dtype, slots=SLOTS, declared_wire_bytes=None, declared_slots=None):
        C = _C()
        self.world, self.slots = world, slots
        esz = torch.empty((), dtype=wire_dtype).element_size()
        self.wires = [Guarded((wire_elems,), (1,), wire_dtype, 0, _poison(wire_dtype, WIRE_POISON[wire_dtype]), DEV)
                      for _ in range(world)]
        self.words = C.allreduce_signal_words(slots)
        self.pads = [Guarded((self.words,), (1,), torch.int32, 0, PAD_POISON, DEV) for _ in range(world)]
        for p in self.pads:
            p.t.zero_()
        wp = [w.t.data_ptr() for w in self.wires]
        sp = [p.t.data_ptr() for p in self.pads]
        self.wire_tab = torch.tensor(wp + [wp[0]] * (MAX_WORLD - world), dtype=torch.int64, device=DEV)
        self.pad_tab = torch.tensor(sp + [sp[0]] * (MAX_WORLD - world), dtype=torch.int64, device=DEV)
        wb = wire_elems * esz if declared_wire_bytes is None else declared_wire_bytes
        ns = slots if declared_slots is None else declared_slots
        self.comms = [C.make_comm(r, world, self.wire_tab.data_ptr(), self.pad_tab.data_ptr(), 0, 0, wb, ns)
                      for r in range(world)]

    def arm(self, rank, epoch):
        """Peers' pads to 0, the launching rank's whole pad to the epoch; seal every wire and pad.
        Returns the epoch's int32 pattern."""
        e = _i32(epoch)
        for p, pad in enumerate(self.pads):
            pad.t.fill_(e if p == rank else 0)
        for g in self.wires + self.pads:
            g.seal()
        assert bool((self.pads[rank].t == e).all()), "the launching rank's pad must hold the epoch: it would wait"
        return e

    def check_pads(self, rank, slot, e, G, phases=(0, 1)):
        """Every peer pad holds the epoch in [slot, phase, cta < G, src = rank] and 0 elsewhere; the
        launching rank's own pad is still all-epoch; nothing outside any pad changed."""
        for p, pad in enumerate(self.pads):
            if p == rank:
                want = torch.full_like(pad.t, e)
            else:
                want = torch.zeros_like(pad.t)
                w4 = want.view(self.slots, 2, MAX_CTAS, MAX_WORLD)
                for ph in phases:
                    w4[slot, ph, :G, rank] = e
            bad = pad.t != want
            if bool(bad.any()):
                i = int(bad.nonzero()[0, 0])
                sl, ph, cta, src = i // (2 * MAX_CTAS * MAX_WORLD), i // (MAX_CTAS * MAX_WORLD) % 2, \
                    i // MAX_WORLD % MAX_CTAS, i % MAX_WORLD
                raise AssertionError("pad of rank %d after rank %d's launch: %d words wrong, first [slot %d, phase %d, "
                                     "cta %d, src %d] = %d, expected %d" % (p, rank, int(bad.sum()), sl, ph, cta, src,
                                                                          int(pad.t[i]), int(want[i])))
            pad.check([pad.t], "signal pad of rank %d" % p)


def _check_f64(red, packed, world, exact, fmt, what):
    """The emulation itself against the float64 sum of the packed values: within half an ulp of the
    result's format, plus, unless every fp32 sum is exact, the error of world - 1 fp32 additions."""
    s64 = sum(p.double() for p in packed)
    bound = _half_ulp(red.float(), fmt)
    if not exact:
        bound = bound + (world - 1) * 2.0 ** -24 * sum(p.double().abs() for p in packed)
    err = (red.double() - s64).abs()
    assert bool((err <= bound).all()), "%s: the fp32 emulation is off the float64 sum by %g (bound %g)" % (
        what, float((err - bound).max()), float(bound[(err - bound).argmax()]))


def _check_pack(packed, grads, s, fmt, what):
    """bf16(g * s) (or fp32(g * s)) against g * s in float64: within half an ulp, plus the fp32 product's
    rounding that precedes the bf16 one."""
    for p, g in zip(packed, grads):
        x = g.double() * s
        bound = _half_ulp(p.float(), fmt) + (2.0 ** -24 * x.abs() if fmt == BF16 else 0.0)
        assert bool(((p.double() - x).abs() <= bound).all()), what + ": pack emulation"


# ------------------------------------------------------------------------------------- all-reduce
SHAPES = [(8, 0), (8 * 31, 8), (4096, 2056), (65536 + 8, 0), ((1 << 20) + 8 * 5, 2056)]
WORLDS = [1, 2, 3, 4, 5, 8, 16]
CTAS = [0, 1, 3, 16, 48, 128, 200]
INVS = ["1/W", "1/3W", "1/2W"]


def _allreduce_cases():
    cases, k = [], 0
    for algo in ("oneshot", "twoshot"):
        for w32 in (False, True):
            for entry in ("pack", "wire"):
                for n, start in SHAPES:
                    cases.append((algo, w32, entry, WORLDS[k % 7], n, start, CTAS[3 * k % 7], INVS[k % 3],
                                  ("exact", "gauss")[k % 2]))
                    k += 1
    cases += [("twoshot", False, "wire", 8, 65536 + 8, 8, 48, "1/W", "spread"),
              ("twoshot", False, "pack", 3, 4096, 2056, 3, "1/3W", "spread"),
              ("oneshot", False, "pack", 5, 4096, 0, 0, "1/W", "spread")]
    return cases


def _bucket_cases():
    """The engine's real buckets (one per distinct size, at its first start): full VGG-F and the mini
    spec, at the default 32 MB and at 0.25 MB.  At 32 MB these include the 8 Mi-element pieces of the
    FC-1 weight, run at world 8.  Algorithm as the engine picks it without multicast."""
    from distributed_vgg_f_b200.models import layout as L
    from distributed_vgg_f_b200.models.vggf import vggf_mini_spec, vggf_spec
    from distributed_vgg_f_b200.parallel.buckets import engine_bucket_plan
    from distributed_vgg_f_b200.parallel.symm import ONESHOT_MAX_BYTES

    cases, k = [], 0
    for spec in (vggf_spec(1000), vggf_mini_spec(3)):
        for mb in (32.0, 0.25):
            seen = {}
            for b in engine_bucket_plan(L.ready_order(spec), mb).buckets:
                seen.setdefault(b.end - b.start, b.start)
            for n, start in sorted(seen.items(), key=lambda x: x[1]):
                algo = "oneshot" if 2 * n <= ONESHOT_MAX_BYTES else "twoshot"
                world = 8 if n >= (1 << 23) else (2, 4, 8)[k % 3]
                # the FC-1 pieces reach the wire straight from the wgrad epilogue: the wire-only entry
                entry = "wire" if n >= (1 << 23) else "pack" if algo == "oneshot" or k % 2 else "wire"
                cases.append((algo, False, entry, world, n, start, 48, "1/W", "gauss"))
                k += 1
    return cases


BUCKET_CASES = _bucket_cases()


def _ar_id(c):
    algo, w32, entry, W, n, start, ctas, inv, mode = c
    return "%s-%s-%s-W%d-n%d-s%d-c%d-%s-%s" % (algo, "f32" if w32 else "bf16", entry, W, n, start, ctas,
                                               inv.replace("/", ""), mode)


def _run_allreduce(algo, w32, entry, W, n, start, max_ctas, inv_kind, mode, seed):
    C = _C()
    wdt = F32 if w32 else BF16
    epv = 4 if w32 else 8
    G = int(C.allreduce_grid(n, W, max_ctas, w32))
    assert G == _grid(n, W, max_ctas, w32)
    inv = _inv(inv_kind, W)
    s = float(torch.tensor(inv, dtype=F32))             # the kernel's fp32 scale
    s_t = torch.tensor(s, dtype=F32, device=DEV)
    gen = _gen(seed)
    grads = [_values(mode, n, gen) for _ in range(W)]
    packed = [(g * s_t).to(wdt) for g in grads]
    _check_pack(packed, grads, s, wdt, "pack")
    # bf16 packs of integers span few bits: their fp32 sums are exact; fp32 packs of g / 3 are not
    exact_sums = mode == "exact" and not w32
    owner = _owner_map(n, G, W, epv)
    if epv == 8:                                       # the Python mirror the engine uses (ZeRO-1 export)
        for r in range(W):
            mask = torch.zeros(n, dtype=torch.bool, device=DEV)
            for a, b in owned_cells(start, n, G, W, r):
                mask[a - start:b - start] = True
            assert torch.equal(mask, owner == r), "owned_cells disagrees with the kernel's decomposition"
    if algo == "oneshot":                              # peers in order 0 .. W-1, fp32 result
        acc = torch.zeros(n, dtype=F32, device=DEV)
        for p in range(W):
            acc = acc + packed[p].float()
        red = acc
        _check_f64(red, packed, W, exact_sums, F32, "one-shot")
    else:                                              # owner r sums r, r+1, ... mod W, rounds once
        acc = torch.zeros(n, dtype=F32, device=DEV)
        for r in range(W):
            sel = owner == r
            a = torch.zeros(int(sel.sum()), dtype=F32, device=DEV)
            for p in range(W):
                a = a + packed[(r + p) % W][sel].float()
            acc[sel] = a
        red = acc.to(wdt)
        _check_f64(red, packed, W, exact_sums, wdt, "two-shot")

    L = start + n + TAIL
    grp = Group(W, L, wdt)
    rng = slice(start, start + n)
    algo_id = C.AR_ONESHOT if algo == "oneshot" else C.AR_TWOSHOT
    slot = seed % SLOTS
    what = _ar_id((algo, w32, entry, W, n, start, max_ctas, inv_kind, mode))

    def launch(r, grad, gout):
        epoch = _next_epoch()
        e = grp.arm(r, epoch)
        for t in (grad, gout):
            if t is not None:
                t.seal()
        n0 = C.launch_count()
        C.allreduce(grp.comms[r], None if grad is None else grad.t, None if gout is None else gout.t, start, n, inv,
                    algo_id, w32, slot, epoch, max_ctas)
        assert C.launch_count() == n0 + 1
        torch.cuda.synchronize()
        grp.check_pads(r, slot, e, G)
        if grad is not None:
            grad.check((), "%s: grad of rank %d (read-only)" % (what, r))

    def check_wire(p, want, r):
        _same_bits(grp.wires[p].t[rng], want, "%s: wire of rank %d after rank %d's launch" % (what, p, r))
        grp.wires[p].check([grp.wires[p].t[rng]], "%s: wire of rank %d" % (what, p))

    def check_out(gout, want, r):
        if gout is None:
            return
        _same_bits(gout.t[rng], want, "%s: grad_out of rank %d" % (what, r))
        gout.check([gout.t[rng]], "%s: grad_out of rank %d" % (what, r))

    if entry == "wire":                                # the producer already wrote bf16(g * s) on every wire
        for p in range(W):
            grp.wires[p].t[rng] = packed[p]
        for r in range(W) if algo == "twoshot" else _some_ranks(W):
            gout = Guarded((L,), (1,), F32, 0, NAN, DEV) if (algo == "oneshot" or r % 2 == 0) else None
            launch(r, None, gout)
            if algo == "oneshot":                      # the wires are only read
                for p in range(W):
                    check_wire(p, packed[p], r)
                check_out(gout, red, r)
            else:                                      # cells of ranks <= r are reduced on every wire
                done = owner <= r
                for p in range(W):
                    check_wire(p, torch.where(done, red, packed[p]), r)
                check_out(gout, torch.where(done, red, packed[r]).float(), r)
    else:
        for r in _some_ranks(W):
            for p in range(W):
                grp.wires[p].t[rng] = packed[p] if p != r else torch.full_like(packed[p], NAN)
            grad = Guarded((L,), (1,), F32, 0, NAN, DEV)
            grad.t[rng] = grads[r]
            gout = Guarded((L,), (1,), F32, 0, NAN, DEV) if (algo == "oneshot" or r % 2 == 0) else None
            launch(r, grad, gout)
            if algo == "oneshot":
                for p in range(W):
                    check_wire(p, packed[p], r)
                check_out(gout, red, r)
            else:
                mine = owner == r
                for p in range(W):
                    check_wire(p, torch.where(mine, red, packed[p]), r)
                check_out(gout, torch.where(mine, red, packed[r]).float(), r)


ALLREDUCE_CASES = _allreduce_cases()


@pytest.mark.parametrize("case", ALLREDUCE_CASES, ids=[_ar_id(c) for c in ALLREDUCE_CASES])
def test_allreduce_emulated_ranks(case):
    """Every shape edge: one vector, ranges that leave cells of high ranks empty, grids shrunk by
    ``want < G``, 1 and 200 (clamped) CTAs, world 1 .. 16, accumulation and node-group scales."""
    _run_allreduce(*case, seed=ALLREDUCE_CASES.index(case))


@pytest.mark.parametrize("case", BUCKET_CASES, ids=[_ar_id(c) for c in BUCKET_CASES])
def test_allreduce_engine_buckets(case):
    _run_allreduce(*case, seed=1000 + BUCKET_CASES.index(case))


# ---------------------------------------------------------------------------------------- ZeRO-1
HP = dict(lr=R._f32(1e-3), beta1=R._f32(0.9), beta2=R._f32(0.999), eps=R._f32(1e-8), weight_decay=R._f32(0.01))
STEP = 3

ZERO1_CASES = [
    (1, 4096, 0, 0, "1/W", "exact"),
    (2, 8, 8, 1, "1/3W", "gauss"),
    (3, 8 * 31, 2056, 3, "1/W", "gauss"),
    (4, 4096, 0, 16, "1/2W", "exact"),
    (5, 65536 + 8, 8, 48, "1/3W", "gauss"),
    (8, 65536 + 8, 2056, 128, "1/W", "exact"),
    (16, (1 << 20) + 8 * 5, 0, 200, "1/W", "gauss"),
    (16, 4096, 8, 0, "1/3W", "gauss"),
    (3, (1 << 20) + 8 * 5, 2056, 16, "1/W", "spread"),
    # the engine's ZeRO-1 buckets (FC weights only, B200_ZERO1_CTAS = 128): full VGG-F at 32 MB and 0.25 MB,
    # the mini spec at 0.25 MB
    (8, 8388608, 2617344, 128, "1/W", "gauss"),
    (4, 65536, 2048, 128, "1/3W", "gauss"),
    (2, 65536, 24576, 128, "1/W", "gauss"),
]


def _z1_id(c):
    W, n, start, ctas, inv, mode = c
    return "W%d-n%d-s%d-c%d-%s-%s" % (W, n, start, ctas, inv.replace("/", ""), mode)


@pytest.mark.parametrize("case", ZERO1_CASES, ids=[_z1_id(c) for c in ZERO1_CASES])
def test_zero1_step_emulated_ranks(case):
    """Two-shot ZeRO-1: every rank run in turn on the wire-only entry, then single ranks on the pack
    entry.  Rank r's p/m/v change exactly on owned_cells (the ranges prepare_export gathers), there
    bit-identical to adam_fused on the reduced bf16 gradient (the update of the replicated path) and
    within the running bound of a float64 Adam; the gathered master equals replicated Adam; every wire
    ends as bf16(new p); the shadows hold what each rank's wire held when it ran; the pack entry
    zeroes the fp32 gradient range and nothing else."""
    W, n, start, max_ctas, inv_kind, mode = case
    C = _C()
    seed = ZERO1_CASES.index(case)
    G = int(C.allreduce_grid(n, W, max_ctas, False))
    inv = _inv(inv_kind, W)
    s_t = torch.tensor(inv, dtype=F32, device=DEV)
    gen = _gen(500 + seed)
    grads = [_values(mode, n, gen) for _ in range(W)]
    packed = [(g * s_t).to(BF16) for g in grads]
    _check_pack(packed, grads, float(s_t), BF16, "pack")
    owner = torch.full((n,), -1, dtype=torch.int8, device=DEV)
    for r in range(W):
        for a, b in owned_cells(start, n, G, W, r):
            owner[a - start:b - start] = r
    assert int(owner.min()) >= 0
    assert torch.equal(owner, _owner_map(n, G, W, 8))
    acc = torch.zeros(n, dtype=F32, device=DEV)
    for r in range(W):
        sel = owner == r
        a = torch.zeros(int(sel.sum()), dtype=F32, device=DEV)
        for p in range(W):
            a = a + packed[(r + p) % W][sel].float()
        acc[sel] = a
    red = acc.to(BF16)
    _check_f64(red, packed, W, mode == "exact", BF16, "zero1 reduce")

    L = start + n + TAIL
    rng = slice(start, start + n)
    p0 = torch.randn(L, generator=gen, device=DEV)
    m0 = torch.randn(L, generator=gen, device=DEV) * 1e-3
    v0 = torch.randn(L, generator=gen, device=DEV).abs() * 1e-6
    # the replicated path: adam_fused on the reduced bf16 gradient, grad_scale 1
    rp, rm, rv = p0.clone(), m0.clone(), v0.clone()
    rw = torch.empty(L, dtype=BF16, device=DEV)
    C.adam(rp[rng], rm[rng], rv[rng], None, red, rw[rng], HP["lr"], HP["beta1"], HP["beta2"], HP["eps"],
           HP["weight_decay"], STEP, 1.0, None)
    ref64 = R.adam_step64(p0[rng], m0[rng], v0[rng], red, step=STEP, grad_scale=1.0, **HP)
    new16 = rp[rng].to(BF16)

    grp = Group(W, L, BF16)
    state = [[Guarded((L,), (1,), F32, 0, NAN, DEV) for _ in range(3)] for _ in range(W)]
    shadow = [Guarded((L,), (1,), BF16, 0, _poison(BF16, SHADOW_POISON), DEV) for _ in range(W)]
    slot = seed % SLOTS
    what = "zero1 " + _z1_id(case)

    def reset(r):
        for g, x0 in zip(state[r], (p0, m0, v0)):
            g.t.copy_(x0)
        _bits(shadow[r].t).fill_(SHADOW_POISON)

    def launch(r, grad):
        epoch = _next_epoch()
        e = grp.arm(r, epoch)
        for g in state[r] + [shadow[r]] + ([grad] if grad is not None else []):
            g.seal()
        n0 = C.launch_count()
        C.zero1_step(grp.comms[r], None if grad is None else grad.t, *(g.t for g in state[r]), shadow[r].t, start, n,
                     inv, C.AR_TWOSHOT, slot, epoch, max_ctas, HP["lr"], HP["beta1"], HP["beta2"], HP["eps"],
                     HP["weight_decay"], STEP)
        assert C.launch_count() == n0 + 1
        torch.cuda.synchronize()
        grp.check_pads(r, slot, e, G)
        mine = owner == r
        for g, x0, ref, name in zip(state[r], (p0, m0, v0), (rp, rm, rv), "pmv"):
            _same_bits(g.t[rng], torch.where(mine, ref[rng], x0[rng]),
                       "%s: %s of rank %d (owned cells: adam_fused bit for bit; elsewhere untouched)" % (what, name, r))
            g.check([g.t[rng]], "%s: %s of rank %d" % (what, name, r))

    def check_wire(p, want, r):
        _same_bits(grp.wires[p].t[rng], want, "%s: wire of rank %d after rank %d's launch" % (what, p, r))
        grp.wires[p].check([grp.wires[p].t[rng]], "%s: wire of rank %d" % (what, p))

    def check_shadow(r, want):
        _same_bits(shadow[r].t[rng], want, "%s: shadow of rank %d" % (what, r))
        shadow[r].check([shadow[r].t[rng]], "%s: shadow of rank %d" % (what, r))

    # every rank in turn on the wire-only entry: the state of a real step, one rank at a time
    for p in range(W):
        grp.wires[p].t[rng] = packed[p]
        reset(p)
    for r in range(W):
        launch(r, None)
        done = owner <= r
        for p in range(W):
            check_wire(p, torch.where(done, new16, packed[p]), r)
        check_shadow(r, torch.where(done, new16, packed[r]))
    for p in range(W):
        check_wire(p, new16, W - 1)
    # what prepare_export gathers: the owned pieces summed over ranks
    for k, (ref, name) in enumerate(zip((rp, rm, rv), "pmv")):
        gathered = torch.zeros(n, dtype=F32, device=DEV)
        for r in range(W):
            piece = torch.zeros(n, dtype=F32, device=DEV)
            for a, b in owned_cells(start, n, G, W, r):
                piece[a - start:b - start] = state[r][k].t[a:b]
            gathered += piece
        assert torch.equal(gathered, ref[rng]), "%s: gathered %s differs from replicated Adam" % (what, name)
        r64, err = ref64[name]
        KC.check(gathered, r64, torch.zeros_like(r64), chain=0, exact=False, err=err, family="zero1_" + name)
        if name == "p":                                  # the last rank saw every cell final
            _same_bits(shadow[W - 1].t[rng], gathered.to(BF16), "%s: shadow of the last rank" % what)

    # the pack entry, one rank at a time from the initial state
    for r in _some_ranks(W):
        reset(r)
        for p in range(W):
            grp.wires[p].t[rng] = packed[p] if p != r else torch.full_like(packed[p], NAN)
        grad = Guarded((L,), (1,), F32, 0, NAN, DEV)
        grad.t[rng] = grads[r]
        launch(r, grad)
        assert int(torch.count_nonzero(grad.t[rng])) == 0, "%s: the gradient range was not zeroed" % what
        grad.check([grad.t[rng]], "%s: grad of rank %d" % (what, r))
        mine = owner == r
        for p in range(W):
            check_wire(p, torch.where(mine, new16, packed[p]), r)
        check_shadow(r, torch.where(mine, new16, packed[r]))


# ------------------------------------------------------------------------------------- broadcast
BCAST_CASES = [(2, 4, 0), (3, 252, 2), (8, 4096, 3), (16, 65540, 15), (5, (1 << 20) + 20, 1), (1, 4096, 0)]


@pytest.mark.parametrize("W,n,root", BCAST_CASES)
def test_broadcast_emulated_ranks(W, n, root):
    """Root stages its fp32 data in its (bf16) wire, the others pull it: bitwise copies, the root's data
    untouched, nothing written past 4n bytes of the wire or past n elements of any buffer."""
    C = _C()
    grp = Group(W, 2 * n + 16, BF16)
    gen = _gen(W * 1000 + n)
    data = []
    for r in range(W):
        d = Guarded((n,), (1,), F32, 0, NAN, DEV)
        d.t.copy_(torch.randn(n, generator=gen, device=DEV))
        data.append(d)
    want = data[root].t.clone()
    slot = n % SLOTS
    for r in [root] + [r for r in range(W) if r != root]:
        epoch = _next_epoch()
        e = grp.arm(r, epoch)
        data[r].seal()
        n0 = C.launch_count()
        C.broadcast(grp.comms[r], data[r].t, root, slot, epoch)
        assert C.launch_count() == n0 + 1
        torch.cuda.synchronize()
        grp.check_pads(r, slot, e, 32)
        staged = grp.wires[root].t[:2 * n]
        for p in range(W):
            grp.wires[p].check([staged] if p == root == r else [], "broadcast: wire of rank %d" % p)
        assert torch.equal(staged.view(torch.int32), want.view(torch.int32)), "the root's wire is not its data"
        if r == root:
            data[r].check((), "broadcast: the root's data")
        else:
            assert torch.equal(data[r].t.view(torch.int32), want.view(torch.int32)), "rank %d: not the root's data" % r
            data[r].check([data[r].t], "broadcast: data of rank %d" % r)


# --------------------------------------------------------------------------------------- barrier
@pytest.mark.parametrize("W,slot", [(1, 0), (2, 3), (5, 1), (16, 2)])
def test_barrier_writes_only_its_words(W, slot):
    C = _C()
    grp = Group(W, 64, BF16)
    for r in range(W):
        epoch = _next_epoch()
        e = grp.arm(r, epoch)
        C.barrier(grp.comms[r], slot, epoch)
        torch.cuda.synchronize()
        grp.check_pads(r, slot, e, 1, phases=(0,))
        for w in grp.wires:
            w.check((), "barrier: wire")


# ------------------------------------------------------------------------------------- refusals
def _refusals():
    """Argument errors of the collective bindings.  The operands are laid out so that even a launch
    that slipped through would stay inside allocated memory and never wait: the wire and pad are
    larger than declared, every pad holds the epoch, the pointer tables have MAX_WORLD entries and
    every short or misaligned tensor is a view into a larger buffer."""
    C = _C()
    W, N, S = 2, 1024, 2                        # declared: 1024-element bf16 wire, 2 slots
    grp = Group(W, 4 * N, BF16, slots=SLOTS, declared_wire_bytes=2 * N, declared_slots=S)
    epoch = 5
    for p in grp.pads:
        p.t.fill_(epoch)
    comm = grp.comms[0]

    def f(n):
        return torch.zeros(4 * N, device=DEV)[:n]

    def mis(n, dt=F32):
        return torch.zeros(4 * N + 16, dtype=dt, device=DEV)[1:n + 1]

    def ar(grad=None, gout=None, start=0, n=N, w32=False, slot=0, algo=None):
        return lambda: C.allreduce(comm, grad, gout, start, n, 0.5, C.AR_TWOSHOT if algo is None else algo, w32,
                                   slot, epoch, 0)

    def z1(grad=None, p=None, m=None, v=None, sh=None, start=0, n=N, slot=0):
        p, m, v = (f(N) if t is None else t for t in (p, m, v))
        sh = torch.zeros(N, dtype=BF16, device=DEV) if sh is None else sh
        return lambda: C.zero1_step(comm, grad, p, m, v, sh, start, n, 0.5, C.AR_TWOSHOT, slot, epoch, 0,
                                    1e-3, 0.9, 0.999, 1e-8, 0.0, 1)

    def mk(rank, world, slots=S):
        return lambda: C.make_comm(rank, world, grp.wire_tab.data_ptr(), grp.pad_tab.data_ptr(), 0, 0, 2 * N, slots)

    return {
        "make_comm rank >= world": mk(2, 2),
        "make_comm negative rank": mk(-1, 2),
        "make_comm world > 16": mk(0, 17),
        "make_comm no slots": mk(0, 2, 0),
        "allreduce short grad": ar(grad=f(N - 8)),
        "allreduce short grad_out": ar(gout=f(N - 8)),
        "allreduce grad short of start + n": ar(grad=f(N - 8), start=8, n=N - 8),
        "allreduce misaligned grad": ar(grad=mis(N)),
        "allreduce misaligned grad_out": ar(gout=mis(N)),
        "allreduce non-contiguous grad": ar(grad=torch.zeros(2 * N, device=DEV)[::2]),
        "allreduce bf16 grad_out": ar(gout=torch.zeros(N, dtype=BF16, device=DEV)),
        "allreduce CPU grad": ar(grad=torch.zeros(N)),
        "allreduce range past the wire": ar(start=8, n=N),
        "allreduce range past the fp32 wire": ar(n=N // 2 + 8, w32=True),
        "allreduce slot >= slots": ar(slot=S),
        "allreduce negative slot": ar(slot=-1),
        "allreduce one-shot without grad_out": ar(algo=C.AR_ONESHOT),
        "zero1_step short grad": z1(grad=f(N - 8)),
        "zero1_step misaligned grad": z1(grad=mis(N)),
        "zero1_step misaligned p": z1(p=mis(N)),
        "zero1_step misaligned m": z1(m=mis(N)),
        "zero1_step misaligned v": z1(v=mis(N)),
        "zero1_step misaligned shadow": z1(sh=mis(N, BF16)),
        "zero1_step range past the wire": z1(start=0, n=N + 8, p=f(N + 8), m=f(N + 8), v=f(N + 8),
                                             sh=torch.zeros(N + 8, dtype=BF16, device=DEV)),
        "zero1_step slot >= slots": z1(slot=S),
        "broadcast past the wire": lambda: C.broadcast(comm, f(N // 2 + 4), 0, 0, epoch),
        "broadcast root >= world": lambda: C.broadcast(comm, f(64), W, 0, epoch),
        "broadcast negative root": lambda: C.broadcast(comm, f(64), -1, 0, epoch),
        "broadcast misaligned data": lambda: C.broadcast(comm, mis(64), 0, 0, epoch),
        "broadcast slot >= slots": lambda: C.broadcast(comm, f(64), 0, S, epoch),
        "barrier slot >= slots": lambda: C.barrier(comm, S, epoch),
        "barrier negative slot": lambda: C.barrier(comm, -1, epoch),
    }


REFUSALS = ["make_comm rank >= world", "make_comm negative rank", "make_comm world > 16", "make_comm no slots",
            "allreduce short grad", "allreduce short grad_out", "allreduce grad short of start + n",
            "allreduce misaligned grad", "allreduce misaligned grad_out", "allreduce non-contiguous grad",
            "allreduce bf16 grad_out", "allreduce CPU grad", "allreduce range past the wire",
            "allreduce range past the fp32 wire", "allreduce slot >= slots", "allreduce negative slot",
            "allreduce one-shot without grad_out", "zero1_step short grad", "zero1_step misaligned grad",
            "zero1_step misaligned p", "zero1_step misaligned m", "zero1_step misaligned v",
            "zero1_step misaligned shadow", "zero1_step range past the wire", "zero1_step slot >= slots",
            "broadcast past the wire", "broadcast root >= world", "broadcast negative root",
            "broadcast misaligned data", "broadcast slot >= slots", "barrier slot >= slots", "barrier negative slot"]


@pytest.mark.parametrize("case", REFUSALS)
def test_host_refuses_before_launching(case):
    """Each argument check raises, and nothing was launched (the native launch counter is unchanged)."""
    from distributed_vgg_f_b200 import ops
    fns = _refusals()
    assert set(fns) == set(REFUSALS)
    torch.cuda.synchronize()
    n0 = ops.launch_count()
    with pytest.raises(RuntimeError):
        fns[case]()
    torch.cuda.synchronize()
    assert ops.launch_count() == n0
