"""The moving average of the weights (--model-ema) on the GPU: the optimizer kernels' EMA instantiations
against torch's eager fp32 update and a float64 bound, ZeRO-1 on emulated ranks, and the engine's EMA
arena, EMA evaluation pass and launches."""
import os

import pytest
import torch

import test_collectives_gpu as TC
from guarded import NAN, Guarded
from distributed_vgg_f_b200.ops import ref as R
from distributed_vgg_f_b200.parallel.symm import owned_cells

pytestmark = pytest.mark.gpu
DEV = "cuda"
F32, BF16 = torch.float32, torch.bfloat16
ARENA_OFF = 4 * 37              # the optimizer cases of test_elementwise_gpu.py: a slice inside the arena
OPT_N = 4 * 135_173
DECAY = 1.0 - min(1.0, (1.0 - 0.99998) * 64 * 32 / 90)       # the default flags at 64 images x 90 epochs


def _C():
    from distributed_vgg_f_b200 import ops
    return ops.require()


def _bits(t):
    return t.view(torch.int32)


def _same_bits(got, want, what):
    bad = _bits(got) != _bits(want)
    n = int(bad.sum())
    if n:
        i = int(bad.nonzero()[0, 0])
        raise AssertionError("%s: %d of %d elements differ; first at %d: got %r, expected %r" %
                             (what, n, got.numel(), i, float(got[i]), float(want[i])))


def _eager(e, p, decay):
    """torch's eager fp32 ema_avg of torchvision: decay * e + (1 - decay) * p."""
    return decay * e + (1 - decay) * p


# ------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("ema_first", [True, False])
@pytest.mark.parametrize("entry", ["adam-g32", "adam-g16", "sgd-first", "sgd-later"])
def test_optimizer_ema_is_torch_eager_on_the_new_weights(entry, ema_first):
    """The EMA instantiation leaves p / m / v / shadow / gradient bit-identical to the plain launch, and its
    EMA is bit-identical to torch's eager fp32 d*e + a*p on that new p (within ema_step64's float64 bound),
    or a copy of p (including -0.0) over a NaN-poisoned EMA on the first update; nothing outside the slice
    of the guarded EMA changes."""
    C = _C()
    g = torch.Generator(device=DEV).manual_seed(5 + 2 * ["adam-g32", "adam-g16", "sgd-first", "sgd-later"].index(entry)
                                                + ema_first)
    s, e = ARENA_OFF, ARENA_OFF + OPT_N
    tot = e + 64
    p = torch.randn(tot, device=DEV, generator=g)
    m = torch.randn(tot, device=DEV, generator=g) * 1e-3
    v = torch.randn(tot, device=DEV, generator=g).abs() * 1e-6
    g32 = torch.randn(tot, device=DEV, generator=g)
    gb = torch.randn(tot, device=DEV, generator=g).to(BF16)
    # p = -0.0 with a zero gradient and zero moments stays -0.0 through both optimizers
    z = torch.arange(s, e, 997, device=DEV)
    p[z], m[z], v[z], g32[z], gb[z] = -0.0, 0.0, 0.0, 0.0, 0.0
    w16 = p.to(BF16)
    adam = entry.startswith("adam")
    g16 = entry == "adam-g16"
    hp = dict(lr=R._f32(1e-3), beta1=R._f32(0.9), beta2=R._f32(0.999), eps=R._f32(1e-8), wd=R._f32(0.01))

    def launch(state, ema=None):
        P, M, V, G32, W16 = state
        extra = {} if ema is None else dict(ema=ema, ema_decay=DECAY, ema_first=ema_first)
        if adam:
            C.adam(P[s:e], M[s:e], V[s:e], None if g16 else G32[s:e], gb[s:e] if g16 else None, W16[s:e], hp["lr"],
                   hp["beta1"], hp["beta2"], hp["eps"], hp["wd"], 3, 0.125, G32[s:e], **extra)
        else:
            C.sgd(P[s:e], M[s:e], G32[s:e], None, W16[s:e], R._f32(0.01), R._f32(0.9), R._f32(1e-4),
                  entry == "sgd-first", 0.125, G32[s:e], **extra)

    plain = [t.clone() for t in (p, m, v, g32, w16)]
    launch(plain)
    e0 = torch.full((OPT_N,), NAN, device=DEV) if ema_first else torch.randn(OPT_N, device=DEV, generator=g)
    ema = Guarded((OPT_N,), (1,), F32, ARENA_OFF, NAN, DEV)
    ema.t.copy_(e0)
    ema.seal()
    fused = [t.clone() for t in (p, m, v, g32, w16)]
    launch(fused, ema.t)
    torch.cuda.synchronize()
    for a, b, name in zip(fused, plain, ("p", "m", "v", "g32", "shadow")):
        if a.dtype == F32:
            _same_bits(a, b, "%s: %s with the EMA on" % (entry, name))
        else:
            assert torch.equal(a.view(torch.int16), b.view(torch.int16)), "%s: %s with the EMA on" % (entry, name)
    ema.check([ema.t], entry + ": ema")
    p_new = plain[0][s:e]
    assert bool((_bits(p_new[z - s]) == _bits(torch.tensor(-0.0, device=DEV))).all()), "the -0.0 weights moved"
    if ema_first:
        _same_bits(ema.t, p_new, entry + ": first EMA update is a copy of p")
        return
    _same_bits(ema.t, _eager(e0, p_new, DECAY), entry + ": EMA against torch's eager fp32 update")
    ref, err = R.ema_step64(e0, p_new, decay=DECAY, first=False)
    assert bool(((ema.t.double() - ref).abs() <= err).all()), entry + ": EMA outside the float64 bound"


def test_host_refuses_bad_ema_operands():
    C = _C()
    z = lambda n, dt=F32: torch.zeros(n, dtype=dt, device=DEV)      # noqa: E731
    base = (z(64), z(64), z(64), z(64), None, None, 1e-3, 0.9, 0.999, 1e-8, 0.0, 1, 1.0, None)
    bad = {"short": dict(ema=z(60)), "dtype": dict(ema=z(64, BF16)), "misaligned": dict(ema=z(65)[1:]),
           "decay": dict(ema=z(64), ema_decay=1.5)}
    for name, kw in bad.items():
        n0 = C.launch_count()
        with pytest.raises(RuntimeError):
            C.adam(*base, **kw)
        with pytest.raises(RuntimeError):
            C.sgd(z(64), z(64), z(64), None, None, 0.1, 0.9, 0.0, True, 1.0, None, **kw)
        assert C.launch_count() == n0, name


# ---------------------------------------------------------------------------------- ZeRO-1, emulated ranks
Z1_CASES = [(1, 4096, 0, 0, True), (2, 8 * 31, 8, 1, False), (3, 65536 + 8, 2056, 16, True),
            (4, 4096, 0, 16, False), (5, 65536 + 8, 8, 48, False), (8, 65536, 2048, 128, True),
            (16, (1 << 20) + 8 * 5, 0, 200, False)]


@pytest.mark.parametrize("case", Z1_CASES, ids=["W%d-n%d-s%d-c%d-%s" % (c[0], c[1], c[2], c[3], "first" if c[4] else "later")
                                                for c in Z1_CASES])
def test_zero1_ema_on_emulated_ranks(case):
    """Two-shot ZeRO-1 with the EMA, every rank in turn on the wire-only entry: on the cells a rank owns
    its EMA is bit-identical to adam with the EMA on the reduced bf16 gradient, elsewhere (and outside
    the range) untouched; the owned pieces summed over ranks are the replicated EMA."""
    W, n, start, max_ctas, first = case
    C = _C()
    seed = Z1_CASES.index(case)
    G = int(C.allreduce_grid(n, W, max_ctas, False))
    gen = torch.Generator(device=DEV).manual_seed(900 + seed)
    inv = 1.0 / W
    packed = [(TC._values("gauss", n, gen) * torch.tensor(inv, device=DEV)).to(BF16) for _ in range(W)]
    owner = torch.full((n,), -1, dtype=torch.int8, device=DEV)
    for r in range(W):
        for a, b in owned_cells(start, n, G, W, r):
            owner[a - start:b - start] = r
    assert int(owner.min()) >= 0
    acc = torch.zeros(n, dtype=F32, device=DEV)
    for r in range(W):
        sel = owner == r
        a = torch.zeros(int(sel.sum()), dtype=F32, device=DEV)
        for q in range(W):
            a = a + packed[(r + q) % W][sel].float()
        acc[sel] = a
    red = acc.to(BF16)

    L = start + n + TC.TAIL
    rng = slice(start, start + n)
    p0 = torch.randn(L, generator=gen, device=DEV)
    m0 = torch.randn(L, generator=gen, device=DEV) * 1e-3
    v0 = torch.randn(L, generator=gen, device=DEV).abs() * 1e-6
    e0 = torch.full((L,), NAN, device=DEV) if first else torch.randn(L, generator=gen, device=DEV)
    HP = TC.HP
    rp, rm, rv, re = p0.clone(), m0.clone(), v0.clone(), e0.clone()
    rw = torch.empty(L, dtype=BF16, device=DEV)
    C.adam(rp[rng], rm[rng], rv[rng], None, red, rw[rng], HP["lr"], HP["beta1"], HP["beta2"], HP["eps"],
           HP["weight_decay"], TC.STEP, 1.0, None, ema=re[rng], ema_decay=DECAY, ema_first=first)
    if not first:
        _same_bits(re[rng], _eager(e0[rng], rp[rng], DECAY), "replicated EMA against torch's eager update")

    grp = TC.Group(W, L, BF16)
    state = [[Guarded((L,), (1,), F32, 0, NAN, DEV) for _ in range(4)] for _ in range(W)]
    shadow = [Guarded((L,), (1,), BF16, 0, TC._poison(BF16, TC.SHADOW_POISON), DEV) for _ in range(W)]
    slot = seed % TC.SLOTS
    for q in range(W):
        grp.wires[q].t[rng] = packed[q]
        for gd, x0 in zip(state[q], (p0, m0, v0, e0)):
            gd.t.copy_(x0)
    for r in range(W):
        epoch = TC._next_epoch()
        grp.arm(r, epoch)
        for gd in state[r]:
            gd.seal()
        n0 = C.launch_count()
        C.zero1_step(grp.comms[r], None, *(gd.t for gd in state[r][:3]), shadow[r].t, start, n, inv, C.AR_TWOSHOT,
                     slot, epoch, max_ctas, HP["lr"], HP["beta1"], HP["beta2"], HP["eps"], HP["weight_decay"],
                     TC.STEP, ema=state[r][3].t, ema_decay=DECAY, ema_first=first)
        assert C.launch_count() == n0 + 1
        torch.cuda.synchronize()
        mine = owner == r
        for gd, x0, ref, name in zip(state[r], (p0, m0, v0, e0), (rp, rm, rv, re), ("p", "m", "v", "ema")):
            _same_bits(gd.t[rng], torch.where(mine, ref[rng], x0[rng]),
                       "W%d: %s of rank %d (owned cells: adam bit for bit; elsewhere untouched)" % (W, name, r))
            gd.check([gd.t[rng]], "W%d: %s of rank %d" % (W, name, r))
    gathered = torch.zeros(n, dtype=F32, device=DEV)
    for r in range(W):
        piece = torch.zeros(n, dtype=F32, device=DEV)
        for a, b in owned_cells(start, n, G, W, r):
            piece[a - start:b - start] = state[r][3].t[a:b]
        gathered += piece
    _same_bits(gathered, re[rng], "W%d: gathered EMA against the replicated EMA" % W)


# ------------------------------------------------------------------------------------------- engine
def _engine(classes=3, optimizer="adam", batch=4, **kw):
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine
    from distributed_vgg_f_b200.models.vggf import build_oracle, vggf_mini_spec

    spec = vggf_mini_spec(classes)
    init = kw.pop("init_state", None) or build_oracle(spec, seed=0).state_dict()
    return NativeEngine(spec, device=torch.device(DEV), batch=batch, lr=1e-3, seed=0, input_hw=64,
                        optimizer=optimizer, weight_decay=1e-4, init_state=init, **kw)


def _batch(b=4, seed=3, classes=3, hw=128):
    from distributed_vgg_f_b200.data import transforms as T
    from distributed_vgg_f_b200.data.loader import FusedBatch

    g = torch.Generator().manual_seed(seed)
    src = torch.randint(0, 256, (b, hw, hw, 3), dtype=torch.uint8, generator=g)
    params = T.sample_train_params(b, hw, hw, g)
    y = torch.randint(0, classes, (b,), generator=g)
    return FusedBatch(src, params, y, (80, 80), None)


def _run_and_emulate(eng, decay, schedule, batches):
    """Train with the EMA on the steps of ``schedule``; after each EMA update the EMA arena must be,
    bit for bit, torch's eager fp32 update applied to a snapshot of the fp32 weights."""
    emu, n = None, 0
    for k, ema in enumerate(schedule):
        eng.train_step(batches[k % len(batches)], ema=ema)
        eng.sync()
        if ema:
            p = eng.p32.clone()
            emu = p if n == 0 else _eager(emu, p, decay)
            n += 1
            _same_bits(eng.ema32, emu, "EMA after update %d" % k)
    assert eng.ema_updates == n
    return emu


@pytest.mark.parametrize("steps", [1, 3])
@pytest.mark.parametrize("optimizer,classes", [("adam", 3), ("sgd", 3), ("adam", 10), ("sgd", 10)])
def test_engine_ema_is_the_eager_update_of_the_weights(optimizer, classes, steps):
    decay = 0.75
    eng = _engine(classes, optimizer, ema_decay=decay)
    assert eng.fused_head == (classes <= 8)
    eng.train_dropout = False
    batches = [_batch(4, seed=s, classes=classes) for s in range(3)]
    _run_and_emulate(eng, decay, [u % steps == 0 for u in range(7)], batches)


@pytest.mark.parametrize("classes", [3, 10])
def test_ema_evaluation_reads_the_ema_weights(classes):
    """The EMA pass reads ema16 weights and ema32 biases.  Its weights are bit-identical to the w16 of a
    second engine that imported export_ema_state(), and its logits and meter match that engine's plain
    pass up to the run-to-run order of the FC forward's fp32 split-K adds (a different order can flip a
    bf16 rounding of an FC output, so logits are not compared bit for bit); they differ from the raw
    weights' pass."""
    from distributed_vgg_f_b200.utils.metrics import DeviceMeter

    eng = _engine(classes, ema_decay=0.5)
    eng.train_dropout = False
    eng.lr = 1e-2                        # weights far from their average: the two passes differ clearly
    for k in range(4):
        eng.train_step(_batch(4, seed=k, classes=classes), ema=True)
    with pytest.raises(RuntimeError, match="prepare_ema"):
        eng.eval_step(_batch(4, classes=classes), ema=True)
    eng.prepare_ema()
    twin = _engine(classes, init_state=eng.export_ema_state())
    assert torch.equal(eng.ema16.view(torch.int16), twin.w16.view(torch.int16))
    batch = _batch(4, seed=11, classes=classes)
    results = []
    for e, kw in ((eng, {"ema": True}), (twin, {}), (eng, {})):
        meter = DeviceMeter(DEV)
        e.set_meter(meter)
        e.eval_step(batch, **kw)
        logits = e.forward_logits(batch, **kw)
        e.sync()
        loss, acc = meter.snapshot()
        results.append((logits, loss.average, acc.correct))
    (la, lsa, _), (lb, lsb, _), (lraw, _, _) = results
    scale = float(lb.abs().max())
    assert float((la - lb).abs().max()) <= 1e-2 * scale and abs(lsa - lsb) <= 1e-2 * abs(lsb)
    assert float((la - lraw).abs().max()) > 1e-1 * scale, "the EMA pass computed with the raw weights"
    assert eng._wsrc is eng.w16 and eng._bsrc is eng.p32


class _Recorder:
    """Stands in for ops._C and records every native call (tensors by shape and dtype)."""

    def __init__(self, C):
        self._C, self.calls = C, []

    def __getattr__(self, name):
        f = getattr(self._C, name)
        if not callable(f) or name == "launch_count":
            return f

        def call(*a, **k):
            self.calls.append((name, _sig(a), _sig(sorted(k.items()))))
            return f(*a, **k)
        return call


def _sig(v):
    if isinstance(v, torch.Tensor):
        return ("tensor", tuple(v.shape), str(v.dtype))
    if isinstance(v, (list, tuple)):
        return tuple(_sig(x) for x in v)
    return v


@pytest.mark.parametrize("optimizer", ["adam", "sgd"])
def test_steps_without_an_ema_update_run_the_calls_of_an_engine_without_the_argument(optimizer, monkeypatch):
    """Over a gradient-only step and two update steps, an engine without ema_decay, one with
    ema_decay=None and one with the EMA on (but not updated on these steps) make the same native calls
    with the same arguments and the same launch counts.  A fourth step that updates the EMA makes the
    calls of the fourth step without it, each optimizer call with the EMA range, decay and first flag
    appended, and the same number of launches."""
    from distributed_vgg_f_b200 import ops

    batch = _batch(4)
    runs, fourth = [], []
    for kw in ({}, {"ema_decay": None}, {"ema_decay": 0.9}):
        rec = _Recorder(ops.require())
        monkeypatch.setattr(ops, "_C", rec)
        eng = _engine(3, optimizer, **kw)
        eng.train_dropout = False
        counts = []
        for k in range(3):
            eng.apply_updates = k > 0
            n0 = ops.launch_count()
            eng.train_step(batch)
            eng.sync()
            counts.append(ops.launch_count() - n0)
        runs.append((list(rec.calls), counts))
        del rec.calls[:]
        n0 = ops.launch_count()
        eng.train_step(batch, ema=bool(kw.get("ema_decay")))
        eng.sync()
        fourth.append((list(rec.calls), ops.launch_count() - n0))
        monkeypatch.undo()
        if kw.get("ema_decay"):
            assert eng.ema_updates == 1
    assert runs[0] == runs[1] == runs[2]
    assert fourth[0] == fourth[1]
    (with_ema, n_ema), (without, n_plain) = fourth[2], fourth[0]
    assert n_ema == n_plain and len(with_ema) == len(without)
    n_opt = 0
    for a, b in zip(with_ema, without):
        if a[0] in ("adam", "sgd"):
            n_opt += 1
            assert a[0] == b[0] and a[1][:len(b[1])] == b[1] and len(a[1]) == len(b[1]) + 3
            assert a[1][-2:] == (0.9, True) and a[1][-3][0] == "tensor"      # the first EMA update
        else:
            assert a == b
    assert n_opt == len(_engine(3, optimizer).plan.buckets)


@pytest.mark.skipif(os.environ.get("B200_SKIP_SLOW", "0") == "1", reason="B200_SKIP_SLOW=1")
def test_full_vggf_ema_every_step():
    """VGG-F at 224^2 and batch 64 with the EMA updated on every step: bit-exact against the eager update
    of the weights' snapshots."""
    from distributed_vgg_f_b200.data import transforms as T
    from distributed_vgg_f_b200.data.loader import FusedBatch
    from distributed_vgg_f_b200.data.synthetic import synthetic_uint8_batch
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine
    from distributed_vgg_f_b200.models.vggf import vggf_spec

    eng = NativeEngine(vggf_spec(3), device=torch.device(DEV), batch=64, lr=1e-4, seed=0, ema_decay=DECAY)
    batches = []
    for s in range(2):
        imgs, labels = synthetic_uint8_batch(64, 128, 3, seed=s)
        batches.append(FusedBatch(torch.from_numpy(imgs).pin_memory(), T.sample_train_params(64, 128, 128).pin_memory(),
                                  torch.from_numpy(labels).pin_memory(), (256, 256), None))
    emu = _run_and_emulate(eng, DECAY, [True] * 3, batches)
    assert not torch.equal(emu, eng.p32), "the EMA is the weights: vacuous"


# ---------------------------------------------------------------------------------------- 2 GPUs
def _zero1_ema_worker(rank, world):
    import torch.distributed as dist

    from distributed_vgg_f_b200.engine.native_engine import NativeEngine
    from distributed_vgg_f_b200.models.vggf import build_oracle, vggf_mini_spec

    dev = torch.device("cuda", rank)
    spec = vggf_mini_spec(3)
    init = build_oracle(spec, seed=0).state_dict()
    kw = dict(device=dev, batch=4, lr=5e-2, seed=0, input_hw=64, init_state=init, allreduce="twoshot",
              bucket_mb=0.25, ema_decay=0.5)
    ref = NativeEngine(spec, **dict(kw, zero1=False))
    z = NativeEngine(spec, **dict(kw, zero1=True))
    assert z.zero1
    for e in (ref, z):
        e.train_dropout = False
        e.eps = 1.0                      # smooth in g: see test_multigpu.py::_zero1_worker
    g = torch.Generator().manual_seed(7 + rank)
    for k in range(3):
        x = torch.randn(4, 3, 64, 64, generator=g).to(torch.bfloat16).float()
        y = torch.randint(0, 3, (4,), generator=g)
        for e in (ref, z):
            e.train_step((x, y), ema=True)
            e.sync()
            dist.barrier()
    assert z._zero1_buckets
    z.prepare_ema()
    for bi, bk in enumerate(z.plan.buckets):
        a, b = z.ema32[bk.start:bk.end], ref.ema32[bk.start:bk.end]
        r = float((a - b).norm() / (b.norm() + 1e-30))
        assert r < 2e-2, "EMA of bucket %d (zero1=%s) differs: rel %g" % (bi, bi in z._zero1_buckets, r)
    e = z.ema32.clone()
    dist.broadcast(e, src=0)
    assert torch.equal(e, z.ema32), "the gathered EMA differs between ranks"


@pytest.mark.multigpu
def test_zero1_ema_matches_replicated_adam_on_two_gpus():
    import test_multigpu as MG

    MG._run(_zero1_ema_worker, 2)
