"""PowerSGD on the sm_90a engine: the four kernels of csrc/powersgd.cu against float64 torch at the shapes VGG-F
compresses (on guarded operands, launched twice), emulated ranks against the hook's arithmetic, and the engine
at world 1 against the hook applied in float64 to the pre-exchange gradient of a deterministic twin."""
import pytest
import torch

import test_deterministic_gpu as TD
from guarded import NAN, Guarded

pytestmark = pytest.mark.gpu
DEV = "cuda"
F32, F64 = torch.float32, torch.float64

# (what, n, m): FC-1, FC-2, classifier.6.0, a 512 x (3*3*512) OHWI convolution, conv0 padded to 64 columns
SHAPES = [("fc1", 4096, 25088), ("fc2", 4096, 4096), ("head", 512, 4096), ("conv", 512, 4608), ("conv0", 64, 64)]
RANKS = [1, 2, 4, 8]


def _ops():
    from distributed_vgg_f_b200 import ops
    ops.require()
    return ops


def orth64(x: torch.Tensor) -> torch.Tensor:
    """torch's _orthogonalize_gram_schmidt in float64, a zero column left at zero."""
    x = x.to(F64).clone()
    for i in range(x.shape[1]):
        nrm = x[:, i].norm()
        x[:, i] = x[:, i] / nrm if nrm > 0 else 0.0
        if i + 1 < x.shape[1]:
            x[:, i + 1:] -= (x[:, i:i + 1] * x[:, i + 1:]).sum(0, keepdim=True) * x[:, i:i + 1]
    return x


def hook64(Ms, q):
    """The hook's compressed update over ranks in float64: Ms = [M_w] (n x m), q the warm-start Q.
    Returns (orth Q, P, Q = sum M^T P / W, G = P Q^T)."""
    q0 = orth64(q)
    p = orth64(sum(M.to(F64) @ q0 for M in Ms))
    qn = sum(M.to(F64).t() @ p for M in Ms) / len(Ms)
    return q0, p, qn, p @ qn.t()


def rel(a, b, scale=None):
    a, b = a.to(F64), b.to(F64)
    s = (scale if scale is not None else b).to(F64).norm()
    return float((a - b).norm() / s) if s > 0 else float((a - b).norm())


def _operands(n, m, r, seed, padded=False):
    g = torch.Generator(device=DEV).manual_seed(seed)
    grad = torch.randn(n, m, device=DEV, generator=g) * 1e-3
    err = torch.randn(n, m, device=DEV, generator=g) * 1e-4
    q = torch.randn(m, r, device=DEV, generator=g)
    if padded:                           # conv0: 27 real columns, zero gradient / error / Q rows at the padding
        grad[:, 27:] = 0
        err[:, 27:] = 0
        q[27:] = 0
    return grad, err, q


def _guard(values, offset=0, poison=NAN):
    t = Guarded(tuple(values.shape), tuple(values.stride()), values.dtype, offset, poison, DEV)
    t.t.copy_(values)
    t.seal()
    return t


@pytest.mark.parametrize("rank", RANKS)
@pytest.mark.parametrize("what,n,m", SHAPES)
def test_kernels_against_float64_on_guarded_operands(what, n, m, rank):
    ops = _ops()
    C = ops.require()
    r = min(n, m, rank)
    grad, err, q_in = _operands(n, m, r, seed=n * 31 + m + r, padded=what == "conv0")
    s = 0.5                               # the mean of a two-batch group
    M_want = grad * s + err               # fp32, one rounding per operation: the kernel's arithmetic exactly

    results = []
    for _ in range(2):                    # a second run on fresh copies: bit-identical results
        q = _guard(q_in)
        ops.psgd_orthogonalize(q.t, rows=m, rank=r)
        g, e = _guard(grad), _guard(err)
        p = _guard(torch.full((n, r), NAN, device=DEV))
        ops.psgd_project(g.t, e.t, q.t, p.t, n=n, m=m, rank=r, scale=s)
        p_proj = p.t.clone()
        ops.psgd_orthogonalize(p.t, rows=n, rank=r)
        ws = _guard(torch.full((ops.psgd_workspace_elems(n, m, r),), NAN, device=DEV))
        q2 = _guard(torch.full((m, r), NAN, device=DEV))
        ops.psgd_backproject(e.t, p.t, q2.t, ws.t, n=n, m=m, rank=r)
        q_back = q2.t.clone()
        M_got = e.t.clone()
        ops.psgd_decompress(p.t, q2.t, g.t, e.t, n=n, m=m, rank=r, alpha=1.0)
        torch.cuda.synchronize()
        for t, w, name in ((q, [q.t], "q"), (g, [g.t], "g"), (e, [e.t], "e"), (p, [p.t], "p"), (ws, [ws.t], "ws"),
                           (q2, [q2.t], "q2")):
            t.check(w, "%s %s r=%d" % (name, what, r))
        results.append((q.t.clone(), p_proj, p.t.clone(), q_back, M_got, g.t.clone(), e.t.clone()))
    for a, b in zip(*results):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), what

    q0, p_proj, p, q_back, M_got, G, e_new = results[0]
    assert torch.equal(M_got, M_want)
    q0_64 = orth64(q_in)
    assert rel(q0, q0_64) < 1e-5
    eye = torch.eye(r, device=DEV, dtype=F64)
    assert (q0.to(F64).t() @ q0.to(F64) - eye).abs().max() < 1e-5
    assert rel(p_proj, M_want.to(F64) @ q0.to(F64)) < 1e-5
    assert rel(p, orth64(p_proj)) < 1e-4
    assert (p.to(F64).t() @ p.to(F64) - eye).abs().max() < 1e-5
    assert rel(q_back, M_want.to(F64).t() @ p.to(F64)) < 1e-5
    G64 = p.to(F64) @ q_back.to(F64).t()
    assert rel(G, G64) < 1e-5
    assert rel(e_new, M_want.to(F64) - G64, scale=M_want) < 1e-5
    assert not torch.isnan(G).any() and not torch.isnan(e_new).any()
    if what == "conv0":
        assert not q_back[27:].any() and not G[:, 27:].any() and not e_new[:, 27:].any()


@pytest.mark.parametrize("rank", RANKS)
def test_zero_gradient_gives_zeros_not_nan(rank):
    ops = _ops()
    n, m = 512, 4608
    g = torch.zeros(n, m, device=DEV)
    e = torch.zeros(n, m, device=DEV)
    q = torch.randn(m, rank, device=DEV)
    p = torch.full((n, rank), NAN, device=DEV)
    ws = torch.empty(ops.psgd_workspace_elems(n, m, rank), device=DEV)
    ops.psgd_orthogonalize(q, rows=m, rank=rank)
    ops.psgd_project(g, e, q, p, n=n, m=m, rank=rank)
    ops.psgd_orthogonalize(p, rows=n, rank=rank)
    ops.psgd_backproject(e, p, q, ws, n=n, m=m, rank=rank)
    ops.psgd_orthogonalize(q, rows=m, rank=rank)
    ops.psgd_decompress(p, q, g, e, n=n, m=m, rank=rank)
    torch.cuda.synchronize()
    for t in (p, q, g, e):
        assert not torch.isnan(t).any() and not t.any()


def test_host_checks_refuse_before_launching():
    ops = _ops()
    C = ops.require()
    z = lambda k: torch.zeros(k, device=DEV)       # noqa: E731
    n0 = C.launch_count()
    with pytest.raises(RuntimeError, match="register budget|40-register"):
        ops.psgd_project(z(64), z(64), z(72), z(72), n=8, m=8, rank=9)
    with pytest.raises(RuntimeError, match="multiple of 4"):
        ops.psgd_project(z(60), z(60), z(12), z(12), n=6, m=10, rank=1)
    with pytest.raises(RuntimeError, match="must hold"):
        ops.psgd_decompress(z(8), z(8), z(63), z(64), n=8, m=8, rank=1)
    with pytest.raises(RuntimeError, match="aligned"):
        ops.psgd_orthogonalize(z(65)[1:], rows=32, rank=2)
    with pytest.raises(RuntimeError, match="workspace"):
        ops.psgd_backproject(z(4096 * 512), z(4096), z(512), z(4), n=4096, m=512, rank=1)
    assert C.launch_count() == n0


@pytest.mark.parametrize("world", [2, 4, 8])
def test_emulated_ranks_match_the_hooks_arithmetic(world):
    """Each rank's project and back-project, the all-reduces summed here; against the hook per rank in float64."""
    ops = _ops()
    n, m, r = 512, 4608, 4
    ranks = [_operands(n, m, r, seed=100 * world + w) for w in range(world)]
    q = ranks[0][2].clone()
    q_in = q.clone()
    ops.psgd_orthogonalize(q, rows=m, rank=r)
    Ms, ps = [], []
    for grad, err, _ in ranks:
        e = err.clone()
        p = torch.empty(n, r, device=DEV)
        ops.psgd_project(grad.clone(), e, q, p, n=n, m=m, rank=r)
        Ms.append(e)
        ps.append(p)
    P = sum(ps)
    ops.psgd_orthogonalize(P, rows=n, rank=r)
    ws = torch.empty(ops.psgd_workspace_elems(n, m, r), device=DEV)
    qs = []
    for M in Ms:
        qw = torch.empty(m, r, device=DEV)
        ops.psgd_backproject(M, P, qw, ws, n=n, m=m, rank=r)
        torch.cuda.synchronize()
        qs.append(qw)
    Q = sum(qs)
    q0, p64, q64, G64 = hook64([grad + err for grad, err, _ in ranks], q_in)
    assert rel(P, p64) < 1e-4
    assert rel(Q / world, q64) < 1e-4
    for M in Ms:
        g = torch.empty(n, m, device=DEV)
        e = M.clone()
        ops.psgd_decompress(P, Q, g, e, n=n, m=m, rank=r, alpha=1.0 / world)
        torch.cuda.synchronize()
        assert rel(g, G64) < 1e-4
        assert rel(e, M.to(F64) - G64, scale=M) < 1e-4


# ------------------------------------------------------------------------------------------- the engine
S = 2
# Gradients with at least r significant directions, so that the float64 hook is a fair yardstick for every compressed
# tensor: 16 samples and 8 classes.  With fewer samples than r, or 3 classes (the logits' gradient rows sum to zero:
# rank <= 2 behind the head), the head's gradients have fewer than r directions and the last columns of P are
# rounding noise in any fp32 Gram-Schmidt.
B = 16
CLASSES = 8


def _engine(**kw):
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine
    from distributed_vgg_f_b200.models.vggf import build_oracle, vggf_mini_spec

    spec = vggf_mini_spec(CLASSES)
    eng = NativeEngine(spec, device=torch.device(DEV), batch=B, lr=1e-3, seed=5, input_hw=64, distributed=False,
                       init_state=build_oracle(spec, seed=1).state_dict(), deterministic=True, **kw)
    eng.train_dropout = False
    return eng


@pytest.mark.parametrize("optimizer,freeze,accum,rank", [("adam", 0, 1, 4), ("sgd", 0, 1, 2), ("adam", 4, 1, 4),
                                                         ("adam", 0, 2, 4)])
def test_engine_matches_the_hook_on_the_twins_gradient(monkeypatch, optimizer, freeze, accum, rank):
    from distributed_vgg_f_b200.parallel import powersgd

    ops = _ops()
    eng = _engine(optimizer=optimizer, freeze_layers=freeze, powersgd_rank=rank, powersgd_start_iter=S)
    plain = _engine(optimizer=optimizer, freeze_layers=freeze)
    twin = _engine(optimizer=optimizer, freeze_layers=freeze)
    twin.apply_updates = False
    assert eng._psgd and all(n not in eng._frozen for n in eng._psgd)
    seen = {}
    real = ops.psgd_decompress

    def record(p, q, g, e, **kw):
        real(p, q, g, e, **kw)
        seen[g.data_ptr()] = g.clone()           # on the comm stream, right behind the launch
    monkeypatch.setattr(ops, "psgd_decompress", record)
    projected = {}
    real_project = ops.psgd_project

    def record_project(g, e, q, p, **kw):
        real_project(g, e, q, p, **kw)
        projected[g.data_ptr()] = (q.clone(), p.clone())     # the orthogonalised warm start and P = M Q
    monkeypatch.setattr(ops, "psgd_project", record_project)
    updates = S + 3
    batches = TD._batches(updates * accum, B, CLASSES, hw=128, mix=False)
    for u in range(1, updates + 1):
        group = batches[(u - 1) * accum:u * accum]
        if u > S:
            eng.sync()
            e_prev, q_prev = eng._psgd_e.clone(), eng._psgd_q.clone()
            twin.import_state(eng.export_state())
            twin.g32.zero_()
            for k, b in enumerate(group):
                twin.train_step(b, update=k == accum - 1)
            twin.sync()
        seen.clear()
        for k, b in enumerate(group):
            eng.train_step(b, update=k == accum - 1)
            if u <= S:
                plain.train_step(b, update=k == accum - 1)
        eng.sync()
        if u <= S:
            plain.sync()
            assert not seen
            assert torch.equal(eng.p32, plain.p32) and torch.equal(eng.m32, plain.m32), u
            continue
        assert len(seen) == len(eng._psgd)
        first = powersgd.initial_q_torch(eng._psgd_rows, eng.seed) if u == S + 1 else None
        for name, (n, m, r, eo, po, qo) in eng._psgd.items():
            g = twin._view(twin.g32, name).reshape(n, m)
            M = g * (1.0 / accum) + e_prev[eo:eo + n * m].view(n, m)
            q0 = powersgd.q_to_native(eng.spec, name, first[name]).to(DEV) if first else \
                q_prev[qo:qo + m * r].view(m, r)
            G = seen[eng._view(eng.g32, name).data_ptr()].view(n, m)
            P = eng._psgd_p[po:po + n * r].view(n, r).to(F64)
            Q = eng._psgd_q[qo:qo + m * r].view(m, r).to(F64)
            e = eng._psgd_e[eo:eo + n * m].view(n, m)
            what = "%s update %d" % (name, u)
            # every stage on the engine's own operands: the warm start, P = M Q, Q = M^T P, G = P Q^T, e = M - G
            q_used, p_proj = projected[eng._view(eng.g32, name).data_ptr()]
            q_used, p_proj = q_used.view(m, r), p_proj.view(n, r)
            assert (q_used.to(F64).t() @ q_used.to(F64) - torch.eye(r, device=DEV, dtype=F64)).abs().max() < 1e-4, what
            assert rel(q_used, orth64(q0)) < 1e-4, what
            assert rel(p_proj, M.to(F64) @ q_used.to(F64)) < 1e-5, what
            MQ = M.to(F64) @ orth64(q0)
            assert rel(Q, M.to(F64).t() @ P) < 1e-5, what
            assert rel(G, P @ Q.t(), scale=M) < 1e-5, what
            assert rel(e, M.to(F64) - G.to(F64), scale=M) < 1e-6, what
            # and the hook's whole update in float64, for every compressed tensor: P spans M orth(Q0), G, e and Q are
            # the hook's
            assert rel(P @ (P.t() @ MQ), MQ) < 1e-3, what
            _, _, q64, G64 = hook64([M], q0)
            assert rel(G, G64, scale=M) < 1e-3, what
            assert rel(e, M.to(F64) - G64, scale=M) < 1e-3, what
            assert rel(Q, q64) < 1e-3, what
        assert not torch.equal(eng.p32, plain.p32)
    assert eng.export_optimizer_state()["powersgd"] == {"rank": rank, "start_iter": S}


def test_rank_zero_makes_the_calls_of_an_engine_without_the_argument(monkeypatch):
    import test_ema_gpu as TE

    ops = _ops()
    runs = []
    for kw in ({}, {"powersgd_rank": 0}):
        rec = TE._Recorder(ops.require())
        monkeypatch.setattr(ops, "_C", rec)
        eng = TE._engine(3, "adam", **kw)
        eng.train_dropout = False
        for k in range(3):
            eng.train_step(TE._batch(4), update=k != 0)
        eng.sync()
        monkeypatch.undo()
        runs.append(list(rec.calls))
    assert runs[0] == runs[1]
    assert not any(c[0].startswith("psgd") for c in runs[0])
