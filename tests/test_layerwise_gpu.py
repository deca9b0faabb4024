"""LAMB and LARS on the GPU: the two-phase kernels against float64 transcriptions of the formulas, on guarded
operands and twice from the same inputs; the engine against the package's optimizer classes (utils/optim.py) on
vggf-mini and on full VGG-F at batch 64, 224²."""
import math

import pytest
import torch

from guarded import NAN, Guarded
from distributed_vgg_f_b200.config import TRAIN
from distributed_vgg_f_b200.parallel.buckets import make_bucket_plan
from distributed_vgg_f_b200.parallel.layerwise import layerwise_plan

pytestmark = pytest.mark.gpu
DEV = "cuda"
F32 = torch.float32
ULP = 2.0 ** -23

# four tensors: two in the first bucket, one cut into three pieces by the 8192-element cap, a last one whose
# weights are all zero (ratio 1); the second takes no decay (not adapted)
SIZES = [("a", 5000), ("b", 300), ("c", 20000), ("d", 64)]
DECAY = {"a": 0.1, "b": 0.0, "c": 0.05, "d": 0.1}


def _ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from distributed_vgg_f_b200 import ops
    ops.require()
    return ops


def _plan():
    bp = make_bucket_plan(SIZES, cap_elems=8192, align=64)
    return bp, layerwise_plan(bp, DECAY.__getitem__, sms=torch.cuda.get_device_properties(0).multi_processor_count)


class Arena:
    """The operands of one layer-wise step over the test plan, each inside a guarded buffer."""

    def __init__(self, bp, kind, g16: bool, ema: bool, seed: int):
        gen = torch.Generator(device=DEV).manual_seed(seed)
        n = bp.total

        def make(dtype, values):
            g = Guarded((n,), (1,), dtype, 0, NAN, DEV)
            g.t.copy_(values)
            return g

        mask = torch.zeros(n, device=DEV)
        for name, numel in SIZES:
            if name != "d":
                mask[bp.offsets[name]:bp.offsets[name] + numel] = 1.0     # padding: zero weight and gradient
        p = torch.randn(n, device=DEV, generator=gen) * mask
        g = torch.randn(n, device=DEV, generator=gen) * 10.0 ** (-3 * torch.rand(n, device=DEV, generator=gen)) * mask
        g[bp.offsets["d"]:bp.offsets["d"] + 64] = torch.randn(64, device=DEV, generator=gen)
        m = torch.randn(n, device=DEV, generator=gen) * 1e-2 * mask
        v = torch.rand(n, device=DEV, generator=gen) * 1e-4 * mask
        self.kind, self.n = kind, n
        self.p, self.m = make(F32, p), make(F32, m)
        self.v = make(F32, v) if kind == "lamb" else None
        self.g32 = make(F32, g)
        self.g16 = make(torch.bfloat16, g.to(torch.bfloat16)) if g16 else None
        self.w16 = Guarded((n,), (1,), torch.bfloat16, 0, NAN, DEV)
        self.ema = make(F32, torch.randn(n, device=DEV, generator=gen) * mask) if ema else None
        self.ws = Guarded((4096,), (1,), F32, 0, NAN, DEV)
        self.ratio = Guarded((8,), (1,), F32, 0, NAN, DEV)

    def all(self):
        return [x for x in (self.p, self.m, self.v, self.g32, self.g16, self.w16, self.ema, self.ws, self.ratio)
                if x is not None]

    def grad64(self):
        return (self.g16.t if self.g16 is not None else self.g32.t).double()


HP = dict(lr=0.02, step=3, grad_scale=0.25, momentum=0.9, first=False, ema_decay=0.75)


def f32(x: float) -> float:
    """x as the kernels see it: rounded to fp32 once."""
    return float(torch.tensor(x, dtype=F32))


def _run(ops, bp, lw, A: Arena, zero: bool):
    """One step over every unit, as the engine issues it: phase 1 of the unit, then the phase 2 it completes."""
    lamb = A.kind == "lamb"
    hyper = dict(beta1=TRAIN.lamb_beta1, beta2=TRAIN.lamb_beta2, eps=TRAIN.lamb_eps, step=HP["step"]) if lamb else \
        dict(momentum=HP["momentum"], first=HP["first"], trust_coeff=TRAIN.lars_trust_coeff, trust_eps=TRAIN.lars_eps)
    for s, _ in lw.units:
        for L in lw.phase1[s]:
            a, b = L.start, L.end
            grad = dict(g16=A.g16.t[a:b]) if A.g16 is not None else dict(g32=A.g32.t[a:b])
            ops.layerwise_step(1, A.kind, A.p.t[a:b], A.m.t[a:b], A.v.t[a:b] if lamb else None,
                               zero=A.g32.t[a:b] if (zero and lamb) else None, ws=A.ws.t, lr=HP["lr"],
                               grad_scale=HP["grad_scale"], segments=L.segments, **grad, **hyper)
        for L in lw.phase2[s]:
            a, b = L.start, L.end
            grad = {}
            if not lamb:
                grad = dict(g16=A.g16.t[a:b]) if A.g16 is not None else dict(g32=A.g32.t[a:b])
                if zero:
                    grad["zero"] = A.g32.t[a:b]
            ema = dict(ema=A.ema.t[a:b], ema_decay=HP["ema_decay"]) if A.ema is not None else {}
            ops.layerwise_step(2, A.kind, A.p.t[a:b], A.m.t[a:b], A.v.t[a:b] if lamb else None, shadow=A.w16.t[a:b],
                               ws=A.ws.t, ratio=A.ratio.t, lr=HP["lr"], grad_scale=HP["grad_scale"],
                               segments=L.segments, **grad, **ema, **hyper)
    torch.cuda.synchronize()


def _reference(bp, A: Arena, p, m, v, g):
    """float64 LAMB / LARS of every tensor from the same (fp32 / bf16) inputs: new p, m, v and the ratios."""
    p, m, g = p.clone(), m.clone(), g * f32(HP["grad_scale"])
    lr = f32(HP["lr"])
    v = v.clone() if v is not None else None
    ratios = []
    for name, _ in SIZES:
        a = bp.offsets[name]
        b = a + -(-bp.numels[name] // bp.align) * bp.align
        wd, P, G = f32(DECAY[name]), p[a:b], g[a:b]
        pn = float(P.norm())
        if A.kind == "lamb":
            b1, b2, eps, t = f32(TRAIN.lamb_beta1), f32(TRAIN.lamb_beta2), f32(TRAIN.lamb_eps), HP["step"]
            m[a:b] = b1 * m[a:b] + (1 - b1) * G
            v[a:b] = b2 * v[a:b] + (1 - b2) * G * G
            u = (m[a:b] / (1 - b1 ** t)) / (v[a:b].sqrt() / math.sqrt(1 - b2 ** t) + eps) + wd * P
            un = float(u.norm())
            r = pn / un if (wd != 0 and pn > 0 and un > 0) else 1.0
            p[a:b] = P - lr * r * u
        else:
            wd = f32(wd)
            gn = float(G.norm())
            r = f32(TRAIN.lars_trust_coeff) * pn / (gn + wd * pn + f32(TRAIN.lars_eps)) \
                if (wd != 0 and pn > 0 and gn > 0) else 1.0
            u = r * (G + wd * P)                         # d
            m[a:b] = u if HP["first"] else f32(HP["momentum"]) * m[a:b] + u
            p[a:b] = P - lr * m[a:b]
        ratios.append((name, r, u))
    return p, m, v, ratios


def _close(got, want, scale, what):
    err = (got.double() - want).abs()
    bad = err > scale
    assert not bool(bad.any()), "%s: %d elements off, worst %.3g against %.3g" % (
        what, int(bad.sum()), float(err.max()), float(scale.max() if torch.is_tensor(scale) else scale))


@pytest.mark.parametrize("kind", ["lamb", "lars"])
@pytest.mark.parametrize("g16,ema,zero", [(False, False, True), (True, True, False), (False, True, False),
                                          (True, False, True)])
def test_layerwise_kernels_match_float64_on_guarded_operands(kind, g16, ema, zero):
    """Several tensors per launch, a tensor fed to phase 1 in three pieces, a tensor without decay and one with
    zero weights; fp32 or bf16 gradients at grad_scale 1/4, EMA and gradient zeroing on and off.  Moments at the
    Adam kernel's bound, ratios within 1e-5, weights within 4 ulp + lr |r u| 1e-5, shadow = RNE(p) bit for bit,
    every guard untouched; then the same step again from the same inputs gives the same bits."""
    ops = _ops()
    bp, lw = _plan()
    assert len(lw.phase1[lw.units[1][0]]) == 1 and lw.slots["c"][1] >= 3
    outs = []
    for rep in range(2):
        A = Arena(bp, kind, g16, ema, seed=7)
        p0, m0 = A.p.t.double(), A.m.t.double()
        v0 = A.v.t.double() if A.v is not None else None
        e0 = A.ema.t.double() if A.ema is not None else None
        g0 = A.grad64()
        for x in A.all():
            x.seal()
        _run(ops, bp, lw, A, zero)
        P, M, V, ratios = _reference(bp, A, p0, m0, v0, g0)
        written = [(A.p, [A.p.t]), (A.m, [A.m.t]), (A.w16, [A.w16.t]), (A.ws, [A.ws.t[:lw.workspace_elems()]]),
                   (A.ratio, [A.ratio.t[:len(SIZES)]])]
        if A.v is not None:
            written.append((A.v, [A.v.t]))
        if A.ema is not None:
            written.append((A.ema, [A.ema.t]))
        if zero:
            written.append((A.g32, [A.g32.t]))
        for x, w in written:
            x.check(w, what="%s operand" % kind)
        for x in A.all():
            if all(x is not y for y, _ in written):
                x.check((), what="%s read-only operand" % kind)
        if kind == "lamb":
            gs = g0 * HP["grad_scale"]
            _close(A.m.t, M, 4 * ULP * (0.9 * m0.abs() + 0.1 * gs.abs()) + 1e-30, "m")
            _close(A.v.t, V, 6 * ULP * (0.999 * v0.abs() + 0.001 * gs * gs) + 1e-30, "v")
        for k, (name, r, u) in enumerate(ratios):
            got = float(A.ratio.t[k])
            assert abs(got - r) <= 1e-5 * abs(r), "%s: ratio %.9g, float64 %.9g" % (name, got, r)
            a = bp.offsets[name]
            b = a + -(-bp.numels[name] // bp.align) * bp.align
            if kind == "lamb":
                tol = 4 * ULP * P[a:b].abs() + HP["lr"] * abs(r) * u.abs() * 1e-5 + 1e-30
            else:        # the buffer: the ratio's error (<= 1e-5) times d, plus a few roundings of each term
                btol = (8 * ULP + 1e-5) * (HP["momentum"] * m0[a:b].abs() + u.abs()) + 1e-30
                _close(A.m.t[a:b], M[a:b], btol, "%s momentum buffer" % name)
                tol = 4 * ULP * P[a:b].abs() + HP["lr"] * (btol + 4 * ULP * M[a:b].abs()) + 1e-30
            _close(A.p.t[a:b], P[a:b], tol, "%s weights" % name)
        assert torch.equal(A.w16.t, A.p.t.to(torch.bfloat16)), "shadow != RNE(p)"
        if A.ema is not None:
            d = HP["ema_decay"]
            want = d * e0 + (1 - d) * A.p.t.double()
            _close(A.ema.t, want, 4 * ULP * (d * e0.abs() + (1 - d) * A.p.t.double().abs()) + 1e-30, "ema")
        if zero:
            assert torch.count_nonzero(A.g32.t) == 0, "the gradient was not cleared"
        outs.append([x.t.clone() for x in (A.p, A.m, A.w16, A.ratio) ])
    for a, b in zip(*outs):
        assert torch.equal(a.view(torch.int16) if a.dtype == torch.bfloat16 else a.view(torch.int32),
                           b.view(torch.int16) if b.dtype == torch.bfloat16 else b.view(torch.int32)), \
            "the same launches twice gave different bits"


# ------------------------------------------------------------------------------------ engine
LR = 1e-3


@pytest.mark.parametrize("kind", ["lamb", "lars"])
def test_vggf_mini_steps_match_the_package_optimizer(kind):
    """vggf-mini steps with a large decay and the biases at 0: from the engine's own state, the package's Lamb /
    Lars with torchvision's two parameter groups, stepped with the bf16-emulating chain's gradients, lands within
    4 lr of every weight; torch's Adam (LAMB) / SGD (LARS) without decay does not."""
    _ops()
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine
    from distributed_vgg_f_b200.models.vggf import build_oracle, vggf_mini_spec
    from distributed_vgg_f_b200.ops import ref as R
    from distributed_vgg_f_b200.utils.optim import Lamb, Lars

    spec = vggf_mini_spec(3)
    wd = 10.0 if kind == "lamb" else 1.0      # LAMB: u ~ wd p, r ~ 1 / wd, steps far below Adam's ~lr
    lr = LR if kind == "lamb" else 0.1
    eng = NativeEngine(spec, device=torch.device(DEV), batch=4, lr=lr, seed=0, input_hw=64, distributed=False,
                       optimizer=kind, weight_decay=wd, bias_weight_decay=0.0,
                       init_state=build_oracle(spec, seed=0).state_dict())
    eng.train_dropout = False
    torch.manual_seed(4)
    for k in range(3):
        x = torch.randn(4, 3, 64, 64, device=DEV).to(torch.bfloat16).float()
        y = torch.randint(0, 3, (4,), device=DEV)
        state = {n: t.to(DEV) for n, t in eng.export_state().items()}
        st = eng.export_optimizer_state()
        _, _, grads = R.emulated_step(spec, state, x, y)
        refs = {}
        plain = torch.optim.Adam if kind == "lamb" else torch.optim.SGD
        for cls in (Lamb if kind == "lamb" else Lars, plain):
            params = {n: t.clone().requires_grad_(True) for n, t in state.items()}
            decay = wd if cls in (Lamb, Lars) else 0.0
            groups = [{"params": [params[n] for n in spec.param_names if not n.endswith(".bias")],
                       "weight_decay": decay},
                      {"params": [params[n] for n in spec.param_names if n.endswith(".bias")], "weight_decay": 0.0}]
            opt = cls(groups, lr=lr, **(dict(momentum=TRAIN.momentum) if cls in (Lars, torch.optim.SGD) else {}))
            for n in spec.param_names:
                params[n].grad = grads[n].to(DEV).float()
                if st["step"]:
                    if kind == "lamb":
                        opt.state[params[n]] = {"exp_avg": st["exp_avg"][n].to(DEV),
                                                "exp_avg_sq": st["exp_avg_sq"][n].to(DEV)}
                        if cls is torch.optim.Adam:
                            opt.state[params[n]]["step"] = torch.tensor(float(st["step"]))
                    else:
                        opt.state[params[n]] = {"momentum_buffer": st["momentum_buffer"][n].to(DEV)}
            for gr in opt.param_groups:
                gr["step"] = st["step"]
            opt.step()
            refs[cls] = {n: t.detach() for n, t in params.items()}
        eng.train_step((x, y))
        eng.sync()
        got = {n: t.to(DEV) for n, t in eng.export_state().items()}
        ratio = dict(zip(eng.layerwise_plans()[False].tensors, eng.trust_ratio.tolist()))
        mine = refs[Lamb if kind == "lamb" else Lars]
        tol = {}
        for n in spec.param_names:
            # LAMB: a flipped sign of a tiny gradient moves an element by up to 2 lr r (the bf16-emulating chain
            # and the engine round differently); LARS: 5 % of the tensor's largest step
            # (the unadapted biases: plain SGD, where the two chains' gradients differ by up to a third of the step)
            move = float((mine[n] - state[n]).abs().max())
            tol[n] = 4 * lr * ratio[n] if kind == "lamb" else (0.05 if ratio[n] != 1.0 else 0.5) * move + 1e-7
            err = float((got[n] - mine[n]).abs().max())
            assert err <= tol[n], "step %d: %s is %.3g from the package's %s (tolerance %.3g)" % (k, n, err, kind,
                                                                                                tol[n])
        weights = [n for n in spec.param_names if not n.endswith(".bias")]
        worst = max(float((got[n] - refs[plain][n]).abs().max()) for n in weights)
        assert worst > 2 * max(tol[n] for n in weights), "the trust ratio is invisible next to the tolerance"


# ------------------------------------------------------------------------------------ full VGG-F
B, HW = 64, 224


def _batch(seed):
    from distributed_vgg_f_b200.data import transforms as T
    from distributed_vgg_f_b200.data.loader import FusedBatch
    from distributed_vgg_f_b200.data.synthetic import synthetic_uint8_batch

    imgs, labels = synthetic_uint8_batch(B, 128, 3, seed=seed)
    params = T.sample_train_params(B, 128, 128, generator=torch.Generator().manual_seed(seed))
    return FusedBatch(torch.from_numpy(imgs).pin_memory(), params.pin_memory(), torch.from_numpy(labels).pin_memory(),
                      (256, 256), None)


def _engine(kind="lamb", **kw):
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine
    from distributed_vgg_f_b200.models.vggf import build_oracle, vggf_spec

    spec = vggf_spec(3)
    lr = kw.pop("lr", 1e-3 if kind in ("lamb", "adam") else 0.1)
    eng = NativeEngine(spec, device=torch.device(DEV), batch=B, lr=lr, seed=0, distributed=False,
                       optimizer=kind, weight_decay=kw.pop("weight_decay", 0.05), bias_weight_decay=0.0,
                       init_state=build_oracle(spec, seed=0).state_dict(), **kw)
    eng.train_dropout = False
    return eng


def _free(*engines):
    for e in engines:
        del e
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _snapshot(eng):
    keep = dict(step_count=eng.step_count, micro_count=eng.micro_count)
    if eng.powersgd_rank:
        keep.update(_psgd_started=eng._psgd_started)
        tensors = {k: getattr(eng, k).clone() for k in ("_psgd_e", "_psgd_p", "_psgd_q")}
    else:
        tensors = {}
    return keep, tensors


def _restore(eng, snap):
    keep, tensors = snap
    for k, v in keep.items():
        setattr(eng, k, v)
    for k, t in tensors.items():
        getattr(eng, k).copy_(t)


def _step_against_package(eng, batches):
    """One update over ``batches`` (an accumulation group) twice from the same state: first with the updates off,
    to read the gradient the update uses, then for real.  Returns, per trainable tensor, the worst weight error
    against the package's optimizer stepped on that gradient, its largest weight change and its largest weight."""
    from distributed_vgg_f_b200.models import layout as L
    from distributed_vgg_f_b200.utils.optim import Lamb, Lars

    spec = eng.spec
    names = eng.trainable_names()
    before = eng.export_state()
    st = eng.export_optimizer_state()
    snap = _snapshot(eng)
    eng.apply_updates = False
    for i, b in enumerate(batches):
        eng.train_step(b, update=i == len(batches) - 1)
    eng.sync()
    # world 1: g32 holds the sum of the group's micro-batch means, except where PowerSGD wrote the mean
    psgd = set(eng._psgd) if eng.powersgd_rank and eng._psgd_now else set()
    grads = {n: L.to_torch(spec, n, eng._view(eng.g32, n)).cpu() / (1 if n in psgd else len(batches)) for n in names}
    eng.g32.zero_()
    _restore(eng, snap)
    eng.apply_updates = True
    for i, b in enumerate(batches):
        eng.train_step(b, update=i == len(batches) - 1)
    eng.sync()
    after = eng.export_state()
    # in float64: torch's fp32 CPU norm of the 103 M elements of classifier.0.weight is off by up to 1e-2
    params = {n: before[n].double().requires_grad_(True) for n in names}
    groups = [{"params": [params[n] for n in names if not n.endswith(".bias")], "weight_decay": eng.weight_decay},
              {"params": [params[n] for n in names if n.endswith(".bias")], "weight_decay": 0.0}]
    cls = Lamb if eng.opt_name == "lamb" else Lars
    opt = cls(groups, lr=eng.lr, **({} if cls is Lamb else dict(momentum=eng.momentum)))
    for n in names:
        params[n].grad = grads[n].double()
        if st["step"]:
            opt.state[params[n]] = ({"exp_avg": st["exp_avg"][n].double(), "exp_avg_sq": st["exp_avg_sq"][n].double()}
                                    if cls is Lamb else {"momentum_buffer": st["momentum_buffer"][n].double()})
    for gr in opt.param_groups:
        gr["step"] = st["step"]
    opt.step()
    for n in spec.param_names:
        if n not in names:
            assert torch.equal(after[n], before[n]), "frozen %s moved" % n
    return {n: (float((after[n].double() - params[n].detach()).abs().max()),
                float((params[n].detach() - before[n].double()).abs().max()),
                float(before[n].abs().max())) for n in names}


def test_vggf_lamb_deterministic_runs_are_bit_identical():
    _ops()
    runs = []
    for _ in range(2):
        eng = _engine(deterministic=True)
        for k in range(2):
            eng.train_step(_batch(k))
        eng.sync()
        runs.append((eng.export_state(), eng.export_optimizer_state(), eng.trust_ratio.cpu().clone()))
        _free(eng)
    (s0, o0, r0), (s1, o1, r1) = runs
    assert torch.equal(r0, r1) and bool((r0 != 1).any())
    for n in s0:
        assert torch.equal(s0[n], s1[n]), n
        assert torch.equal(o0["exp_avg_sq"][n], o1["exp_avg_sq"][n]), n


@pytest.mark.parametrize("case", ["accum2_lamb", "freeze13_lars", "powersgd_lamb", "lars"])
def test_vggf_update_matches_the_package_optimizer(case):
    """An accumulation group of two micro-batches, 13 frozen layers, a PowerSGD-compressed update (start iter 2)
    and plain LARS: the engine's update equals the package's optimizer on the same gradient, to fp32 rounding."""
    _ops()
    kind = "lars" if "lars" in case else "lamb"
    kw = dict(deterministic=True)
    if case.startswith("freeze"):
        kw["freeze_layers"] = 13
    if case.startswith("powersgd"):
        kw.update(powersgd_rank=2, powersgd_start_iter=2)
    eng = _engine(kind, **kw)
    for k in range(2):                          # updates 1 and 2; the third is compressed under PowerSGD
        eng.train_step(_batch(10 + k))
    batches = [_batch(20), _batch(21)] if case.startswith("accum2") else [_batch(20)]
    rows = _step_against_package(eng, batches)
    _free(eng)
    for n, (err, move, top) in rows.items():
        assert move > 0, "%s: %s did not move" % (case, n)
        # fp32 rounding: the ratio and the update to ~1e-5 of the step, and a few ulp of the weights
        assert err <= 1e-3 * move + 4 * ULP * top, "%s: %s is %.3g from the package's update (step %.3g)" % (
            case, n, err, move)


def test_vggf_lamb_resume_equals_the_uninterrupted_run(tmp_path):
    from distributed_vgg_f_b200.utils import checkpoint as ckpt

    _ops()
    a = _engine(deterministic=True)
    for k in range(2):
        a.train_step(_batch(30 + k))
    ckpt.save_checkpoint(str(tmp_path / "c.pt"), a, None, 1, {})
    a.train_step(_batch(32))
    a.sync()
    want = a.export_state()
    _free(a)
    b = _engine(deterministic=True)
    ckpt.load_checkpoint(str(tmp_path / "c.pt"), b)
    b.train_step(_batch(32))
    b.sync()
    got = b.export_state()
    _free(b)
    for n in want:
        assert torch.equal(want[n], got[n]), n


@pytest.mark.parametrize("kind", ["lamb", "lars"])
def test_vggf_launches_per_step_add_the_planned_phase2_count(kind):
    from distributed_vgg_f_b200 import ops

    _ops()
    counts = {}
    for opt in ("adam", kind):
        eng = _engine(opt)
        eng.train_step(_batch(40))
        eng.sync()
        n0 = ops.launch_count()
        eng.train_step(_batch(41))
        eng.sync()
        counts[opt] = ops.launch_count() - n0
        if opt == kind:
            phase2 = eng.layerwise_plans()[False].phase2_count()
        _free(eng)
    assert counts[kind] == counts["adam"] + phase2, counts
