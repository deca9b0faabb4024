"""Knowledge distillation on the sm_90a kernels: the distillation losses (head_ce_kd, cross_entropy_kd) against
float64 on guarded operands, the forward-only teacher engine against ops.ref.emulated_step, and engine steps with a
teacher against emulated_step given the teacher's logits, from vggf-mini up to full-size VGG-F and vggf11."""
import os

import pytest
import torch

import test_deterministic_gpu as TD
import test_mixing_gpu as TM
from guarded import guarded

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _ops():
    from distributed_vgg_f_b200 import ops
    ops.require()
    return ops


def _soft(form, B, C, y):
    """(eps, MixDraw or None, float probability targets or None)."""
    T = TM._T()
    if form == "none":
        return 0.0, None, None
    if form == "smooth":
        return 0.1, None, None
    mix = T.MixDraw("mixup", 0.37, (0, 0, 0, 0))
    return 0.05, mix, T.mixed_targets(y, C, mix).double()


def _check(loss, dl, meter, B, ref):
    want = float(ref["loss"])
    assert abs(loss - want) <= 1e-4 * max(1.0, abs(want)), (loss, want)
    want_dl = ref["dlogits"]
    err = (dl - want_dl).abs()
    assert bool((err <= want_dl.abs() * 2.0 ** -8 + 1e-6 * float(want_dl.abs().max()) + 1e-9).all()), float(err.max())
    assert abs(float(meter[0]) - want * B) <= 1e-4 * max(1.0, abs(want)) * B
    assert int(meter[1]) == int(ref["meter"][1]) and int(meter[2]) == B


def _teacher_logits(B, C, g, logits=None):
    """Teacher logits: near the student's for some rows (small KL), far for others."""
    u = torch.randn(B, C, generator=g) * 2.5
    if logits is not None:
        u[::2] = logits.cpu()[::2] + 0.3 * torch.randn(u[::2].shape, generator=g)
    return u


# ------------------------------------------------------------------------------------------ loss kernels
@pytest.mark.parametrize("C", [2, 3, 8])
@pytest.mark.parametrize("B", [1, 7, 64, 256])
@pytest.mark.parametrize("K", [64, 512, 1024])
@pytest.mark.parametrize("alpha,temperature", [(0.5, 1.0), (0.5, 4.0), (1.0, 1.0), (1.0, 4.0)])
@pytest.mark.parametrize("form", ["none", "smooth", "mix"])
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("accumulate", [False, True])
def test_head_ce_kd_matches_float64(C, B, K, alpha, temperature, form, weighted, accumulate):
    ops = _ops()
    from distributed_vgg_f_b200.ops import ref as R

    g = torch.Generator().manual_seed(C * 100003 + B * 101 + K)
    h = torch.relu(torch.randn(B, K, generator=g)).to(torch.bfloat16)
    W = (torch.randn(C, K, generator=g) * (1.5 / K ** 0.5)).to(torch.bfloat16)
    bias = torch.randn(C, generator=g) * 0.1
    y = TM._labels(B, C, g)
    cw = (torch.rand(C, generator=g) + 0.5) if weighted else None
    eps, mix, soft = _soft(form, B, C, y)
    u = _teacher_logits(B, C, g, (h.float() @ W.float().t() + bias))
    gl = guarded((B, C), (C, 1), torch.float32, 0, float("nan"), DEV)
    gdl = guarded((B, 8), (8, 1), torch.bfloat16, 0, 9.0, DEV, torch.zeros(B, 8))
    gdW = guarded((C, K), (K, 1), torch.float32, 0, 3.0, DEV, torch.full((C, K), 3.0))
    gdb = guarded((C,), (1,), torch.float32, 0, 0.25, DEV, torch.full((C,), 0.25))
    gdh = guarded((B, K), (K, 1), torch.bfloat16, 0, 7.0, DEV)
    gu = guarded((B, C), (C, 1), torch.float32, 0, float("nan"), DEV, u)
    for t in (gl, gdl, gdW, gdb, gdh, gu):
        t.seal()
    meter, loss = torch.zeros(4, device=DEV), torch.zeros(1, device=DEV)
    n0 = ops.launch_count()
    ops.require().head_ce_kd(h.to(DEV), W.to(DEV), bias.to(DEV), y.to(DEV), gl.t, gdl.t, 8, gdW.t, gdb.t, gdh.t, 2.0,
                             True, meter, loss, None if cw is None else cw.to(DEV), accumulate,
                             ops.soft_targets(eps, mix), gu.t, alpha, temperature)
    torch.cuda.synchronize()
    assert ops.launch_count() - n0 == 1
    gl.check([gl.t], "logits")
    gdl.check([gdl.t[:, :C]], "dlogits")
    gdW.check([gdW.t], "dW")
    gdb.check([gdb.t], "db")
    gdh.check([gdh.t], "dh")
    gu.check((), "teacher logits")
    assert torch.count_nonzero(gdl.t[:, C:]) == 0
    ref = R.kd_cross_entropy64(gl.t.cpu(), u, y, alpha=alpha, temperature=temperature, class_weights=cw,
                               label_smoothing=eps, soft_target=soft)
    _check(float(loss), gdl.t[:, :C].double().cpu(), meter.cpu(), B, ref)
    ref = R.head_ce64(h, W, bias, dl_used=gdl.t[:, :C].cpu(), drop_scale=2.0, relu=True)
    lr, lm = ref["logits"]
    assert bool(((gl.t.double().cpu() - lr).abs() <= 1e-4 * lm + 1e-6).all())
    for name, got in (("dW", gdW.t - (3.0 if accumulate else 0.0)), ("db", gdb.t - 0.25)):
        r, m = ref[name]
        assert bool(((got.double().cpu() - r).abs() <= 1e-4 * m + 1e-5 * (3.0 if accumulate else 0.0) + 1e-9).all()), name
    r, m = ref["dh"]
    assert bool(((gdh.t.double().cpu() - r).abs() <= r.abs() * 2.0 ** -8 + 1e-5 * m + 1e-12).all())


@pytest.mark.parametrize("C", [9, 100, 1000])
@pytest.mark.parametrize("B", [1, 7, 64, 256])
@pytest.mark.parametrize("alpha,temperature", [(0.5, 1.0), (0.5, 4.0), (1.0, 1.0), (1.0, 4.0)])
@pytest.mark.parametrize("form", ["none", "smooth", "mix"])
@pytest.mark.parametrize("weighted", [False, True])
def test_cross_entropy_kd_matches_float64(C, B, alpha, temperature, form, weighted):
    ops = _ops()
    from distributed_vgg_f_b200.ops import ref as R

    g = torch.Generator().manual_seed(C * 1000 + B + 5)
    logits = torch.randn(B, C, generator=g) * 3
    if B > 4:
        logits[4, 1] = logits[4, 0] = logits[4].max() + 1          # a tie: the first maximum counts
    y = TM._labels(B, C, g)
    cw = (torch.rand(C, generator=g) + 0.5) if weighted else None
    eps, mix, soft = _soft(form, B, C, y)
    u = _teacher_logits(B, C, g, logits)
    ldd = C + (8 - C % 8) % 8
    gdl = guarded((B, ldd), (ldd, 1), torch.bfloat16, 0, 9.0, DEV)
    gz = guarded((B, C), (C, 1), torch.float32, 0, float("nan"), DEV, logits)
    gu = guarded((B, C), (C, 1), torch.float32, 0, float("nan"), DEV, u)
    for t in (gdl, gz, gu):
        t.seal()
    meter, loss = torch.zeros(4, device=DEV), torch.zeros(1, device=DEV)
    ops.cross_entropy_kd(gz.t, y.to(DEV), gu.t, alpha=alpha, temperature=temperature, dlogits=gdl.t, ldd=ldd,
                         meter=meter, loss_out=loss, class_weights=None if cw is None else cw.to(DEV),
                         label_smoothing=eps, mix=mix)
    torch.cuda.synchronize()
    gdl.check([gdl.t], "dlogits")
    gz.check((), "logits")
    gu.check((), "teacher logits")
    assert torch.count_nonzero(gdl.t[:, C:]) == 0
    ref = R.kd_cross_entropy64(logits, u, y, alpha=alpha, temperature=temperature, class_weights=cw,
                               label_smoothing=eps, soft_target=soft)
    _check(float(loss), gdl.t[:, :C].double().cpu(), meter.cpu(), B, ref)


def test_kd_entries_refuse_bad_operands():
    ops = _ops()
    C_ = ops.require()
    B, C, K = 4, 3, 64
    h = torch.zeros(B, K, dtype=torch.bfloat16, device=DEV)
    W = torch.zeros(C, K, dtype=torch.bfloat16, device=DEV)
    bias, y = torch.zeros(C, device=DEV), torch.zeros(B, dtype=torch.int64, device=DEV)
    logits, dl = torch.zeros(B, C, device=DEV), torch.zeros(B, 8, dtype=torch.bfloat16, device=DEV)
    good = torch.zeros(B, C, device=DEV)
    bad_teachers = [torch.zeros(B - 1, C, device=DEV), torch.zeros(B, C + 1, device=DEV),
                    torch.zeros(B, C, device=DEV, dtype=torch.float64), torch.zeros(C, B, device=DEV).t(),
                    torch.zeros(B * C, device=DEV), torch.zeros(B, C)]
    cases = [(t, 0.5, 4.0) for t in bad_teachers]
    cases += [(good, a, T) for a, T in ((0.0, 4.0), (-0.1, 4.0), (1.5, 4.0), (0.5, 0.0), (0.5, -1.0),
                                        (0.5, float("inf")), (0.5, float("nan")), (float("nan"), 4.0))]
    n0 = ops.launch_count()
    for teacher, a, T in cases:
        with pytest.raises(RuntimeError):
            C_.head_ce_kd(h, W, bias, y, logits, dl, 8, None, None, None, 1.0, True, None, None, None, False, None,
                          teacher, a, T)
        with pytest.raises(RuntimeError):
            C_.cross_entropy_kd(logits, y, dl, 8, None, None, 1.0 / B, None, teacher, a, T)
    assert ops.launch_count() == n0
    # the operand checks head_ce makes apply to head_ce_kd as well
    with pytest.raises(RuntimeError, match="head_ce_kd: db must have C elements"):
        C_.head_ce_kd(h, W, bias, y, logits, dl, 8, torch.zeros(C, K, device=DEV), torch.zeros(1, device=DEV), None,
                      1.0, True, None, None, None, False, None, good, 0.5, 4.0)
    assert ops.launch_count() == n0


# ------------------------------------------------------------------------------------------ teacher engine
def _rounded_oracle(spec, seed):
    from distributed_vgg_f_b200.models.vggf import build_oracle

    oracle = build_oracle(spec, seed=seed)
    with torch.no_grad():
        for p in oracle.parameters():
            if p.dim() > 1:
                p.copy_(p.to(torch.bfloat16).float())
    return oracle


def _teacher(spec, seed, batch, hw, **kw):
    from distributed_vgg_f_b200.engine.native_engine import TeacherEngine

    oracle = _rounded_oracle(spec, seed)
    return oracle, TeacherEngine(spec, torch.device(DEV), batch, oracle.state_dict(), input_hw=hw, **kw)


@pytest.mark.parametrize("model,hw,b", [("vggf", 224, 8), ("vggf-mini", 64, 4)])
def test_teacher_engine_logits_match_the_emulated_forward(model, hw, b):
    from distributed_vgg_f_b200.models.vggf import get_spec
    from distributed_vgg_f_b200.ops import ref as R

    spec = get_spec(model, 3)
    oracle, t = _teacher(spec, 7, b, hw)
    g = torch.Generator().manual_seed(2)
    x = torch.randn(b, 3, hw, hw, generator=g)
    y = torch.randint(0, 3, (b,), generator=g)
    t._set_hw(t.HW)
    n = t._stage_input((x, y))
    got = t.forward_teacher(t.x_nhwc, t.labels_dev, n).clone()
    torch.cuda.synchronize()
    state = {k: v.detach().to(DEV) for k, v in oracle.state_dict().items()}
    want = R.emulated_step(spec, state, R.rb(x.to(DEV)), y.to(DEV))[0]
    err = float((got - want).norm() / want.norm())
    assert err < 2e-2, err
    # forward only: no gradient, moment, EMA or wire arena, no backward buffer, no comm or optimizer stream
    for name in ("g32", "m32", "v32", "arena", "comm_stream", "opt_stream", "fc_dz", "fc_dacc", "dbuf", "dfeat"):
        assert getattr(t, name, None) is None, name
    assert t.ema32 is None and getattr(t, "ema16", None) is None
    params = sum(p.numel() for p in oracle.parameters())
    assert t.p32.numel() >= params and t.device_bytes() >= 6 * params


# ------------------------------------------------------------------------------------------ engine steps
def _mini_pair(classes, **kw):
    """vggf-mini student (TM._engine) and a differently seeded vggf-mini teacher, batch 4 at 64 x 64."""
    spec, oracle, eng = TM._engine(classes, **kw)
    os.environ["B200_FUSE_POOL"] = "0"
    try:
        toracle, teacher = _teacher(spec, 5, 4, 64, deterministic=eng.deterministic)
    finally:
        os.environ.pop("B200_FUSE_POOL", None)
    return spec, oracle, eng, teacher


def _override(eng, b):
    return {"acts": [a[:b].permute(0, 3, 1, 2).float() for a in eng.acts],
            "feat": eng.feat.permute(0, 3, 1, 2).float(),
            "fc_y": [t[:b].float() if t is not None else None for t in eng.fc_y],
            "logits": eng.logits[:b].clone()}


def _grad_errors(spec, eng, grads, names=None):
    from distributed_vgg_f_b200.models import layout as L

    worst = {}
    for name in names or spec.param_names:
        ref = L.to_native(spec, name, grads[name])
        g = eng._view(eng.g32, name)
        worst[name] = max(float((g - ref).abs().max() / (ref.abs().max() + 1e-12)),
                          float((g - ref).norm() / (ref.norm() + 1e-20)))
    return worst


@pytest.mark.parametrize("classes", [3, 10])           # fused head / GEMM head + cross_entropy_kd
@pytest.mark.parametrize("form", ["plain", "mixup+smooth", "accum2", "freeze"])
def test_engine_step_with_a_teacher_matches_emulated_step(capsys, classes, form):
    from distributed_vgg_f_b200.ops import ref as R

    T = TM._T()
    eps = 0.1 if "smooth" in form else 0.0
    kw = dict(label_smoothing=eps)
    if form == "freeze":
        kw["freeze_layers"] = 3
    spec, oracle, eng, teacher = _mini_pair(classes, **kw)
    assert eng.fused_head == (classes <= 8) and teacher.fused_head == (classes <= 8)
    eng.set_distillation(teacher, 0.7, 3.0)
    eng.train_dropout = False
    eng.apply_updates = False
    b = 4
    mix = T.MixDraw("mixup", 0.3, (0, 0, 0, 0)) if "mixup" in form else None
    state = {k: v.detach().to(DEV) for k, v in oracle.state_dict().items()}
    want = {n: 0.0 for n in spec.param_names}
    for k in range(2 if form == "accum2" else 1):
        batch = TM._fused_batch(b, mix, seed=3 + k, classes=classes)
        got_loss = float(eng.train_step(batch, update=form != "accum2" or k == 1))
        eng.sync()
        x = eng.x_nhwc[:b, ..., :3].permute(0, 3, 1, 2).float()
        u = teacher.logits[:b].clone()
        soft = None if mix is None else T.mixed_targets(batch.labels, classes, mix).to(DEV)
        _, loss, grads = R.emulated_step(spec, state, x, batch.labels.to(DEV), override=_override(eng, b),
                                         soft_target=soft, label_smoothing=eps, teacher_logits=u, distill_alpha=0.7,
                                         distill_temperature=3.0)
        assert abs(got_loss - float(loss)) < 1e-4 * max(1.0, abs(float(loss)))
        want = {n: want[n] + grads[n] for n in spec.param_names}
    worst = _grad_errors(spec, eng, want, eng.trainable_names())
    with capsys.disabled():
        print("\n[distill grad err, %s, C=%d] worst %.1e" % (form, classes, max(worst.values())))
    bad = {k: v for k, v in worst.items() if v > 2e-2}
    assert not bad, bad


@pytest.mark.parametrize("classes", [3, 10])
def test_engine_distillation_loss_with_class_weights(classes):
    """Class weights shape the CE term alone: the step's loss and dlogits against kd_cross_entropy64 on the engine's
    own logits and the teacher's."""
    from distributed_vgg_f_b200.ops import ref as R

    spec, oracle, eng, teacher = _mini_pair(classes)
    cw = torch.linspace(0.5, 2.0, classes)
    eng.set_class_weights(cw)
    eng.set_distillation(teacher, 0.5, 4.0)
    eng.train_dropout, eng.apply_updates = False, False
    batch = TM._fused_batch(4, None, classes=classes)
    got = float(eng.train_step(batch))
    eng.sync()
    ref = R.kd_cross_entropy64(eng.logits[:4].cpu(), teacher.logits[:4].cpu(), batch.labels, alpha=0.5,
                               temperature=4.0, class_weights=cw)
    assert abs(got - float(ref["loss"])) <= 1e-4 * max(1.0, float(ref["loss"]))
    dl = eng.fc_dz[-1][:4, :classes].double().cpu()
    assert bool(((dl - ref["dlogits"]).abs() <= ref["dlogits"].abs() * 2.0 ** -8 + 1e-6).all())


def test_eval_and_forward_logits_ignore_the_teacher():
    from distributed_vgg_f_b200.utils.metrics import DeviceMeter

    _, _, eng, teacher = _mini_pair(3)
    eng.set_distillation(teacher, 0.5, 4.0)
    batch = TM._fused_batch(4, None)
    meter = DeviceMeter(DEV)
    eng.set_meter(meter)
    eng.eval_step(batch)
    eng.sync()
    want = torch.nn.functional.cross_entropy(eng.logits[:4].double(), batch.labels.to(DEV))
    assert abs(meter.snapshot()[0].average - float(want)) < 1e-4


def test_set_distillation_refuses_a_mismatched_teacher():
    _, _, eng, teacher = _mini_pair(3)
    for a, T in ((0.0, 4.0), (1.5, 4.0), (0.5, 0.0), (0.5, float("inf"))):
        with pytest.raises(ValueError):
            eng.set_distillation(teacher, a, T)
    from distributed_vgg_f_b200.models.vggf import vggf_mini_spec

    _, other = _teacher(vggf_mini_spec(4), 1, 4, 64)
    with pytest.raises(ValueError, match="classes"):
        eng.set_distillation(other, 0.5, 4.0)
    _, other = _teacher(teacher.spec, 1, 8, 64)
    with pytest.raises(ValueError, match="batch"):
        eng.set_distillation(other, 0.5, 4.0)


def test_calls_without_a_teacher_and_launches_with_one(monkeypatch):
    """Without a teacher (never set, or set to None) the engine makes the same native calls with the same arguments
    and the same launches; with one, every step adds exactly the teacher's forward launches and swaps the loss
    launch for its distillation form."""
    ops = _ops()
    batch = TM._fused_batch(4, None)
    runs = []
    for mode in ("never", "none", "teacher"):
        rec = TM._Recorder(ops.require())
        monkeypatch.setattr(ops, "_C", rec)
        _, _, eng, teacher = _mini_pair(3)
        if mode != "never":
            eng.set_distillation(teacher if mode == "teacher" else None)
        eng.train_dropout = False
        rec.calls.clear()
        counts = []
        for k in range(3):
            eng.apply_updates = k > 0
            n0 = ops.launch_count()
            eng.train_step(batch)
            eng.sync()
            counts.append(ops.launch_count() - n0)
        n0 = ops.launch_count()
        teacher.forward_teacher(eng.x_nhwc, eng.labels_dev, 4)
        eng.sync()
        teacher_launches = ops.launch_count() - n0
        monkeypatch.undo()
        runs.append((rec.calls, counts, teacher_launches))
    assert runs[0][0] == runs[1][0] and runs[0][1] == runs[1][1]
    names = {c[0] for c in runs[0][0]}
    assert not names & {"head_ce_kd", "cross_entropy_kd"}
    with_t = {c[0] for c in runs[2][0]}
    assert "head_ce_kd" in with_t
    assert all(c == n + runs[2][2] for c, n in zip(runs[2][1], runs[0][1])), (runs[2][1], runs[0][1], runs[2][2])


# ------------------------------------------------------------------------------------------ full size
def _full(model, **kw):
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine
    from distributed_vgg_f_b200.models.vggf import get_spec

    os.environ["B200_FUSE_POOL"] = "0"       # the un-pooled activations gate the reference's backward
    try:
        spec = get_spec(model, 3)
        oracle = _rounded_oracle(spec, 0)
        eng = NativeEngine(spec, device=torch.device(DEV), batch=64, lr=1e-4, seed=0, input_hw=224,
                           init_state=oracle.state_dict(), **kw)
        tspec = get_spec("vggf", 3)
        _, teacher = _teacher(tspec, 9, 64, 224, deterministic=eng.deterministic)
    finally:
        os.environ.pop("B200_FUSE_POOL", None)
    return spec, oracle, eng, teacher


@pytest.mark.parametrize("model", ["vggf", "vggf11"])
def test_full_size_step_with_a_vggf_teacher_matches_emulated_step(capsys, model):
    from distributed_vgg_f_b200.ops import ref as R

    spec, oracle, eng, teacher = _full(model)
    eng.set_distillation(teacher, 0.5, 4.0)
    eng.train_dropout, eng.apply_updates = False, False
    batch = TD._batches(1, 64, 3, mix=False)[0]
    got = float(eng.train_step(batch))
    eng.sync()
    b = 64
    x = eng.x_nhwc[:b, ..., :3].permute(0, 3, 1, 2).float()
    state = {k: v.detach().to(DEV) for k, v in oracle.state_dict().items()}
    _, loss, grads = R.emulated_step(spec, state, x, batch.labels.to(DEV), override=_override(eng, b),
                                     teacher_logits=teacher.logits[:b].clone(), distill_alpha=0.5,
                                     distill_temperature=4.0)
    assert abs(got - float(loss)) < 1e-4 * max(1.0, abs(float(loss)))
    worst = _grad_errors(spec, eng, grads)
    with capsys.disabled():
        print("\n[distill full size %s] loss %.4f, worst grad err %.1e" % (model, got, max(worst.values())))
    bad = {k: v for k, v in worst.items() if v > 2e-2}
    assert not bad, bad


def test_full_size_deterministic_runs_are_bit_identical_and_leave_the_teacher_unchanged():
    batches = TD._batches(3, 64, 3)
    out = []
    for _ in range(2):
        spec, _, eng, teacher = _full("vggf", deterministic=True)
        before = (teacher.p32.clone(), teacher.w16.clone())
        eng.set_distillation(teacher, 0.5, 4.0)
        losses = [float(eng.train_step(bt)) for bt in batches]
        eng.sync()
        assert torch.equal(teacher.p32, before[0]) and torch.equal(teacher.w16, before[1])
        out.append((losses, eng.p32.clone(), eng.m32.clone()))
        del eng, teacher
    assert out[0][0] == out[1][0]
    assert torch.equal(out[0][1], out[1][1]) and torch.equal(out[0][2], out[1][2])
    assert all(v == v for v in out[0][0])
