"""--freeze-layers on the sm_90a engine: the default path's native calls, the trainable gradients at every
kind of cut against the unfrozen engine, the frozen state over ten updates, the float oracle, ema_kernel
against torch's eager update on guarded operands, the EMA of frozen tensors against AveragedModel's
arithmetic, repeatability under --deterministic and a checkpoint round trip."""
import pytest
import torch

import test_deterministic_gpu as TD
import test_ema_gpu as TE
from guarded import NAN, Guarded

pytestmark = pytest.mark.gpu
DEV = "cuda"
F32, BF16 = torch.float32, torch.bfloat16


def _ops():
    from distributed_vgg_f_b200 import ops
    ops.require()
    return ops


def _same_bits(got, want, what):
    TE._same_bits(got.reshape(-1), want.reshape(-1), what)


# ------------------------------------------------------------------------------------------ default path
def test_no_frozen_layer_makes_the_calls_of_an_engine_without_the_argument(monkeypatch):
    """freeze_layers=0: the same native calls with the same arguments and the same launches as an engine
    built without the argument, over a gradient-only step and two update steps; full-size arenas."""
    ops = _ops()
    runs = []
    for kw in ({}, {"freeze_layers": 0}):
        rec = TE._Recorder(ops.require())
        monkeypatch.setattr(ops, "_C", rec)
        eng = TE._engine(3, "adamw", ema_decay=0.5, **kw)
        eng.train_dropout = False
        counts = []
        for k in range(3):
            n0 = ops.launch_count()
            eng.train_step(TE._batch(4), update=k != 0, ema=k != 0)
            eng.sync()
            counts.append(ops.launch_count() - n0)
        monkeypatch.undo()
        assert eng.n_grad == eng.plan.total == eng.g32.numel() == eng.m32.numel() == eng.p32.numel()
        runs.append((list(rec.calls), counts))
    assert runs[0] == runs[1]
    assert not any(c[0] == "ema_update" for c in runs[0][0])


# ------------------------------------------------------------------------------------- trainable gradients
# (model, frozen count, batch, side): a cut after a pooled conv (4, 10), after an unpooled conv (8),
# classifier.0 first (13), the linear probe on the fused head (16) and on VGG-16's GEMM head (15)
CUTS = [("vggf-mini", 4, 4, 64), ("vggf-mini", 8, 4, 64), ("vggf-mini", 13, 4, 64), ("vggf-mini", 16, 4, 64),
        ("vggf", 10, 64, 224), ("vggf", 8, 64, 224), ("vggf", 13, 64, 224), ("vggf", 16, 64, 224),
        ("vgg16", 15, 16, 224)]
_REF = {}


def _grads(model, batch, hw, n):
    """One deterministic step without dropout and without an update: (engine, its gradient arena)."""
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine
    from distributed_vgg_f_b200.models.vggf import build_oracle, get_spec

    classes = 1000 if model == "vgg16" else 3
    spec = get_spec(model, classes)
    init = build_oracle(spec, seed=1).state_dict()
    eng = NativeEngine(spec, device=torch.device(DEV), batch=batch, lr=1e-3, seed=0, input_hw=hw, init_state=init,
                       deterministic=True, freeze_layers=n)
    eng.train_dropout = False
    eng.apply_updates = False
    eng.train_step(TD._batches(1, batch, classes, hw=256 if hw == 224 else 128, mix=False)[0])
    eng.sync()
    return eng, eng.g32.clone()


@pytest.mark.parametrize("model,n,batch,hw", CUTS)
def test_trainable_gradients_are_the_unfrozen_engines_bit_for_bit(model, n, batch, hw):
    ops = _ops()
    key = (model, batch, hw)
    if key not in _REF:
        _REF.clear()
        ref_eng, ref = _grads(model, batch, hw, 0)
        _REF[key] = ({name: ref_eng._view(ref, name).clone() for name in ref_eng.plan.order})
        del ref_eng, ref
    ref = _REF[key]
    eng, g = _grads(model, batch, hw, n)
    assert eng.fused_head == (model != "vgg16")
    frozen = set(eng.spec.frozen_param_names(n))
    assert g.numel() == eng.n_grad < eng.p32.numel()
    for name in eng.trainable_names():
        assert torch.equal(eng._view(g, name), ref[name]), "%s (%d frozen)" % (name, n)
        assert bool(ref[name].abs().sum() > 0), name
    assert all(eng.plan.offsets[t] >= eng.n_grad for t in frozen)


# ------------------------------------------------------------------------------------ frozen state stays put
class _Writes:
    """Stands in for ops._C: records every call's name and the byte ranges of its tensor arguments."""

    def __init__(self, C):
        self._C, self.calls = C, []

    def __getattr__(self, name):
        f = getattr(self._C, name)
        if not callable(f) or name == "launch_count":
            return f

        def call(*a, **k):
            spans = [(t.data_ptr(), t.data_ptr() + t.numel() * t.element_size())
                     for t in list(a) + list(k.values()) if isinstance(t, torch.Tensor)]
            self.calls.append((name, spans))
            return f(*a, **k)
        return call


@pytest.mark.parametrize("n", [4, 13])
def test_frozen_state_stays_put_over_ten_updates(monkeypatch, capsys, n):
    """AdamW with weight decay and bias decay, MixUp, two micro-batches per update, ten updates: the frozen
    ranges of p32 and w16 never change, only the frozen layers' forward launches take them as an operand,
    every update's optimizer launches cover exactly [0, T), and the first trainable layer runs no dgrad."""
    from distributed_vgg_f_b200.data import transforms as T
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine
    from distributed_vgg_f_b200.models.vggf import build_oracle, vggf_mini_spec

    ops = _ops()
    spec = vggf_mini_spec(3)
    eng = NativeEngine(spec, device=torch.device(DEV), batch=4, lr=1e-2, seed=0, input_hw=64, optimizer="adamw",
                       weight_decay=0.05, bias_weight_decay=0.01, init_state=build_oracle(spec, seed=0).state_dict(),
                       freeze_layers=n)
    T0, total = eng.n_grad, eng.plan.total
    p0, w0, t0 = eng.p32[T0:].clone(), eng.w16[T0:].clone(), eng.p32[:T0].clone()
    ptr = lambda t, i: t.data_ptr() + i * t.element_size()      # noqa: E731
    frozen = ((ptr(eng.p32, T0), ptr(eng.p32, total)), (ptr(eng.w16, T0), ptr(eng.w16, total)))
    rec = _Writes(ops.require())
    monkeypatch.setattr(ops, "_C", rec)
    per_step, marks = [], []
    for k in range(20):
        b = TE._batch(4, seed=k)
        mixed = b._replace(mix=T.MixDraw("mixup", 0.3 + 0.02 * k, (0, 0, 0, 0)))
        n0 = ops.launch_count()
        marks.append(len(rec.calls))
        eng.train_step(mixed, update=k % 2 == 1)
        eng.sync()
        per_step.append(ops.launch_count() - n0)
    marks.append(len(rec.calls))
    monkeypatch.undo()
    assert eng.step_count == 10
    _same_bits(eng.p32[T0:], p0, "frozen p32")
    assert torch.equal(eng.w16[T0:].view(torch.int16), w0.view(torch.int16)), "frozen w16"
    assert not torch.equal(eng.p32[:T0], t0), "the trainable weights did not move"
    forward = ("conv_fprop", "conv_fprop_pool", "conv0_fprop")
    span = lambda t: (t.data_ptr(), t.data_ptr() + t.numel() * t.element_size())      # noqa: E731
    # written only by classifier.0's dgrad GEMM (fc_dacc[0]) and its fc_grad_act (dfeat)
    head_in = (span(eng.fc_dacc[0]), span(eng.dfeat))
    for k in range(20):
        calls = rec.calls[marks[k]:marks[k + 1]]
        into_features = [name for name, spans in calls
                         if any(a < f1 and f0 < b for a, b in spans for f0, f1 in head_in)]
        n_gemm = sum(1 for c in calls if c[0] == "gemm")
        n_act = sum(1 for c in calls if c[0] == "fc_grad_act")
        if n >= len(spec.convs):                 # classifier.0 is the first trainable layer
            assert into_features == [], into_features
            assert (n_gemm, n_act) == (3 + 2 * 3 - 1, 2), (n_gemm, n_act)      # 3 forward, 3 wgrad, 2 dgrad
        else:
            assert sorted(set(into_features)) == ["avgpool_bwd", "fc_grad_act", "gemm"] or \
                sorted(set(into_features)) == ["fc_grad_act", "gemm"], into_features
            assert (n_gemm, n_act) == (3 + 2 * 3, 3), (n_gemm, n_act)
        touching = [name for name, spans in calls
                    if any(a < f1 and f0 < b for a, b in spans for f0, f1 in frozen)]
        assert set(touching) <= set(forward), touching
        assert len(touching) == n, touching                    # each frozen conv's forward, once
        dgrads = [c for c in calls if c[0] == "conv_dgrad"]
        assert len(dgrads) == max(0, len(spec.convs) - n - 1)  # none at the cut, none below it
        if n >= len(spec.convs):
            assert not any(c[0] in ("conv_wgrad", "unpool2x2", "maxpool_relu_bwd", "avgpool_bwd") for c in calls)
        opt = [spans[0] for name, spans in calls if name in ("adam", "sgd")]
        if k % 2 == 0:
            assert not opt
            continue
        lo = ptr(eng.p32, 0)
        cover = sorted(opt)
        assert cover[0][0] == lo and cover[-1][1] == ptr(eng.p32, T0), "optimizer range"
        assert all(x[1] == y[0] for x, y in zip(cover, cover[1:])), "gaps or overlaps in the optimizer launches"
    with capsys.disabled():
        print("\n[freeze %d] native launches per micro-batch (gradient-only, update): %d, %d"
              % (n, per_step[0], per_step[1]))


# ---------------------------------------------------------------------------------------- float oracle
@pytest.mark.parametrize("n", [2, 8, 13, 16])
def test_frozen_engine_gradients_match_the_emulated_step(n):
    """The trainable gradients of the frozen engine against ops.ref.emulated_step (which differentiates a
    model without frozen tensors: freezing leaves the trainable gradients as they are), at the tolerance of
    the engine tests; the step of a model with requires_grad_(False) has no gradient for the rest."""
    import test_mixing_gpu as TM
    from distributed_vgg_f_b200.models import layout as L
    from distributed_vgg_f_b200.ops import ref as R

    spec, oracle, eng = TM._engine(3, freeze_layers=n)
    eng.train_dropout = False
    eng.apply_updates = False
    b = 4
    batch = TM._fused_batch(b, None)
    got_loss = float(eng.train_step(batch))
    eng.sync()
    x = eng.x_nhwc[:b, ..., :3].permute(0, 3, 1, 2).float()
    override = {"acts": [a[:b].permute(0, 3, 1, 2).float() for a in eng.acts],
                "feat": eng.feat.permute(0, 3, 1, 2).float(),
                "fc_y": [t[:b].float() if t is not None else None for t in eng.fc_y],
                "logits": eng.logits[:b].clone()}
    state = {k: v.detach().to(DEV) for k, v in oracle.state_dict().items()}
    _, loss, grads = R.emulated_step(spec, state, x, batch.labels.to(DEV), override=override)
    assert abs(got_loss - float(loss)) < 1e-4
    bad = {}
    for name in eng.trainable_names():
        ref = L.to_native(spec, name, grads[name])
        g = eng._view(eng.g32, name)
        err = max(float((g - ref).abs().max() / (ref.abs().max() + 1e-12)),
                  float((g - ref).norm() / (ref.norm() + 1e-20)))
        if err > 2e-2:
            bad[name] = err
    assert not bad, bad
    # the torch model with the leading layers frozen: no gradient there, the same ones elsewhere
    from distributed_vgg_f_b200.models.vggf import freeze_leading_layers_
    frozen = set(freeze_leading_layers_(oracle, n))
    assert {k for k, p in oracle.named_parameters() if not p.requires_grad} == frozen
    assert set(eng.trainable_names()) == set(spec.param_names) - frozen


# ------------------------------------------------------------------------------------------- ema_kernel
@pytest.mark.parametrize("n,offset", [(4, 0), (1, 4), (7, 8), (1023, 12), (4 * 135_173 + 3, 4), (1 << 20, 0)])
@pytest.mark.parametrize("first", [True, False])
def test_ema_kernel_is_torch_eager_on_guarded_operands(n, offset, first):
    C = _ops().require()
    g = torch.Generator(device=DEV).manual_seed(n + first)
    p_vals = torch.randn(n, device=DEV, generator=g)
    p_vals[::97] = -0.0
    e0 = torch.full((n,), NAN, device=DEV) if first else torch.randn(n, device=DEV, generator=g)
    p = Guarded((n,), (1,), F32, offset, NAN, DEV)
    p.t.copy_(p_vals)
    p.seal()
    ema = Guarded((n,), (1,), F32, offset, NAN, DEV)
    ema.t.copy_(e0)
    ema.seal()
    n0 = C.launch_count()
    _ops().ema_update(p.t, ema.t, decay=TE.DECAY, first=first)
    torch.cuda.synchronize()
    assert C.launch_count() == n0 + 1
    p.check((), "p")
    ema.check([ema.t], "ema")
    want = p_vals if first else TE._eager(e0, p_vals, TE.DECAY)
    _same_bits(ema.t, want, "ema_kernel n=%d first=%s" % (n, first))


def test_ema_update_host_checks_refuse_before_launching():
    C = _ops().require()
    z = lambda k, dt=F32: torch.zeros(k, dtype=dt, device=DEV)      # noqa: E731
    bad = [(z(64), z(60), 0.5), (z(64), z(64, BF16), 0.5), (z(64, BF16), z(64), 0.5), (z(65)[1:], z(64), 0.5),
           (z(64), z(65)[1:], 0.5), (z(64), z(64), 1.5), (z(64), z(64), -0.1)]
    for p, e, d in bad:
        n0 = C.launch_count()
        with pytest.raises(RuntimeError):
            C.ema_update(p, e, d, False)
        assert C.launch_count() == n0
    n0 = C.launch_count()
    C.ema_update(z(0), z(0), 0.5, True)                    # nothing to average: no launch
    assert C.launch_count() == n0


@pytest.mark.parametrize("n,optimizer", [(13, "adam"), (4, "sgd"), (16, "adamw")])
def test_engine_ema_of_frozen_tensors_is_averagedmodels_arithmetic(n, optimizer):
    """The whole EMA arena after every EMA update is torch's eager d*e + (1-d)*p on a snapshot of the weights
    (AveragedModel stepped by hand): the frozen range by ema_kernel, the rest by the optimizer kernels."""
    decay = 0.75
    eng = TE._engine(3, optimizer, ema_decay=decay, freeze_layers=n)
    eng.train_dropout = False
    batches = [TE._batch(4, seed=s) for s in range(3)]
    TE._run_and_emulate(eng, decay, [u % 2 == 0 for u in range(7)], batches)
    assert eng.n_grad < eng.p32.numel()


# -------------------------------------------------------------------------------------- repeatability
def test_vggf_with_features_frozen_trains_bit_for_bit_twice():
    from distributed_vgg_f_b200.models.vggf import vggf_spec

    spec, batches = vggf_spec(3), TD._batches(20, 64, 3)
    kw = dict(batch=64, hw=224, accum=2, optimizer="adamw", label_smoothing=0.1, ema_decay=0.9, weight_decay=1e-4,
              deterministic=True, freeze_layers=13)
    e1, s1 = TD._train(spec, batches, **kw)
    assert e1.ema_updates == 10 and e1.m32.numel() == e1.n_grad < e1.p32.numel()
    del e1
    _, s2 = TD._train(spec, batches, **kw)
    TD._assert_same(s1, s2)


# ------------------------------------------------------------------------------------------- checkpoint
def test_checkpoint_round_trip_with_frozen_layers(tmp_path):
    from distributed_vgg_f_b200.utils import checkpoint as ckpt

    eng = TE._engine(3, "adam", ema_decay=0.5, freeze_layers=8)
    for k in range(3):
        eng.train_step(TE._batch(4, seed=k), ema=True)
    eng.sync()
    path = str(tmp_path / "f.pt")
    ckpt.save_checkpoint(path, eng, None, 1, {}, model_ema=True)
    payload = torch.load(path, weights_only=True)
    names = eng.spec.param_names
    assert set(payload["model"]) == {"module." + k for k in names}
    assert set(payload["model_ema"]) == {"n_averaged"} | {"module." + k for k in names}
    st = payload["optimizer"]
    assert st["frozen_layers"] == 8
    assert set(st["exp_avg"]) == set(st["exp_avg_sq"]) == set(eng.trainable_names()) and len(st["exp_avg"]) == 34 - 16
    back = TE._engine(3, "adam", ema_decay=0.5, freeze_layers=8)
    ckpt.load_checkpoint(path, back, model_ema=True)
    for arena in ("p32", "m32", "v32", "ema32"):
        assert torch.equal(getattr(back, arena), getattr(eng, arena)), arena
    assert back.step_count == 3 and back.ema_updates == 3
    other = TE._engine(3, "adam", ema_decay=0.5)
    with pytest.raises(ValueError, match="--freeze-layers 8, this run has --freeze-layers 0"):
        ckpt.load_checkpoint(path, other, model_ema=True)
    ckpt.load_checkpoint(path, other, model_ema=True, skip_frozen_mismatch=True)      # --eval-only
    assert torch.equal(other.p32, eng.p32)


# ------------------------------------------------------------------------------- several updates vs torch
@pytest.mark.parametrize("n", [8, 13, 16])
def test_frozen_engine_updates_match_torch_adamw_with_requires_grad_off(n):
    """Three AdamW updates (a large decay, biases at 0) of vggf-mini with the first n layers frozen: from the
    engine's own state before each step, torch.optim.AdamW over the parameters left with requires_grad on,
    stepped with the bf16-emulating chain's gradients (ops.ref.emulated_step) and the engine's exported
    moments, lands within 4 lr of every trainable weight; the frozen weights stay bit for bit where they
    started, as torch leaves them, and the moments exist for the trainable tensors only."""
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine
    from distributed_vgg_f_b200.models.vggf import build_oracle, freeze_leading_layers_, vggf_mini_spec
    from distributed_vgg_f_b200.ops import ref as R

    lr, wd = 1e-3, 100.0                          # keep = 1 - lr * wd = 0.9: the decay is visible
    spec = vggf_mini_spec(3)
    eng = NativeEngine(spec, device=torch.device(DEV), batch=4, lr=lr, seed=0, input_hw=64, distributed=False,
                       optimizer="adamw", weight_decay=wd, bias_weight_decay=0.0, freeze_layers=n,
                       init_state=build_oracle(spec, seed=0).state_dict())
    eng.train_dropout = False
    start = {k: t.to(DEV) for k, t in eng.export_state().items()}
    torch.manual_seed(4)
    for k in range(3):
        x = torch.randn(4, 3, 64, 64, device=DEV).to(BF16).float()
        y = torch.randint(0, 3, (4,), device=DEV)
        state = {name: t.to(DEV) for name, t in eng.export_state().items()}
        st = eng.export_optimizer_state()
        assert set(st["exp_avg"]) == set(eng.trainable_names()) and st["frozen_layers"] == n
        _, _, grads = R.emulated_step(spec, state, x, y)
        model = build_oracle(spec).to(DEV)
        with torch.no_grad():
            for name, p in model.named_parameters():
                p.copy_(state[name])
        frozen = set(freeze_leading_layers_(model, n))
        named = [(name, p) for name, p in model.named_parameters() if p.requires_grad]
        opt = torch.optim.AdamW([{"params": [p for name, p in named if not name.endswith(".bias")], "weight_decay": wd},
                                 {"params": [p for name, p in named if name.endswith(".bias")], "weight_decay": 0.0}],
                                lr=lr)
        for name, p in named:
            p.grad = grads[name].to(DEV).float()
            if st["step"]:
                opt.state[p] = {"step": torch.tensor(float(st["step"])), "exp_avg": st["exp_avg"][name].to(DEV),
                                "exp_avg_sq": st["exp_avg_sq"][name].to(DEV)}
        opt.step()
        want = dict(model.named_parameters())
        eng.train_step((x, y))
        eng.sync()
        got = {name: t.to(DEV) for name, t in eng.export_state().items()}
        for name in spec.param_names:
            if name in frozen:
                assert torch.equal(got[name], start[name]) and torch.equal(want[name].detach(), start[name]), name
            else:
                err = float((got[name] - want[name].detach()).abs().max())
                assert err <= 4 * lr, "step %d: %s is %.3g from torch's AdamW" % (k, name, err)
