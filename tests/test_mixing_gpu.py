"""Label smoothing, MixUp and CutMix on the sm_90a kernels: the mixed input transforms against the
unmixed kernel and the float oracles, the soft-target losses against float64 F.cross_entropy and
autograd, and engine steps against ops.ref.emulated_step."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _ops():
    from distributed_vgg_f_b200 import ops
    ops.require()
    return ops


def _T():
    from distributed_vgg_f_b200.data import transforms as T
    return T


# ------------------------------------------------------------------------------------- input kernels
def _uniform(b, seed=0):
    T = _T()
    g = torch.Generator().manual_seed(seed)
    src = torch.randint(0, 256, (b, 96, 112, 3), dtype=torch.uint8, generator=g)
    return src, T.sample_train_params(b, 96, 112, g)


def _ragged(b, seed=0):
    T = _T()
    g = torch.Generator().manual_seed(seed)
    sizes = [(90, 120), (300, 200), (64, 64), (150, 151), (77, 333), (40, 500), (256, 256)]
    hw = [sizes[i % len(sizes)] for i in range(b)]
    geom = T.ragged_geometry(hw, train=True)
    data = torch.randint(0, 256, (int(sum(h * w * 3 for h, w in hw)),), dtype=torch.uint8, generator=g)
    params = torch.cat([T.sample_train_params(1, h, w, g) for h, w in hw])
    return data, geom, params


def _run(ragged, b, mix, hw=64, B=8):
    """The kernel's NHWC4 output for the first b samples of a batch (the buffer holds B)."""
    ops = _ops()
    out = torch.full((B, hw, hw, 4), 7.0, dtype=torch.bfloat16, device=DEV)
    if ragged:
        data, geom, params = _ragged(b)
        inter = torch.empty(ops.ragged_inter_bytes(geom), dtype=torch.uint8, device=DEV)
        ops.augment_ragged(data.to(DEV), geom.to(DEV), params.to(DEV), inter, out[:b], geom, params, out_hw=hw, mix=mix)
    else:
        src, params = _uniform(b)
        ops.augment(src.to(DEV), params.to(DEV), out[:b], (128, 128), out_hw=hw, mode="nhwc", pad=4, mix=mix)
    torch.cuda.synchronize()
    assert bool((out[b:].float() == 7.0).all())          # nothing past the batch is written
    return out[:b]


def _reference(ragged, b, hw=64):
    T = _T()
    if ragged:
        data, geom, params = _ragged(b)
        return T.ragged_reference(data, geom, params, out_hw=hw).to(torch.float64)
    src, params = _uniform(b)
    return T.augment_reference(src, params, (128, 128), out_hw=hw).to(torch.float64)


@pytest.mark.parametrize("ragged", [False, True])
@pytest.mark.parametrize("b", [8, 5, 1])
@pytest.mark.parametrize("box", [(10, 3, 41, 60), (0, 0, 64, 64), (5, 5, 5, 9)])
def test_cutmix_is_the_partner_inside_the_box_and_the_sample_outside(ragged, b, box):
    T = _T()
    plain = _run(ragged, b, None)
    x1, y1, x2, y2 = box
    got = _run(ragged, b, T.MixDraw("cutmix", 1.0 - (x2 - x1) * (y2 - y1) / 64 ** 2, box))
    want = plain.clone()
    partner = (torch.arange(b) - 1) % b
    want[:, y1:y2, x1:x2] = plain[partner][:, y1:y2, x1:x2]
    assert torch.equal(got, want)                         # bit for bit


@pytest.mark.parametrize("ragged", [False, True])
@pytest.mark.parametrize("b", [8, 5, 1])
@pytest.mark.parametrize("lam", [0.3, 0.5, 0.93])
def test_mixup_is_within_one_bf16_rounding_of_the_float64_blend(ragged, b, lam):
    T = _T()
    got = _run(ragged, b, T.MixDraw("mixup", lam, (0, 0, 0, 0)))[..., :3].permute(0, 3, 1, 2).double().cpu()
    ref = _reference(ragged, b)
    want = lam * ref + (1.0 - lam) * ref[(torch.arange(b) - 1) % b]
    # half a bf16 ulp of the value (plus fp32 evaluation noise); the rare pixels whose nearest-neighbour
    # rotation lands on an exact tie differ from the float oracle with or without mixing
    bad = (got - want).abs() > want.abs() * 2.0 ** -8 + 1e-5
    assert float(bad.double().mean()) < 2e-3
    assert torch.count_nonzero(_run(ragged, b, T.MixDraw("mixup", lam, (0, 0, 0, 0)))[..., 3]) == 0


def test_mixed_augment_refuses_bad_draws():
    ops, T = _ops(), _T()
    src, params = _uniform(2)
    out = torch.empty(2, 64, 64, 4, dtype=torch.bfloat16, device=DEV)
    n0 = ops.launch_count()
    for mix in (T.MixDraw("cutmix", 0.5, (0, 0, 65, 10)), T.MixDraw("cutmix", 0.5, (20, 0, 10, 10)),
                T.MixDraw("mixup", 1.5, (0, 0, 0, 0))):
        with pytest.raises(RuntimeError):
            ops.augment(src.to(DEV), params.to(DEV), out, (128, 128), out_hw=64, mode="nhwc", pad=4, mix=mix)
    with pytest.raises(ValueError):
        ops.augment(src.to(DEV), params.to(DEV), out, (128, 128), out_hw=64, mode="im2col", pad=64,
                    mix=T.MixDraw("mixup", 0.5, (0, 0, 0, 0)))
    assert ops.launch_count() == n0


# -------------------------------------------------------------------------------------- loss kernels
_FORMS = ["smooth", "mixup", "mixup+smooth", "cutmix-tie"]


def _form(form):
    """(eps, MixDraw or None)."""
    T = _T()
    return {"smooth": (0.1, None), "mixup": (0.0, T.MixDraw("mixup", 0.37, (0, 0, 0, 0))),
            "mixup+smooth": (0.2, T.MixDraw("mixup", 0.81, (0, 0, 0, 0))),
            "cutmix-tie": (0.05, T.MixDraw("cutmix", 0.5, (0, 0, 112, 224)))}[form]


def _expected(logits, target, C, eps, mix, cw):
    """float64 F.cross_entropy on torchvision's targets, its autograd dlogits, and the meter."""
    T = _T()
    z = logits.double().cpu().requires_grad_(True)
    t = target.cpu()
    tgt = t if mix is None else T.mixed_targets(t, C, mix).double()
    w = None if cw is None else cw.double().cpu()
    loss = F.cross_entropy(z, tgt, weight=w, label_smoothing=eps)
    loss.backward()
    cls = t if mix is None else T.mixed_targets(t, C, mix).argmax(1)      # float32 targets, first maximum
    correct = int((z.detach().argmax(1) == cls).sum())
    return float(loss.detach()), z.grad, correct


def _check(loss, dl, meter, B, exp):
    want_loss, want_dl, correct = exp
    assert abs(loss - want_loss) <= 1e-4 * max(1.0, abs(want_loss)), (loss, want_loss)
    err = (dl - want_dl).abs()
    assert bool((err <= want_dl.abs() * 2.0 ** -8 + 1e-6 * float(want_dl.abs().max()) + 1e-9).all()), float(err.max())
    assert abs(float(meter[0]) - want_loss * B) <= 1e-4 * max(1.0, abs(want_loss)) * B
    assert int(meter[1]) == correct and int(meter[2]) == B


def _labels(B, C, g):
    y = torch.randint(0, C, (B,), generator=g)
    if B > 3:
        y[2] = y[1]                                # a row whose partner has the same label
    return y


@pytest.mark.parametrize("C", [3, 10, 1000])
@pytest.mark.parametrize("B", [1, 7, 64, 256])
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("form", _FORMS)
def test_cross_entropy_soft_matches_float64_cross_entropy(C, B, weighted, form):
    ops = _ops()
    g = torch.Generator().manual_seed(C * 1000 + B)
    logits = (torch.randn(B, C, generator=g) * 3).to(DEV)
    if B > 4:
        logits[4, 1] = logits[4, 0] = logits[4].max() + 1          # a tie: the first maximum counts
    y = _labels(B, C, g)
    cw = (torch.rand(C, generator=g) + 0.5).to(DEV) if weighted else None
    eps, mix = _form(form)
    ldd = C + (8 - C % 8) % 8
    dl = torch.full((B, ldd), 9.0, dtype=torch.bfloat16, device=DEV)
    meter = torch.zeros(4, device=DEV)
    loss = torch.zeros(1, device=DEV)
    ops.cross_entropy(logits, y.to(DEV), dl, ldd, meter, loss, class_weights=cw, label_smoothing=eps, mix=mix)
    torch.cuda.synchronize()
    assert torch.count_nonzero(dl[:, C:]) == 0
    _check(float(loss), dl[:, :C].double().cpu(), meter.cpu(), B, _expected(logits, y, C, eps, mix, cw))


@pytest.mark.parametrize("C", [2, 3, 8])
@pytest.mark.parametrize("B", [1, 7, 64, 256])
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("form", _FORMS)
def test_head_ce_soft_matches_float64_cross_entropy_and_its_backward(C, B, weighted, form):
    ops = _ops()
    from distributed_vgg_f_b200.ops import ref as R

    K = 512
    g = torch.Generator().manual_seed(C * 1000 + B + 7)
    h = torch.relu(torch.randn(B, K, generator=g)).to(torch.bfloat16).to(DEV)
    W = (torch.randn(C, K, generator=g) * 0.05).to(torch.bfloat16).to(DEV)
    bias = (torch.randn(C, generator=g) * 0.1).to(DEV)
    y = _labels(B, C, g)
    cw = (torch.rand(C, generator=g) + 0.5).to(DEV) if weighted else None
    eps, mix = _form(form)
    logits = torch.empty(B, C, device=DEV)
    dl = torch.zeros(B, 8, dtype=torch.bfloat16, device=DEV)
    dW = torch.full((C, K), 3.0, device=DEV)
    db = torch.full((C,), 0.25, device=DEV)
    dh = torch.empty(B, K, dtype=torch.bfloat16, device=DEV)
    meter = torch.zeros(4, device=DEV)
    loss = torch.zeros(1, device=DEV)
    _ops().require().head_ce(h, W, bias, y.to(DEV), logits, dl, 8, dW, db, dh, 2.0, True, meter, loss, cw, False,
                             ops.soft_targets(eps, mix))
    torch.cuda.synchronize()
    exp = _expected(logits, y, C, eps, mix, cw)
    _check(float(loss), dl[:, :C].double().cpu(), meter.cpu(), B, exp)
    ref = R.head_ce64(h, W, bias, dl_used=dl[:, :C], drop_scale=2.0, relu=True)
    lr, lm = ref["logits"]
    assert bool(((logits.double() - lr).abs() <= 1e-4 * lm + 1e-6).all())
    for name, got in (("dW", dW), ("db", db - 0.25)):
        r, m = ref[name]
        assert bool(((got.double() - r).abs() <= 1e-4 * m + 1e-9).all()), name
    r, m = ref["dh"]
    assert bool(((dh.double() - r).abs() <= r.abs() * 2.0 ** -8 + 1e-5 * m + 1e-12).all())


# ------------------------------------------------------------------------------------------- engine
def _engine(classes, batch=4, **kw):
    import os

    from distributed_vgg_f_b200.engine.native_engine import NativeEngine
    from distributed_vgg_f_b200.models.vggf import build_oracle, vggf_mini_spec

    os.environ["B200_FUSE_POOL"] = "0"       # the un-pooled activations gate the reference's backward
    try:
        spec = vggf_mini_spec(classes)
        oracle = build_oracle(spec, seed=0)
        with torch.no_grad():
            for p in oracle.parameters():
                if p.dim() > 1:
                    p.copy_(p.to(torch.bfloat16).float())
        eng = NativeEngine(spec, device=torch.device(DEV), batch=batch, lr=1e-3, seed=0, input_hw=64,
                           init_state=oracle.state_dict(), **kw)
    finally:
        os.environ.pop("B200_FUSE_POOL", None)
    return spec, oracle, eng


def _fused_batch(b, mix, seed=3, classes=3):
    from distributed_vgg_f_b200.data.loader import FusedBatch

    T = _T()
    g = torch.Generator().manual_seed(seed)
    src = torch.randint(0, 256, (b, 128, 128, 3), dtype=torch.uint8, generator=g)
    params = T.sample_train_params(b, 128, 128, g)
    y = torch.randint(0, classes, (b,), generator=g)
    return FusedBatch(src, params, y, (80, 80), None, mix)


@pytest.mark.parametrize("classes", [3, 10])          # fused head / GEMM head + cross_entropy kernel
@pytest.mark.parametrize("form", ["smooth", "mixup", "cutmix", "cutmix+smooth"])
@pytest.mark.parametrize("b", [4, 3])
def test_engine_step_matches_emulated_step_on_the_same_mixed_inputs(capsys, classes, form, b):
    from distributed_vgg_f_b200.models import layout as L
    from distributed_vgg_f_b200.ops import ref as R

    T = _T()
    eps = 0.1 if "smooth" in form else 0.0
    mix = {"smooth": None, "mixup": T.MixDraw("mixup", 0.3, (0, 0, 0, 0)),
           "cutmix": T.MixDraw("cutmix", 1 - 40 * 30 / 64 ** 2, (20, 10, 60, 40)),
           "cutmix+smooth": T.MixDraw("cutmix", 1 - 64 * 20 / 64 ** 2, (0, 30, 64, 50))}[form]
    spec, oracle, eng = _engine(classes, label_smoothing=eps)
    assert eng.fused_head == (classes <= 8)
    eng.train_dropout = False
    eng.apply_updates = False
    batch = _fused_batch(b, mix, classes=classes)
    got_loss = float(eng.train_step(batch))
    eng.sync()
    x = eng.x_nhwc[:b, ..., :3].permute(0, 3, 1, 2).float()       # the mixed input the kernel wrote
    # which is the mixed transform of the batch
    plain = T.augment_reference(batch.images_u8.to(DEV), batch.params, (80, 80), out_hw=64)
    want_x = T.apply_mix(plain, batch.labels.to(DEV), mix)
    assert float((x - want_x).abs().median()) < 5e-3
    override = {"acts": [a[:b].permute(0, 3, 1, 2).float() for a in eng.acts],
                "feat": eng.feat.permute(0, 3, 1, 2).float(),
                "fc_y": [t[:b].float() if t is not None else None for t in eng.fc_y],
                "logits": eng.logits[:b].clone()}
    soft = None if mix is None else T.mixed_targets(batch.labels, classes, mix).to(DEV)
    state = {k: v.detach().to(DEV) for k, v in oracle.state_dict().items()}
    _, loss, grads = R.emulated_step(spec, state, x, batch.labels.to(DEV), override=override, soft_target=soft,
                                     label_smoothing=eps)
    assert abs(got_loss - float(loss)) < 1e-4
    worst = {}
    for name in spec.param_names:
        ref = L.to_native(spec, name, grads[name])
        g = eng._view(eng.g32, name)
        worst[name] = max(float((g - ref).abs().max() / (ref.abs().max() + 1e-12)),
                          float((g - ref).norm() / (ref.norm() + 1e-20)))
    with capsys.disabled():
        print("\n[grad err, %s, C=%d, b=%d] worst %.1e" % (form, classes, b, max(worst.values())))
    bad = {k: v for k, v in worst.items() if v > 2e-2}
    assert not bad, bad


def test_eval_loss_stays_plain_cross_entropy():
    from distributed_vgg_f_b200.utils.metrics import DeviceMeter

    _, _, eng = _engine(3, label_smoothing=0.3)
    batch = _fused_batch(4, None)
    meter = DeviceMeter(DEV)
    eng.set_meter(meter)
    eng.eval_step(batch)
    eng.sync()
    want = F.cross_entropy(eng.logits[:4].double(), batch.labels.to(DEV))
    assert abs(meter.snapshot()[0].average - float(want)) < 1e-4


class _Recorder:
    """Stands in for ops._C and records every native call: its name and its arguments (tensors by shape
    and dtype, everything else by value)."""

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


@pytest.mark.parametrize("ragged", [False, True])
def test_flags_off_run_the_calls_of_an_engine_without_the_arguments(ragged, monkeypatch):
    """With the flags at 0 the engine makes exactly the native calls, with the same arguments, and the same
    launches as an engine built without them, over a gradient-only step and two update steps.  The
    gradients of the first step, taken from the same weights, agree up to the order of the fp32 split-K
    red.adds, which varies from run to run (after an update that order has already moved the weights, and
    Adam turns the difference into one of up to lr per weight, so later steps are not compared)."""
    from distributed_vgg_f_b200.data.loader import RaggedBatch

    ops = _ops()
    if ragged:
        data, geom, params = _ragged(4)
        batch = RaggedBatch(data, geom, params, torch.tensor([0, 2, 1, 1]), None)
    else:
        batch = _fused_batch(4, None)
    runs = []
    for kw in ({}, {"label_smoothing": 0.0}):
        rec = _Recorder(ops.require())
        monkeypatch.setattr(ops, "_C", rec)
        _, _, eng = _engine(3, **kw)
        eng.train_dropout = False
        counts, grads = [], None
        for k in range(3):
            eng.apply_updates = k > 0
            n0 = ops.launch_count()
            eng.train_step(batch)
            eng.sync()
            counts.append(ops.launch_count() - n0)
            if k == 0:                   # raw gradients of the initial weights; the update steps start from zero
                grads = eng.g32.clone()
                eng.g32.zero_()
        monkeypatch.undo()
        runs.append((rec.calls, counts, grads))
    assert runs[0][0] == runs[1][0] and runs[0][1] == runs[1][1]
    names = {c[0] for c in runs[0][0]}
    assert not names & {"augment_mixed", "augment_ragged_mixed", "cross_entropy_soft"}
    assert all(len(c[1]) <= 16 for c in runs[0][0] if c[0] == "head_ce")        # no soft-target argument
    a, r = runs[1][2], runs[0][2]
    assert float((a - r).norm() / r.norm()) < 1e-3 and float((a - r).abs().max() / r.abs().max()) < 1e-2


def test_mixed_training_steps_are_finite():
    T = _T()
    _, _, eng = _engine(3, batch=8, label_smoothing=0.1)
    eng.train_dropout = False
    losses = []
    for k in range(30):
        mix = T.draw_mix(0.2, 1.0, 0, 0, 0, k, hw=64)
        losses.append(float(eng.train_step(_fused_batch(8, mix, seed=1))))
    assert all(v == v and abs(v) < 1e3 for v in losses)
