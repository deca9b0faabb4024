"""Test-time augmentation (--val-tta) on the device: the view augment kernels of both input paths against the CPU
references on guarded operands, the view-mean reduction against float64, eval_step in every mode against the
per-view emulated forward, full-size VGG-F against the torch-op engine, the EMA pass, the distillation teacher's
score, and the launch count of an evaluation batch."""
import os

import numpy as np
import pytest
import torch

from distributed_vgg_f_b200 import ops
from distributed_vgg_f_b200.config import DATA
from distributed_vgg_f_b200.data import transforms as T
from distributed_vgg_f_b200.data.loader import FusedBatch, RaggedBatch
from distributed_vgg_f_b200.ops import ref
from distributed_vgg_f_b200.utils.metrics import DeviceMeter
from guarded import NAN, guarded

pytestmark = pytest.mark.gpu
DEV = "cuda"
MODES = ["flip", "five-crop", "ten-crop"]


def _fused(n, H, W, resize, seed=0, C=3):
    rng = np.random.default_rng(seed)
    src = torch.from_numpy(rng.integers(0, 256, (n, H, W, 3), dtype=np.uint8))
    lab = torch.from_numpy(rng.integers(0, C, n)).to(torch.int64)
    return FusedBatch(src, T.val_params(n, H, W), lab, T.resized_dims(False, H, W, resize), None)


def _ragged(sizes, resize, seed=0, C=3):
    rng = np.random.default_rng(seed)
    imgs = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in sizes]
    data = torch.from_numpy(np.concatenate([a.reshape(-1) for a in imgs]))
    params = torch.cat([T.val_params(1, h, w) for h, w in sizes])
    lab = torch.from_numpy(rng.integers(0, C, len(sizes))).to(torch.int64)
    return RaggedBatch(data, T.ragged_geometry(sizes, False, resize), params, lab, None)


# ------------------------------------------------------------------------------------- view augment kernels
@pytest.mark.parametrize("mode", MODES)
def test_augment_view_matches_the_reference_on_guarded_operands(mode):
    batch = _fused(3, 100, 130, 71, seed=1)          # resized 71 x 92: centre offsets end in .5
    n, OH = 3, 64
    src = guarded(tuple(batch.images_u8.shape), (100 * 130 * 3, 130 * 3, 3, 1), torch.uint8, 0, 255, DEV,
                  batch.images_u8)
    prm = guarded((n, 8), (8, 1), torch.float32, 0, 0.0, DEV, batch.params)
    for v in T.tta_views(mode):
        out = guarded((n, OH, OH, 4), (OH * OH * 4, OH * 4, 4, 1), torch.bfloat16, 0, NAN, DEV)
        for g in (src, prm, out):
            g.seal()
        ops.augment_view(src.t, prm.t, out.t, batch.resized_hw, v, out_hw=OH)
        torch.cuda.synchronize()
        for g, w, name in ((src, (), "src"), (prm, (), "params"), (out, (out.t,), "out")):
            g.check(w, name)
        # the chain is aug_sample's, whose bilinear blend nvcc may contract into FMAs: the output is the reference
        # rounded to bf16, give or take one rounding step (and a last-bit difference before normalisation near 0)
        want = T.augment_reference(batch.images_u8, batch.params, batch.resized_hw, out_hw=OH, view=v)
        want = want.permute(0, 2, 3, 1)
        got = out.t[..., :3].cpu().float()
        assert bool(((got - want).abs() <= want.abs() / 128 + 1e-4).all()), v
        assert float((got != want.to(torch.bfloat16).float()).float().mean()) <= 1e-2, v
        assert bool((out.t[..., 3].view(torch.int16) == 0).all())


@pytest.mark.parametrize("mode", MODES)
def test_augment_ragged_views_match_the_reference_on_guarded_operands(mode):
    """Pass 1 once over the union of the views, pass 2 per view: bit for bit the Pillow-exact reference."""
    batch = _ragged([(90, 133), (133, 90), (300, 41), (71, 71)], 71, seed=2)
    n, OH = 4, 64
    need = ops.ragged_inter_bytes(batch.geom)
    src = guarded((batch.data_u8.numel(),), (1,), torch.uint8, 0, 255, DEV, batch.data_u8)
    geom = guarded((n, 5), (5, 1), torch.int64, 0, 0, DEV, batch.geom)
    prm = guarded((n, 8), (8, 1), torch.float32, 0, 0.0, DEV, batch.params)
    inter = guarded((need,), (1,), torch.uint8, 0, 255, DEV)
    views = T.tta_views(mode)
    for i, v in enumerate(views):
        out = guarded((n, OH, OH, 4), (OH * OH * 4, OH * 4, 4, 1), torch.bfloat16, 0, NAN, DEV)
        for g in (src, geom, prm, inter, out):
            g.seal()
        ops.augment_ragged_view(src.t, geom.t, prm.t, inter.t, out.t, batch.geom, batch.params, v, out_hw=OH,
                                pass1=views if i == 0 else ())
        torch.cuda.synchronize()
        for g, w, name in ((src, (), "src"), (geom, (), "geom"), (prm, (), "params"),
                           (inter, (inter.t,) if i == 0 else (), "inter"), (out, (out.t,), "out")):
            g.check(w, name)
        want = T.ragged_reference(batch.data_u8, batch.geom, batch.params, out_hw=OH, view=v).permute(0, 2, 3, 1)
        assert torch.equal(out.t[..., :3].cpu().view(torch.int16), want.to(torch.bfloat16).view(torch.int16)), v


def test_view_entries_refuse_bad_views():
    batch = _fused(2, 80, 80, 71)
    C = ops.require()
    src, prm = batch.images_u8.to(DEV), batch.params.to(DEV)
    out = torch.empty(2, 64, 64, 4, dtype=torch.bfloat16, device=DEV)
    for view, hw in ((6, 64), (-1, 64), (T.TTA_FLIP | 7, 64), (0, 72)):
        with pytest.raises(RuntimeError):
            C.augment_view(src, prm, out, 71, 71, hw, hw, view, list(DATA.mean), list(DATA.std))


# ---------------------------------------------------------------------------------------------- reduction
def _reduce(z, t, acc, meter, loss):
    V = z.shape[0]
    for v in range(V):
        ops.tta_accumulate(z[v], t, acc, view=v, views=V, meter=meter, loss_out=loss)


@pytest.mark.parametrize("C", [3, 1000])
@pytest.mark.parametrize("b", [64, 37])
@pytest.mark.parametrize("V", [2, 5, 10])
def test_tta_accumulate_matches_float64(C, b, V):
    B = 64
    g = torch.Generator().manual_seed(C * 100 + b + V)
    z = (torch.randn(V, b, C, generator=g) * 4).to(DEV)
    t = torch.randint(0, C, (b,), generator=g).to(DEV)
    z[:, 0] = 0.0                                         # a tie across every class
    runs = []
    for _ in range(2):
        acc = torch.full((B + 1, C), NAN, dtype=torch.float32, device=DEV)   # rows >= b stay untouched
        meter = torch.zeros(4, dtype=torch.float32, device=DEV)
        loss = torch.zeros(1, dtype=torch.float32, device=DEV)
        _reduce(z, t, acc, meter, loss)
        torch.cuda.synchronize()
        assert bool(torch.isnan(acc[b:]).all())
        runs.append((acc[:b].clone(), meter.clone(), loss.clone()))
    want = ref.tta_reduce64(z.cpu(), t.cpu())
    acc, meter, loss = runs[0]
    assert float((acc.double().cpu() / V - want["probs"]).abs().max()) <= 1e-6
    assert abs(float(meter[0]) - float(want["meter"][0])) <= 1e-4 * max(1.0, float(want["meter"][0]))
    assert float(meter[1]) == float(want["meter"][1]) and float(meter[2]) == b
    assert abs(float(loss) - float(want["loss"])) <= 1e-5 * max(1.0, float(want["loss"]))
    for a, b_ in zip(runs[0], runs[1]):
        assert torch.equal(a.view(torch.int32), b_.view(torch.int32))


def test_tta_accumulate_refuses_bad_operands():
    C = ops.require()
    z = torch.zeros(4, 3, device=DEV)
    t = torch.zeros(4, dtype=torch.int64, device=DEV)
    acc = torch.zeros(4, 3, device=DEV)
    C.tta_accumulate(z, t, acc, None, None, 0, 2)
    for args in ((z, t, acc, None, None, 2, 2), (z, t, acc, None, None, -1, 2), (z, t, acc, None, None, 0, 11),
                 (z, t, acc, None, None, 0, 0), (z, t, acc[:3], None, None, 0, 2), (z, t[:3], acc, None, None, 0, 2),
                 (z, t, acc, torch.zeros(2, device=DEV), None, 0, 2)):
        with pytest.raises(RuntimeError):
            C.tta_accumulate(*args)


# ----------------------------------------------------------------------------------------------- engine
def _engine(spec, batch, hw, **kw):
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine

    os.environ.pop("B200_FUSE_POOL", None)
    return NativeEngine(spec, device=torch.device(DEV), batch=batch, lr=1e-3, seed=0, input_hw=hw, eval_hw=hw,
                        distributed=False, **kw)


def _emulated_score(spec, state, batch, hw, views):
    """float64 view-mean score of the emulated forward (ops.ref) of each view's reference input."""
    logits = []
    for v in views:
        x, y = batch.to_float("cpu", out_hw=hw, view=v)
        logits.append(ref.emulated_step(spec, {k: t.cpu() for k, t in state.items()}, x, y)[0].double())
    return ref.tta_reduce64(torch.stack(logits), batch.labels)


def _eval_meter(eng, batches, ema=False):
    m = DeviceMeter(DEV)
    eng.set_meter(m)
    for b in batches:
        eng.eval_step(b, ema=ema)
    eng.sync()
    eng.set_meter(None)
    return m.buf.double().cpu()


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("ragged", [False, True])
def test_eval_step_matches_the_emulated_forward_of_each_view(mode, ragged):
    from distributed_vgg_f_b200.models.vggf import vggf_mini_spec

    spec = vggf_mini_spec(3)
    eng = _engine(spec, 8, 64)
    eng.set_val_tta(mode)
    batch = _ragged([(90, 133), (133, 90), (71, 71), (80, 300), (100, 100)], 71, seed=4) if ragged \
        else _fused(5, 96, 120, 72, seed=4)
    got = _eval_meter(eng, [batch])
    want = _emulated_score(spec, eng.export_state(), batch, 64, T.tta_views(mode))
    assert abs(float(got[0]) - float(want["meter"][0])) <= 2e-2 * max(1.0, float(want["meter"][0]))
    assert float(got[2]) == 5
    logits = eng.forward_logits(batch)
    assert tuple(logits.shape) == (5, len(T.tta_views(mode)), 3)


def _oracle_probs(spec, state, batch, hw, views):
    from distributed_vgg_f_b200.models.vggf import build_oracle

    net = build_oracle(spec, seed=0).to(DEV).eval()
    net.load_state_dict(state)
    m = DeviceMeter(DEV)
    with torch.no_grad():
        zs = [net(batch.to_float(DEV, out_hw=hw, view=v)[0]) for v in views]
        m.add_tta(zs, batch.labels.to(DEV))
        probs = sum(torch.softmax(z, 1) for z in zs) / len(zs)
    return probs, m.buf.double().cpu()


@pytest.mark.parametrize("hw,resize", [(224, 256), (288, 320)])
def test_full_vggf_ten_crop_matches_the_torch_op_engine(hw, resize):
    from distributed_vgg_f_b200.models.vggf import vggf_spec

    spec = vggf_spec(1000)
    eng = _engine(spec, 64, hw)
    eng.set_val_tta("ten-crop")
    batch = _fused(64, 256, 300, resize, seed=5, C=1000)
    got = _eval_meter(eng, [batch])
    views = T.tta_views("ten-crop")
    probs, want = _oracle_probs(spec, eng.export_state(), batch, hw, views)
    assert abs(float(got[0]) - float(want[0])) <= 2e-2 * float(want[0])
    assert float(got[2]) == 64
    mine = sum(torch.softmax(eng.forward_logits(batch)[:, v], 1) for v in range(len(views))) / len(views)
    assert float((mine - probs).abs().max()) <= 2e-2 * float(probs.abs().max())


def test_ema_pass_and_teacher_score_use_the_views():
    from distributed_vgg_f_b200.engine.native_engine import TeacherEngine
    from distributed_vgg_f_b200.models.vggf import vggf_mini_spec

    spec = vggf_mini_spec(3)
    eng = _engine(spec, 8, 64, ema_decay=0.5)
    eng.set_val_tta("ten-crop")
    train = _fused(8, 96, 96, 72, seed=6)
    train = train._replace(params=T.sample_train_params(8, 96, 96, torch.Generator().manual_seed(0)))
    eng.train_step(train, ema=True)
    eng.prepare_ema()
    batch = _fused(6, 96, 120, 72, seed=7)
    views = T.tta_views("ten-crop")
    got = _eval_meter(eng, [batch], ema=True)
    want = _emulated_score(spec, eng.export_ema_state(), batch, 64, views)
    assert abs(float(got[0]) - float(want["meter"][0])) <= 2e-2 * max(1.0, float(want["meter"][0]))
    teacher = TeacherEngine(spec, torch.device(DEV), 8, eng.export_state(), input_hw=64, eval_hw=64)
    teacher.set_val_tta("ten-crop")
    got = _eval_meter(teacher, [batch])
    want = _emulated_score(spec, eng.export_state(), batch, 64, views)
    assert abs(float(got[0]) - float(want["meter"][0])) <= 2e-2 * max(1.0, float(want["meter"][0]))


@pytest.mark.parametrize("ragged", [False, True])
def test_launch_count_of_an_evaluation_batch(ragged):
    """V x (augment + forward + head) + V reductions; a ragged batch adds its one shared horizontal pass.  With
    "none" the count is the single-crop pass's."""
    from distributed_vgg_f_b200.models.vggf import vggf_spec

    eng = _engine(vggf_spec(3), 8, 224)
    batch = _ragged([(300, 260)] * 8, 256, seed=8) if ragged else _fused(8, 200, 240, 256, seed=8)

    def count():
        n0 = ops.launch_count()
        eng.eval_step(batch)
        eng.sync()
        return ops.launch_count() - n0

    count()
    single = count()
    eng.set_val_tta("none")
    assert count() == single
    for mode in MODES:
        eng.set_val_tta(mode)
        V = len(T.tta_views(mode))
        per_view = single - 1 if ragged else single        # a ragged single crop runs both passes
        assert count() == V * per_view + V + (1 if ragged else 0), mode
