"""--deterministic on the GPU: the PARTIAL split-K epilogues, splitk_reduce and colsum_det against float64
references and, bit for bit, against the fp32-order emulation; and whole training runs repeated from the
same seed.  Every comparison of two runs is two runs compared once."""
import pytest
import torch

import kernel_check as K
from distributed_vgg_f_b200.ops import ref as R

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
POISON = float("nan")


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from distributed_vgg_f_b200 import ops as O
    O.require()
    torch.cuda.set_device(0)
    return O


def _workspace(splits: int, slice_elems: int, tail: int = 4096):
    """A poisoned workspace with room for ``tail`` floats a launch must leave alone."""
    return torch.full((splits * slice_elems + tail,), POISON, dtype=torch.float32, device=DEV)


def _slices(ws, splits, slice_elems, n):
    """The slices a launch wrote as [splits, n]; everything behind them must still be poison and every
    slice element must have been written."""
    used = splits * slice_elems
    assert bool(torch.isnan(ws[used:]).all()), "a partial launch wrote behind its slices"
    s = ws[:used].view(splits, slice_elems)[:, :n]
    assert not bool(torch.isnan(s).any()), "a slice element was left unwritten"
    return s


def _check_reduce(ops, ws, s, dst_shape, slice_elems, alpha=1.0):
    """splitk_reduce of the slices ``s`` (a view of ``ws``), with and without accumulate, bit for bit
    against the ordered fp32 emulation."""
    splits, n = s.shape
    for accumulate in (False, True):
        dst = torch.randn(dst_shape, device=DEV)
        before = dst.clone()
        ops.splitk_reduce(ws, dst, n, splits, slice_elems=slice_elems, alpha=alpha, accumulate=accumulate)
        want = R.splitk_reduce_ordered(s, before.flatten()[:n] if accumulate else None, alpha)
        assert torch.equal(dst.flatten()[:n].cpu(), want), "splitk_reduce differs from the fp32-order emulation"
        assert torch.equal(dst.flatten()[n:], before.flatten()[n:])


# ------------------------------------------------------------------------------------ the reducer
@pytest.mark.parametrize("n,splits,slice_elems", [(4096, 1, 4096), (4096, 7, 4096), (1000, 13, 1000),
                                                  (1002, 6, 1004), (64 * 4096, 8, 64 * 4096), (6, 3, 8)])
def test_splitk_reduce_matches_the_ordered_emulation_and_float64(ops, n, splits, slice_elems):
    """Slice counts around the four-loads-in-flight unroll, an element count that is not whole float4s (the
    scalar tail, with the slices still float4-aligned), with and without accumulate and alpha."""
    g = torch.Generator(device=DEV).manual_seed(n + splits)
    ws = torch.randn(splits * slice_elems + 64, generator=g, device=DEV)
    s = ws[:splits * slice_elems].view(splits, slice_elems)[:, :n]
    for alpha in (1.0, 0.37):
        _check_reduce(ops, ws, s, (n + 8,), slice_elems, alpha)
    dst = torch.zeros(n, device=DEV)
    ops.splitk_reduce(ws, dst, n, splits, slice_elems=slice_elems, alpha=0.37)
    ref, err = R.splitk_reduce64(s, None, 0.37)
    assert bool(((dst.double() - ref).abs() <= 2 * err + 1e-300).all())


def test_splitk_reduce_refuses_bad_workspaces(ops):
    ws, dst = torch.zeros(4096, device=DEV), torch.zeros(1024, device=DEV)
    with pytest.raises(RuntimeError, match="workspace holds"):
        ops.splitk_reduce(ws, dst, 1024, 5, slice_elems=1024)
    with pytest.raises(RuntimeError, match="aligned"):
        ops.splitk_reduce(ws[1:], dst, 1024, 2, slice_elems=1024)
    with pytest.raises(RuntimeError, match="float4"):
        ops.splitk_reduce(ws, dst, 1000, 2, slice_elems=1002)
    with pytest.raises(RuntimeError, match="dst must hold"):
        ops.splitk_reduce(ws, dst, 2048, 2, slice_elems=2048)


# ------------------------------------------------------------------------------------ column sums
@pytest.mark.parametrize("C", [64, 128, 256, 512, 4096])
@pytest.mark.parametrize("rows", [64, 1000, 12544])
def test_colsum_det(ops, C, rows):
    C_ = ops.require()
    gen = K.generator(C + rows, DEV)
    dz = K.operand((rows, C), "gauss", rows, gen, DEV)
    blocks = C_.colsum_partial_blocks(rows, C, C_.sm_count())
    ws = _workspace(blocks, C)
    assert C_.colsum_partial(dz, ws, rows, C, 1.0) == blocks
    s = _slices(ws, blocks, C, C)
    ref, mag = R.bias_grad64(dz, C, rows=rows)
    K.check(s.double().sum(0), ref, mag, chain=rows, exact=False, family="colsum_det", what="C%d rows%d" % (C, rows))
    _check_reduce(ops, ws, s, (C,), C)
    db = torch.ones(C, device=DEV)
    assert ops.colsum_det(dz, db, ws, rows, C, accumulate=True) == blocks
    assert torch.equal(db.cpu(), R.splitk_reduce_ordered(s, torch.ones(C)))
    with pytest.raises(RuntimeError, match="workspace must hold"):
        C_.colsum_partial(dz, ws[:blocks * C - 4], rows, C, 1.0)


# ---------------------------------------------------------------------------- convolution wgrads
# (N, H, Cin, Cout): the halo kernel (Cin 64), the generic kernel at 64-, 128- and 256-wide tiles, and a
# pixel count whose last split is ragged
WGRAD_SHAPES = [(4, 32, 64, 64), (2, 16, 64, 128), (4, 28, 128, 256), (8, 14, 256, 512), (64, 14, 512, 512),
                (3, 14, 128, 128), (2, 12, 64, 64)]


@pytest.mark.parametrize("N,H,Cin,Cout", WGRAD_SHAPES)
def test_conv_wgrad_partial(ops, N, H, Cin, Cout):
    C_ = ops.require()
    gen = K.generator(N * H + Cin + Cout, DEV)
    dz = K.operand((N, H, H, Cout), "gauss", N * H * H, gen, DEV)
    x = K.operand((N, H, H, Cin), "gauss", N * H * H, gen, DEV)
    n = Cout * 9 * Cin
    splits = C_.conv_wgrad_splits(N, H, H, Cin, Cout, C_.sm_count())
    ws = _workspace(splits, n)
    assert C_.conv_wgrad_partial(dz, x, ws, 1.0) == splits
    s = _slices(ws, splits, n, n)
    ref, mag = R.conv3x3_wgrad64(dz, x)
    K.check(s.double().sum(0).view_as(ref), ref, mag, chain=N * H * H, exact=False, family="wgrad_partial",
            what="%dx%d^2 %d->%d, %d splits" % (N, H, Cin, Cout, splits))
    _check_reduce(ops, ws, s, (Cout, 3, 3, Cin), n)
    with pytest.raises(RuntimeError, match="workspace holds"):
        C_.conv_wgrad_partial(dz, x, ws[:splits * n - 4], 1.0)


@pytest.mark.parametrize("N,H", [(1, 8), (2, 64), (8, 224)])
def test_conv0_wgrad_partial(ops, N, H):
    """(1, 8): one 64-pixel k-block, so the CTA's second consumer has none and its slice must be zeros."""
    C_ = ops.require()
    gen = K.generator(N + H, DEV)
    dz = K.operand((N, H, H, 64), "gauss", N * H * H, gen, DEV)
    x4 = K.operand((N, H, H, 4), "gauss", N * H * H, gen, DEV)
    x4[..., 3] = 0
    splits = C_.conv0_wgrad_splits(N, H, H, C_.sm_count())
    ws = _workspace(splits, 4096)
    assert C_.conv0_wgrad_partial(dz, x4, ws) == splits
    s = _slices(ws, splits, 4096, 4096)
    if (N, H) == (1, 8):
        assert splits == 2 and bool((s[1] == 0).all()) and bool((s[0] != 0).any())
    ref, mag = R.conv0_wgrad64(dz, x4)
    K.check(s.double().sum(0).view_as(ref), ref, mag, chain=N * H * H, exact=False, family="conv0_partial",
            what="%dx%d^2" % (N, H))
    _check_reduce(ops, ws, s, (64, 64), 4096)


# ------------------------------------------------------------------------------------------ GEMMs
# FC forward (K-major A), FC dgrad (MN-major A) at a ragged batch, and the im2col layer-0 wgrad
@pytest.mark.parametrize("M,N,Kd,a_mn,b_mn,transposed,ksplit", [
    (4096, 64, 25088, False, False, True, 8), (512, 64, 4096, False, False, True, 64),
    (4096, 30, 4096, True, False, True, 8), (1000, 64, 4096, False, False, True, 8),
    (64, 64, 64 * 56 * 56, True, True, False, 296)])
def test_gemm_partial(ops, M, N, Kd, a_mn, b_mn, transposed, ksplit):
    C_ = ops.require()
    gen = K.generator(M + N + Kd, DEV)
    a = K.operand((Kd, M) if a_mn else (M, Kd), "gauss", Kd, gen, DEV, scale=0.1)
    b = K.operand((Kd, N) if b_mn else (N, Kd), "gauss", Kd, gen, DEV)
    n, splits = M * N, C_.gemm_splits(Kd, ksplit)
    se = C_.workspace_slice(n)
    ws = _workspace(splits, se)
    assert C_.gemm_partial(a, a_mn, b, b_mn, M, N, Kd, ws, M if transposed else N, transposed, 1.0, ksplit, 0) == splits
    s = _slices(ws, splits, se, n)
    ref, mag = R.gemm64(a, b, M=M, N=N, K=Kd, a_mn=a_mn, b_mn=b_mn, epi="f32_atomic_t" if transposed else "f32_atomic")
    K.check(s.double().sum(0).view_as(ref), ref, mag, chain=Kd, exact=False, family="gemm_partial",
            what="%dx%dx%d" % (M, N, Kd))
    _check_reduce(ops, ws, s, tuple(ref.shape), se)


# ---------------------------------------------------------------------------------- whole steps
def _batches(count, b, classes, hw=256, seed=11, mix=True):
    from distributed_vgg_f_b200.data import transforms as T
    from distributed_vgg_f_b200.data.loader import FusedBatch

    out = []
    for k in range(count):
        g = torch.Generator().manual_seed(seed + k)
        src = torch.randint(0, 256, (b, hw, hw, 3), dtype=torch.uint8, generator=g)
        params = T.sample_train_params(b, hw, hw, g)
        y = torch.randint(0, classes, (b,), generator=g)
        draw = T.MixDraw("mixup", 0.3 + 0.03 * k, (0, 0, 0, 0)) if mix else None
        out.append(FusedBatch(src, params, y, (hw, hw), None, draw))
    return out


def _train(spec, batches, *, batch, hw, accum, **kw):
    """A fresh engine, one update per ``accum`` batches; the state afterwards and every batch's loss."""
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine

    eng = NativeEngine(spec, device=torch.device(DEV), batch=batch, lr=1e-3, seed=5, input_hw=hw, **kw)
    losses = []
    for k, bt in enumerate(batches):
        update = (k + 1) % accum == 0
        losses.append(eng.train_step(bt, update=update, ema=update and eng.ema32 is not None).clone())
    eng.sync()
    state = {n: getattr(eng, n).clone() for n in ("p32", "m32", "v32", "ema32", "w16") if getattr(eng, n) is not None}
    state["loss"] = torch.cat(losses)
    return eng, state


def _assert_same(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert torch.equal(a[k], b[k]), "%s differs between two runs from the same seed" % k
    assert bool(torch.isfinite(a["loss"]).all())


def test_vggf_trains_bit_for_bit_twice(ops):
    """Full VGG-F, batch 64, 224^2, Adam, dropout, label smoothing, MixUp, two batches per update, EMA: ten
    updates, run twice from the same seed with two fresh engines."""
    from distributed_vgg_f_b200.models.vggf import vggf_spec

    spec, batches = vggf_spec(3), _batches(20, 64, 3)
    kw = dict(batch=64, hw=224, accum=2, optimizer="adam", label_smoothing=0.1, ema_decay=0.9, weight_decay=1e-4,
              deterministic=True)
    e1, s1 = _train(spec, batches, **kw)
    assert e1._ws is not None and e1.ema_updates == 10
    del e1
    _, s2 = _train(spec, batches, **kw)
    _assert_same(s1, s2)


@pytest.mark.parametrize("model,optimizer", [("vgg16", "adam"), ("vggf", "sgd")])
def test_gemm_head_and_sgd_train_bit_for_bit_twice(ops, model, optimizer):
    """VGG-16 with 1000 classes (the GEMM head and cross_entropy kernel) and SGD: three updates of two batches."""
    from distributed_vgg_f_b200.models import get_spec

    classes = 1000 if model == "vgg16" else 3
    spec, batches = get_spec(model, classes), _batches(6, 16, classes)
    kw = dict(batch=16, hw=224, accum=2, optimizer=optimizer, momentum=0.9, deterministic=True)
    e1, s1 = _train(spec, batches, **kw)
    assert e1.fused_head == (model != "vgg16")
    del e1
    _, s2 = _train(spec, batches, **kw)
    _assert_same(s1, s2)


def test_first_step_gradients_agree_with_the_default_step(ops):
    """Same weights, same batch, no update: the deterministic gradients differ from the atomic ones by
    summation order only."""
    from distributed_vgg_f_b200.models.vggf import vggf_spec

    spec, batches = vggf_spec(3), _batches(1, 16, 3, mix=False)
    grads = []
    for det in (False, True):
        from distributed_vgg_f_b200.engine.native_engine import NativeEngine
        eng = NativeEngine(spec, device=torch.device(DEV), batch=16, lr=1e-3, seed=5, deterministic=det)
        eng.apply_updates = False
        eng.train_step(batches[0])
        eng.sync()
        grads.append((eng, eng.g32.clone()))
    (eng, g0), (_, g1) = grads
    for name in eng.plan.order:
        a, b = eng._view(g0, name).double(), eng._view(g1, name).double()
        scale = float(a.abs().max()) + 1e-30
        assert float((a - b).abs().max()) <= 2e-3 * scale, name


def test_flag_off_is_the_engine_without_the_argument(ops, monkeypatch):
    import test_ema_gpu as TE

    runs = []
    for kw in ({}, {"deterministic": False}):
        rec = TE._Recorder(ops.require())
        monkeypatch.setattr(ops, "_C", rec)
        eng = TE._engine(3, "adam", **kw)
        counts = []
        for k in range(3):
            n0 = ops.launch_count()
            eng.train_step(TE._batch(4), update=k != 1)
            eng.sync()
            counts.append(ops.launch_count() - n0)
        monkeypatch.undo()
        assert eng._ws is None
        runs.append((list(rec.calls), counts))
    assert runs[0] == runs[1]
    assert not any(c[0] in ("splitk_reduce", "colsum_partial", "conv_wgrad_partial", "gemm_partial") for c in runs[0][0])


def test_deterministic_mini_engine_uses_no_atomic_split(ops, monkeypatch):
    """Under the flag no split-K GEMM, no conv wgrad and no fused column sum is launched in its atomic form."""
    import test_ema_gpu as TE

    rec = TE._Recorder(ops.require())
    monkeypatch.setattr(ops, "_C", rec)
    eng = TE._engine(3, "adam", deterministic=True)
    eng.train_step(TE._batch(4))
    eng.sync()
    monkeypatch.undo()
    names = [c[0] for c in rec.calls]
    assert "conv_wgrad" not in names and "conv0_wgrad" not in names
    assert "conv_wgrad_partial" in names and "splitk_reduce" in names and "colsum_partial" in names
    C = ops.require()
    for name, args, _ in rec.calls:
        if name == "gemm":
            assert args[9] not in (C.EPI_F32_ATOMIC_T,) and (args[9] != C.EPI_F32_ATOMIC or args[12] <= 1)
        if name == "conv_dgrad":
            assert args[4] is None
        if name in ("unpool2x2", "maxpool_relu_bwd"):
            assert args[3] is None


def test_nvls_is_refused(ops):
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine
    from distributed_vgg_f_b200.models.vggf import vggf_mini_spec

    with pytest.raises(ValueError, match="nvls"):
        NativeEngine(vggf_mini_spec(3), device=torch.device(DEV), batch=4, input_hw=64, allreduce="nvls",
                     deterministic=True)
