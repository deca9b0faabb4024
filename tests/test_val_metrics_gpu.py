"""Per-class evaluation metrics (--val-metrics) on the device: class_metrics_kernel against ops.ref on guarded operands
(planted ties in logits, view sums that tie only after the division by V, two runs), the host checks, eval_step with a
confusion meter for the fused head and the GEMM + cross-entropy head in every --val-tta mode against the engine's own
forward_logits, the launch count of an evaluation batch, and a CLI run of the native engine with and without the flag."""
import contextlib
import io
import json
import os
import re

import numpy as np
import pytest
import torch

from distributed_vgg_f_b200 import ops
from distributed_vgg_f_b200.data import transforms as T
from distributed_vgg_f_b200.data.loader import FusedBatch
from distributed_vgg_f_b200.ops import ref
from distributed_vgg_f_b200.utils.metrics import DeviceMeter, class_metrics
from guarded import fmax, guarded

pytestmark = pytest.mark.gpu
DEV = "cuda"
MODES = ["none", "flip", "five-crop", "ten-crop"]
I64_POISON = torch.tensor([0x5A5A5A5A5A5A5A5A, -7], dtype=torch.int64)


# ------------------------------------------------------------------------------------------------ kernel
def _after_division_ties(n, V, seed):
    """n pairs a < a' of adjacent fp32 view sums with a / V == a' / V in fp32."""
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < n:
        a = np.float32(rng.uniform(0.05, float(V)))
        b = np.nextafter(a, np.float32(np.inf), dtype=np.float32)
        if np.float32(a / np.float32(V)) == np.float32(b / np.float32(V)):
            out.append((float(a), float(b)))
    return out


def _scores(C, b, V, seed):
    """fp32 scores [b][C] with planted ties: logits (V = 1) or view sums (V > 1), and labels."""
    g = torch.Generator().manual_seed(seed)
    t = torch.randint(0, C, (b,), generator=g)
    if V == 1:
        s = (torch.randn(b, C, generator=g) * 3).float()
        s[0] = 0.5                                            # a tie across every class
        for r in range(1, min(b, 12)):                        # ties at the maximum and at the label's score
            j, k = int(t[r]), (int(t[r]) + 1 + r) % C
            s[r, j] = s[r, k] = float(s[r].max()) + (0.0 if r % 2 else -1.0)
        return s, t
    s = torch.rand(b, C, generator=g) * (0.5 * V / C)
    for r, (a, a2) in enumerate(_after_division_ties(min(b, 16), V, seed)):
        j, k = (r * 7) % C, (r * 7 + 1 + r) % C
        if j == k:
            continue
        lo, hi = min(j, k), max(j, k)
        s[r, lo], s[r, hi] = a, a2                            # the larger sum sits at the higher index
        s[r] = torch.where(s[r] > a2, torch.full_like(s[r], a / 2), s[r])
        s[r, lo], s[r, hi] = a, a2
        t[r] = hi if r % 2 else lo
    return s.float(), t


def _guarded_launch(s, t, views, base=None):
    b, C = s.shape
    sc = guarded((b, C), (C, 1), torch.float32, 0, fmax(torch.float32), DEV, s)
    tg = guarded((b,), (1,), torch.int64, 0, 0, DEV, t)
    M0 = base if base is not None else torch.zeros(C, C, dtype=torch.int64)
    cm = guarded((C, C), (C, 1), torch.int64, 0, I64_POISON, DEV, M0)
    t5 = guarded((1,), (1,), torch.int64, 0, I64_POISON, DEV, torch.tensor([3]))
    for x in (sc, tg, cm, t5):
        x.seal()
    ops.class_metrics(sc.t, tg.t, cm.t, t5.t, views=views)
    torch.cuda.synchronize()
    for x, w, name in ((sc, (), "scores"), (tg, (), "target"), (cm, (cm.t,), "confusion"), (t5, (t5.t,), "top5")):
        x.check(w, name)
    return cm.t.cpu() - M0, int(t5.t) - 3


@pytest.mark.parametrize("C", [3, 8, 1000])
@pytest.mark.parametrize("b", [64, 37])
@pytest.mark.parametrize("V", [1, 10])
def test_kernel_matches_the_reference_on_guarded_operands(C, b, V):
    s, t = _scores(C, b, V, seed=C * 100 + b + V)
    if V > 1:                                                 # the planted pairs tie only after the division
        assert bool((s.argmax(1) != (s / V).argmax(1)).any())
    g = torch.Generator().manual_seed(b)
    base = torch.randint(0, 1000, (C, C), generator=g)       # the kernel adds to what M holds
    runs = [_guarded_launch(s, t, V, base) for _ in range(2)]
    want_M, want5 = ref.class_metrics(s, t, views=V)
    for M, top5 in runs:
        assert torch.equal(M, want_M) and top5 == want5
        assert int(M.sum()) == b
    # the engine's correct-counts use the same first maximum: compare with the loss kernels' meters
    if V == 1:
        meter = torch.zeros(4, dtype=torch.float32, device=DEV)
        ops.cross_entropy(s.to(DEV), t.to(DEV), meter=meter, loss_out=torch.zeros(1, device=DEV))
        assert int(runs[0][0].trace()) == int(meter[1])


def test_view_sums_tied_after_division_go_to_the_lower_class():
    V, C = 10, 8
    (a, a2), = _after_division_ties(1, V, seed=3)
    s = torch.zeros(2, C)
    s[:, 2], s[:, 5] = a, a2
    t = torch.tensor([5, 2])
    M, top5 = _guarded_launch(s, t, V)
    assert int(M[5, 2]) == 1 and int(M[2, 2]) == 1 and top5 == 2    # sums differ, means tie: class 2 predicted
    M1, _ = _guarded_launch(s, t, 1)
    assert int(M1[5, 5]) == 1 and int(M1[2, 5]) == 1                # undivided, class 5 is the larger


def test_rank_counts_ties_below_the_label_as_ahead():
    C = 8
    s = torch.zeros(3, C)
    s[0, :6] = 1.0                       # label 5 tied with 0..4: rank 5, not top-5
    s[1, :6] = 1.0                       # label 4: rank 4
    s[2, 7] = 2.0
    s[2, :4] = 3.0                       # label 7: four classes above it: rank 4
    M, top5 = _guarded_launch(s, torch.tensor([5, 4, 7]), 1)
    assert top5 == 2 and int(M[5, 0]) == int(M[4, 0]) == int(M[7, 0]) == 1


def test_host_checks_refuse_bad_operands():
    C = ops.require()
    s = torch.zeros(4, 3, device=DEV)
    t = torch.zeros(4, dtype=torch.int64, device=DEV)
    M = torch.zeros(3, 3, dtype=torch.int64, device=DEV)
    k = torch.zeros(1, dtype=torch.int64, device=DEV)
    C.class_metrics(s, t, M, k, 1)
    bad = ((s, t, M[:2], k, 1),                                            # undersized M
           (s, t, torch.zeros(4, 4, dtype=torch.int64, device=DEV), k, 1),   # C mismatch
           (s, t, M.view(-1), k, 1),
           (s, t, M.int(), k, 1), (s, t, M, k.int(), 1), (s.half(), t, M, k, 1), (s, t.int(), M, k, 1),
           (s, t[:3], M, k, 1), (s, t, M, k[:0], 1), (s, t, M, k, 0), (s, t, M, k, 11),
           (s.t(), t, M, k, 1), (s, t, M.cpu(), k, 1))
    for args in bad:
        with pytest.raises(RuntimeError):
            C.class_metrics(*args)


# ------------------------------------------------------------------------------------------------ engine
def _engine(spec, batch, hw):
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine

    os.environ.pop("B200_FUSE_POOL", None)
    return NativeEngine(spec, device=torch.device(DEV), batch=batch, lr=1e-3, seed=0, input_hw=hw, eval_hw=hw,
                        distributed=False, deterministic=True)


def _fused(n, H, W, resize, seed, C):
    rng = np.random.default_rng(seed)
    src = torch.from_numpy(rng.integers(0, 256, (n, H, W, 3), dtype=np.uint8))
    lab = torch.from_numpy(rng.integers(0, C, n)).to(torch.int64)
    return FusedBatch(src, T.val_params(n, H, W), lab, T.resized_dims(False, H, W, resize), None)


def _own_counts(eng, batches, C, mode):
    """The counts of the engine's own forward_logits: the logits, or their view sums rebuilt by tta_accumulate."""
    M, top5 = torch.zeros(C, C, dtype=torch.int64), 0
    for batch in batches:
        z = eng.forward_logits(batch)
        y = batch.labels
        if mode == "none":
            m, k = ref.class_metrics(z, y)
        else:
            V = z.shape[1]
            acc = torch.empty(z.shape[0], C, dtype=torch.float32, device=DEV)
            for v in range(V):
                ops.tta_accumulate(z[:, v].contiguous(), y.to(DEV), acc, view=v, views=V)
            m, k = ref.class_metrics(acc, y, views=V)
        M += m
        top5 += k
    return M, top5


@pytest.mark.parametrize("head,C", [("fused", 3), ("gemm", 1000)])
@pytest.mark.parametrize("mode", MODES)
def test_eval_step_counts_what_forward_logits_predicts(head, C, mode):
    from distributed_vgg_f_b200.models.vggf import vggf_spec

    eng = _engine(vggf_spec(C), 16, 64)
    assert eng.fused_head == (head == "fused")
    eng.set_val_tta(mode)
    batches = [_fused(16, 80, 96, 72, seed=1, C=C), _fused(9, 90, 72, 72, seed=2, C=C)]
    m = DeviceMeter(DEV, C)
    eng.set_meter(m)
    for batch in batches:
        eng.eval_step(batch)
    eng.sync()
    eng.set_meter(None)
    assert int(m.confusion.sum()) == 25 == int(m.buf[2])
    assert int(m.confusion.trace()) == int(m.buf[1])
    M, top5 = _own_counts(eng, batches, C, mode)
    assert torch.equal(m.confusion.cpu(), M) and int(m.top5) == top5
    _, acc = m.snapshot()
    assert acc.classes == class_metrics(M.numpy(), top5)


def test_ema_pass_counts_with_the_moving_average():
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine
    from distributed_vgg_f_b200.models.vggf import vggf_spec

    eng = NativeEngine(vggf_spec(3), device=torch.device(DEV), batch=8, lr=1e-3, seed=0, input_hw=64, eval_hw=64,
                       distributed=False, deterministic=True, ema_decay=0.5)
    train = _fused(8, 96, 96, 72, seed=6, C=3)
    eng.train_step(train._replace(params=T.sample_train_params(8, 96, 96, torch.Generator().manual_seed(0))), ema=True)
    eng.prepare_ema()
    batch = _fused(8, 96, 96, 72, seed=7, C=3)
    m = DeviceMeter(DEV, 3)
    eng.set_meter(m)
    eng.eval_step(batch, ema=True)
    eng.sync()
    eng.set_meter(None)
    want, _ = ref.class_metrics(eng.forward_logits(batch, ema=True), batch.labels)
    assert torch.equal(m.confusion.cpu(), want) and int(m.confusion.trace()) == int(m.buf[1])


@pytest.mark.parametrize("mode", MODES)
def test_one_more_launch_per_evaluation_batch(mode):
    from distributed_vgg_f_b200.models.vggf import vggf_spec

    eng = _engine(vggf_spec(3), 8, 224)
    eng.set_val_tta(mode)
    batch = _fused(8, 200, 240, 256, seed=8, C=3)

    def count(meter):
        eng.set_meter(meter)
        n0 = ops.launch_count()
        eng.eval_step(batch)
        eng.sync()
        return ops.launch_count() - n0

    count(None)
    plain = count(None)
    assert count(DeviceMeter(DEV)) == plain
    assert count(DeviceMeter(DEV, 3)) == plain + 1


# ---------------------------------------------------------------------------------------------------- CLI
def test_native_cli_run_with_and_without_the_flag(synth_root, tmp_path):
    from distributed_vgg_f_b200 import cli

    base = ["-iu", "tcp://127.0.0.1:29999", "-rn", "0", "-ws", "1", "-rd", synth_root, "-mb", "8", "-ep", "1",
            "--model", "vggf-mini", "--engine", "native", "--deterministic", "--model-ema", "--model-ema-steps", "1",
            "--val-tta", "flip"]
    out = {}
    for flag in (False, True):
        log = str(tmp_path / ("log%d.jsonl" % flag))
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            assert cli.main(base + ["--log-jsonl", log] + (["--val-metrics"] if flag else [])) == 0
        lines = [s for s in buf.getvalue().splitlines() if not s.startswith(("Namespace(", "[Perf]"))]
        out[flag] = (lines, json.loads(open(log).read().splitlines()[0]))
    (off, a), (on, b) = out[False], out[True]
    assert [s for s in on if s in off] == off
    new = [s for s in on if s not in off]
    assert len(new) == 2 * 4
    assert re.match(r"^\[Info\] Epoch: 1/1, test balanced acc: [\d.]+%\.$", new[0])
    assert new[1].startswith("[Info] Epoch: 1/1, test class edible: support 4, ")
    assert re.match(r"^\[Info\] Epoch: 1/1, EMA test balanced acc: [\d.]+%\.$", new[4])
    for k in a:
        if k not in ("time", "phase_ms", "host_times"):
            assert a[k] == b[k], k
    for key in ("test", "ema_test"):
        M = np.array(b[key + "_confusion"])
        assert int(M.sum()) == 12 and int(np.trace(M)) == round(b[key + "_acc"] * 12)
