"""Per-class evaluation metrics (--val-metrics) without a GPU: the flag, the derivations against numpy on hand-built
matrices, the DeviceMeter counts of both torch-op reductions against numpy and ops.ref with tied scores, CLI runs with
and without the flag (raw weights, EMA, --eval-only), and --shard-eval at two gloo ranks."""
import contextlib
import io
import json
import re
import socket

import numpy as np
import pytest
import torch

from distributed_vgg_f_b200.ops import ref
from distributed_vgg_f_b200.utils.metrics import DeviceMeter, class_metrics, class_report

BASE = ["-iu", "tcp://127.0.0.1:29999", "-rn", "0", "-ws", "1", "-nc", "-mb", "4", "--model", "vggf-tiny",
        "--engine", "oracle", "--train-crop-size", "64", "--val-crop-size", "64", "--train-resize-size", "72",
        "--val-resize-size", "72"]
NEW_KEYS = {"confusion", "support", "recall", "precision", "balanced_acc"}


def _parse(extra):
    from distributed_vgg_f_b200 import cli
    return cli.parse_command_line(["-iu", "x", "-rn", "0", "-ws", "1", "-rd", "/r"] + extra, init=False)


# ------------------------------------------------------------------------------------------------ flag
def test_flag_is_off_by_default_and_leaves_the_namespace_alone():
    args = _parse([])
    assert not getattr(args, "val_metrics", False)
    assert "val_metrics" not in vars(args)          # the printed namespace and checkpoint args are unchanged
    assert _parse(["--val-metrics"]).val_metrics is True


# ----------------------------------------------------------------------------------------- derivations
def _numpy_metrics(M):
    M = np.asarray(M, dtype=np.float64)
    rows, cols, d = M.sum(1), M.sum(0), np.diag(M)
    with np.errstate(invalid="ignore", divide="ignore"):
        recall, precision = d / rows, d / cols
    return recall, precision, np.nanmean(recall)


def _same(got, want):
    """None where numpy has NaN, else equal to 1e-12."""
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert (g is None) == bool(np.isnan(w)), (got, want)
        assert g is None or abs(g - w) <= 1e-12


def test_class_without_support_and_class_never_predicted():
    M = [[3, 1, 0, 0],
         [0, 0, 0, 0],           # class 1: no support -> recall undefined, left out of the balanced accuracy
         [2, 0, 5, 0],
         [1, 0, 1, 0]]           # class 3: never predicted -> precision undefined
    m = class_metrics(M)
    recall, precision, bal = _numpy_metrics(M)
    _same(m["recall"], recall)
    _same(m["precision"], precision)
    assert m["recall"][1] is None and m["precision"][3] is None and m["precision"][1] == 0.0
    assert abs(m["balanced_acc"] - bal) <= 1e-12
    assert abs(m["balanced_acc"] - (3 / 4 + 5 / 7 + 0) / 3) <= 1e-12
    assert m["support"] == [4, 0, 7, 2] and m["confusion"] == M
    assert "acc5" not in m                          # C <= 5: no top-5


def test_balanced_accuracy_is_sklearns_formula():
    rng = np.random.default_rng(3)
    y = rng.integers(0, 7, 400)
    y[y == 4] = 5                                   # one class without support
    p = np.where(rng.random(400) < 0.6, y, rng.integers(0, 7, 400))
    M = np.zeros((7, 7), np.int64)
    np.add.at(M, (y, p), 1)
    m = class_metrics(M, top5=321)
    per = np.array([M[c, c] / M[c].sum() for c in range(7) if M[c].sum()])
    assert abs(m["balanced_acc"] - per.mean()) <= 1e-12
    assert m["acc5"] == 321 / 400


@pytest.mark.parametrize("C", [5, 6])
def test_acc5_only_above_five_classes(C):
    m = class_metrics(np.eye(C, dtype=np.int64), top5=C)
    assert ("acc5" in m) == (C > 5)
    lines = class_report("Epoch: 1/1, ", "test", m)
    assert ("acc@5" in lines[0]) == (C > 5) and len(lines) == 1 + C


def test_undefined_ratios_are_null_in_json_and_dashes_in_the_report():
    m = class_metrics(np.zeros((6, 6), np.int64), top5=0)
    text = json.dumps(m)
    assert "NaN" not in text and json.loads(text)["balanced_acc"] is None and json.loads(text)["acc5"] is None
    lines = class_report("Evaluation: ", "EMA test", m, ["a", "b"])
    assert lines[0] == "[Info] Evaluation: EMA test balanced acc: -, EMA test acc@5: -."
    assert lines[1] == ("[Info] Evaluation: EMA test class a: support 0, recall -, precision -, "
                        "confusion row [0, 0, 0, 0, 0, 0].")
    assert lines[3].startswith("[Info] Evaluation: EMA test class 2: ")   # unnamed classes go by index


def test_report_stops_listing_classes_above_32():
    assert len(class_report("", "test", class_metrics(np.eye(32, dtype=np.int64), 32))) == 33
    assert len(class_report("", "test", class_metrics(np.eye(33, dtype=np.int64), 33))) == 1


# ------------------------------------------------------------------------------------------ the counts
def _numpy_counts(scores, target):
    """First maximum and the label's rank #{s_c > s_y} + #{c < y : s_c == s_y}, in numpy."""
    s = np.asarray(scores, dtype=np.float32)
    B, C = s.shape
    M = np.zeros((C, C), np.int64)
    top5 = 0
    for r in range(B):
        y = int(target[r])
        M[y, int(np.argmax(s[r]))] += 1
        rank = int((s[r] > s[r, y]).sum() + (s[r, :y] == s[r, y]).sum())
        top5 += rank < 5
    return M, top5


def _tied(C, b=23, seed=0, V=None):
    g = torch.Generator().manual_seed(seed * 1000 + C)
    shape = (b, C) if V is None else (V, b, C)
    z = torch.randint(-3, 4, shape, generator=g).float()  # small integers: many ties
    t = torch.randint(0, C, (b,), generator=g)
    z[..., 0, :] = 1.0                                    # a tie across every class
    return z, t


@pytest.mark.parametrize("C", [3, 8, 40])
def test_add_reference_counts_match_numpy_and_ref(C):
    z, t = _tied(C)
    m = DeviceMeter("cpu", C)
    m.add_reference(z[:11], t[:11])
    m.add_reference(z[11:], t[11:])
    M, top5 = _numpy_counts(z.numpy(), t.numpy())
    assert torch.equal(m.confusion, torch.from_numpy(M)) and int(m.top5) == top5
    assert int(m.confusion.trace()) == int(m.buf[1])
    rM, rtop5 = ref.class_metrics(z, t)
    assert torch.equal(rM, m.confusion) and rtop5 == top5
    _, acc = m.snapshot()
    assert acc.classes == class_metrics(M, top5)
    m.reset()
    assert int(m.counts.abs().sum()) == 0


@pytest.mark.parametrize("C,V", [(3, 2), (8, 10), (40, 5)])
def test_add_tta_counts_the_view_mean(C, V):
    z, t = _tied(C, V=V, seed=1)
    m = DeviceMeter("cpu", C)
    m.add_tta(list(z), t)
    acc = sum(torch.softmax(v, 1) for v in z)             # the fp32 sum in view order, then / V as the kernel does
    M, top5 = _numpy_counts((acc / V).numpy(), t.numpy())
    assert torch.equal(m.confusion, torch.from_numpy(M)) and int(m.top5) == top5
    assert int(m.confusion.trace()) == int(m.buf[1])
    rM, rtop5 = ref.class_metrics(acc, t, views=V)
    assert torch.equal(rM, m.confusion) and rtop5 == top5


def test_ref_skips_rows_without_a_maximum():
    z = torch.tensor([[float("nan")] * 4, [-float("inf")] * 4, [float("nan"), 2.0, 2.0, 1.0]])
    M, top5 = ref.class_metrics(z, torch.tensor([0, 1, 3]))
    assert int(M.sum()) == 1 and int(M[3, 1]) == 1 and top5 == 1


def test_meter_without_a_class_count_allocates_nothing():
    m = DeviceMeter("cpu")
    assert m.counts is None and m.confusion is None and m.top5 is None
    m.add_reference(torch.zeros(2, 3), torch.tensor([0, 1]))
    assert m.snapshot()[1].classes is None


# -------------------------------------------------------------------------------------------- CLI runs
def _main(argv):
    from distributed_vgg_f_b200 import cli

    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        assert cli.main(argv) == 0
    return buf.getvalue()


def _lines(text):
    """The report without the namespace line (it names the flags) and the timing lines."""
    return [s for s in text.splitlines() if not s.startswith(("Namespace(", "[Perf]"))]


@pytest.fixture(scope="module")
def runs(tmp_path_factory, synth_root):
    """One epoch of vggf-tiny with --model-ema, with and without --val-metrics, saved and logged."""
    d = tmp_path_factory.mktemp("val_metrics_runs")
    out = {}
    for flag in (False, True):
        ck, log = str(d / ("ck%d.pt" % flag)), str(d / ("log%d.jsonl" % flag))
        torch.manual_seed(0)                        # dropout draws from the global generator: the same masks
        text = _main(BASE + ["-rd", synth_root, "-ep", "1", "--seed", "5", "--model-ema", "--model-ema-steps", "1",
                             "--save", ck, "--log-jsonl", log] + (["--val-metrics"] if flag else []))
        out[flag] = (text, ck, [json.loads(s) for s in open(log).read().splitlines()])
    return out


def _split(off, on):
    """(lines of ``on`` that ``off`` has too, in order; the others) -- asserting the shared ones are ``off``'s."""
    off, on = _lines(off), _lines(on)
    new = [s for s in on if s not in off]
    assert [s for s in on if s in off] == off
    return new


CLASS_LINE = re.compile(r"^\[Info\] (.*?)(EMA test|test) class (\w+): support (\d+), recall ([\d.]+%|-), "
                        r"precision ([\d.]+%|-), confusion row \[([\d, ]+)\]\.$")


def _check_new_lines(new, head, rec, names):
    """The new lines are exactly: per pass, its balanced-accuracy line and one line per class, from ``rec``."""
    want = []
    for what, key in (("test", "test"), ("EMA test", "ema_test")):
        m = {k: rec[key + "_" + k] for k in NEW_KEYS | ({"acc5"} if key + "_acc5" in rec else set())}
        want += class_report(head, what, m, names)
    assert new == want
    for s in new[1:1 + len(names)]:
        assert CLASS_LINE.match(s), s


def _check_record(rec, n_val, C):
    for key in ("test", "ema_test"):
        M = np.array(rec[key + "_confusion"])
        assert M.shape == (C, C) and int(M.sum()) == n_val
        assert rec[key + "_support"] == M.sum(1).tolist()
        assert int(np.trace(M)) == round(rec[key + "_acc"] * n_val)
        assert rec[key + "_balanced_acc"] == class_metrics(M)["balanced_acc"]


NAMES = ["edible", "other", "toy"]


def test_training_run_adds_exactly_the_new_lines_and_keys(runs):
    (off, ck_off, recs_off), (on, ck_on, recs_on) = runs[False], runs[True]
    new = _split(off, on)
    _check_new_lines(new, "Epoch: 1/1, ", recs_on[0], NAMES)
    assert len(new) == 2 * (1 + 3)
    a, b = recs_off[0], recs_on[0]
    extra = {k for k in b if k not in a}
    assert extra == {p + "_" + k for p in ("test", "ema_test") for k in NEW_KEYS}
    for k in a:
        if k != "time":
            assert a[k] == b[k], k
    _check_record(b, 12, 3)
    assert "val_metrics" not in torch.load(ck_off, weights_only=False)["args"]
    assert torch.load(ck_on, weights_only=False)["args"]["val_metrics"] is True


def test_eval_only_reports_what_the_training_run_logged(runs, synth_root):
    """--eval-only of the checkpoint scores the weights the epoch's passes scored: the same counts, both passes."""
    _, ck, recs = runs[True]
    text = {flag: _main(BASE + ["-rd", synth_root, "--eval-only", "--resume", ck, "--model-ema"]
                        + (["--val-metrics"] if flag else [])) for flag in (False, True)}
    _check_new_lines(_split(text[False], text[True]), "Evaluation: ", recs[0], NAMES)


def test_more_than_five_classes_reports_acc5(synth_root, tmp_path):
    log = str(tmp_path / "log.jsonl")
    text = _main(BASE + ["-rd", synth_root, "-ep", "1", "--num-classes", "8", "--val-metrics", "--log-jsonl", log])
    rec = json.loads(open(log).read().splitlines()[0])
    assert {k for k in rec if k.startswith("test_")} == {"test_loss", "test_acc", "test_acc5"} | {
        "test_" + k for k in NEW_KEYS}
    assert rec["test_acc"] <= rec["test_acc5"] <= 1.0
    new = [s for s in _lines(text) if " balanced acc: " in s or " test class " in s]
    m = {k: rec["test_" + k] for k in NEW_KEYS | {"acc5"}}
    assert new == class_report("Epoch: 1/1, ", "test", m, NAMES)
    assert new[-1].startswith("[Info] Epoch: 1/1, test class 7: support 0, recall -, ")
    M = np.array(rec["test_confusion"])
    assert M.shape == (8, 8) and int(M.sum()) == 12 and int(np.trace(M)) == round(rec["test_acc"] * 12)


# ------------------------------------------------------------------------------------- two gloo ranks
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _rank_main(rank, world, port, root, ck, out, tta):
    import torch.distributed as dist

    from distributed_vgg_f_b200.data.loader import DataManager
    from distributed_vgg_f_b200.models.vggf import build_oracle, get_spec
    from distributed_vgg_f_b200.trainer import Trainer
    from distributed_vgg_f_b200.utils.checkpoint import strip_module_prefix

    dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%d" % port, rank=rank, world_size=world)
    net = build_oracle(get_spec("vggf-tiny", 3), seed=0)
    net.load_state_dict(strip_module_prefix(torch.load(ck, weights_only=True)["model"]))
    kw = {} if tta == "none" else dict(tta=tta)
    val = DataManager(root, 3, train=False, world_size=world, rank=rank, shard_eval=True, resize_size=72,
                      crop_size=64, **kw)
    tr = Trainer(net, None, [], val.get_loader(), torch.device("cpu"), verbose_throughput=False, shard_eval=True,
                 val_tta=tta, val_metrics=True, class_names=val.class_names)
    _, acc = tr._evaluate()
    if rank == 0:
        torch.save((acc.correct, acc.count, acc.classes), out)
    dist.destroy_process_group()


@pytest.mark.parametrize("tta", ["none", "flip"])
def test_shard_eval_at_two_gloo_ranks_sums_to_the_one_process_matrix(runs, synth_root, tmp_path, tta):
    import torch.multiprocessing as mp

    _, ck, _ = runs[False]
    res = {}
    for world in (2, 1):
        out = str(tmp_path / ("w%d.pt" % world))
        mp.spawn(_rank_main, args=(world, _free_port(), synth_root, ck, out, tta), nprocs=world, join=True)
        res[world] = torch.load(out, weights_only=False)
    assert res[2][1] == res[1][1] == 12
    assert res[2][2]["confusion"] == res[1][2]["confusion"]
    assert sum(res[2][2]["confusion"][c][c] for c in range(3)) == res[2][0]


@pytest.mark.parametrize("pipeline", ["fused", "stream", "reference"])
@pytest.mark.parametrize("tta", ["none", "ten-crop"])
def test_every_pipeline_and_view_mode_counts_every_sample(runs, synth_root, pipeline, tta):
    _, ck, _ = runs[True]
    text = _main(BASE + ["-rd", synth_root, "--eval-only", "--resume", ck, "--val-metrics", "--pipeline", pipeline,
                         "--val-tta", tta])
    acc = float(re.search(r"^\[Info\] Evaluation: test loss: [\d.]+, test acc: ([\d.]+)%\.$", text, re.M).group(1))
    rows = [CLASS_LINE.match(s) for s in text.splitlines()]
    M = np.array([[int(v) for v in r.group(7).split(",")] for r in rows if r])
    assert M.shape == (3, 3) and int(M.sum()) == 12
    assert int(np.trace(M)) == round(acc * 12 / 100)
    bal = re.search(r"^\[Info\] Evaluation: test balanced acc: ([\d.]+)%\.$", text, re.M).group(1)
    assert bal == "{:.2f}".format(100 * class_metrics(M)["balanced_acc"])
