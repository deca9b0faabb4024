"""Knowledge distillation without a GPU: the flags and their refusals, strict teacher loading, the float64 reference
against an independent numpy / scipy formula and against autograd, the torch-op trainer's objective, CLI runs on a
synthetic folder, and two gloo ranks against one process at the doubled batch."""
import contextlib
import io
import json
import re
import socket

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from scipy.special import log_softmax

BASE = ["-iu", "tcp://127.0.0.1:29999", "-rn", "0", "-ws", "1", "-nc", "-mb", "4", "--model", "vggf-tiny",
        "--engine", "oracle"]


def _parse(extra):
    from distributed_vgg_f_b200 import cli
    return cli.parse_command_line(["-iu", "x", "-rn", "0", "-ws", "1", "-rd", "/r"] + extra, init=False)


# ------------------------------------------------------------------------------------------------ flags
def test_defaults_leave_distillation_off():
    a = _parse([])
    assert a.distill_teacher is None and a.distill_teacher_model is None
    assert a.distill_alpha == 0.5 and a.distill_temperature == 4.0


@pytest.mark.parametrize("extra", [["--distill-alpha", "0"], ["--distill-alpha", "1.5"], ["--distill-alpha", "-1"],
                                   ["--distill-temperature", "0"], ["--distill-temperature", "-2"],
                                   ["--distill-temperature", "inf"], ["--distill-temperature", "nan"],
                                   ["--eval-only"]])
def test_cli_refuses_bad_distillation_flags(extra):
    with pytest.raises(SystemExit), contextlib.redirect_stderr(io.StringIO()):
        _parse(["--distill-teacher", "t.pt"] + extra)


@pytest.mark.parametrize("alpha,temperature", [("1", "4"), ("0.01", "1"), ("0.5", "0.5")])
def test_cli_accepts_the_ranges_edges(alpha, temperature):
    a = _parse(["--distill-teacher", "t.pt", "--distill-alpha", alpha, "--distill-temperature", temperature,
                "--distill-teacher-model", "vggf"])
    assert a.distill_alpha == float(alpha) and a.distill_temperature == float(temperature)


# ------------------------------------------------------------------------------------------ teacher file
def _state(model="vggf-tiny", C=3, seed=0):
    from distributed_vgg_f_b200.models.vggf import build_oracle, get_spec
    return build_oracle(get_spec(model, C), seed=seed).state_dict()


def test_teacher_loads_from_a_checkpoint_or_a_state_dict_and_takes_the_checkpoints_model(tmp_path):
    from distributed_vgg_f_b200.utils import checkpoint as ckpt

    st = _state("vggf-mini")
    p = str(tmp_path / "ck.pt")
    torch.save({"format": ckpt.FORMAT, "model": ckpt.add_module_prefix(st), "args": {"model": "vggf-mini"}}, p)
    name, got = ckpt.load_teacher_state(p, 3, None, "vggf-tiny")
    assert name == "vggf-mini" and all(torch.equal(got[k], st[k]) for k in st)
    assert ckpt.load_teacher_state(p, 3, "vggf-mini", "vggf-tiny")[0] == "vggf-mini"
    plain = str(tmp_path / "plain.pt")
    torch.save(_state("vggf-tiny"), plain)
    assert ckpt.load_teacher_state(plain, 3, None, "vggf-tiny")[0] == "vggf-tiny"      # the student's model
    with pytest.raises(ValueError, match="does not hold a whole vggf-mini"):
        ckpt.load_teacher_state(plain, 3, "vggf-mini", "vggf-tiny")


def test_teacher_loading_is_strict(tmp_path):
    from distributed_vgg_f_b200.utils import checkpoint as ckpt

    with pytest.raises(FileNotFoundError, match="no such file"):
        ckpt.load_teacher_state(str(tmp_path / "missing.pt"), 3)
    st = _state()
    cases = {"missing": {k: v for k, v in st.items() if k != "features.0.bias"},
             "shape": dict(st, **{"classifier.0.weight": st["classifier.0.weight"][:, :-1]}),
             "unexpected": dict(st, extra=torch.zeros(1))}
    for what, bad in cases.items():
        p = str(tmp_path / (what + ".pt"))
        torch.save(bad, p)
        with pytest.raises(ValueError, match="does not hold a whole vggf-tiny"):
            ckpt.load_teacher_state(p, 3, "vggf-tiny")
    p = str(tmp_path / "classes.pt")
    torch.save(_state(C=5), p)
    with pytest.raises(ValueError, match="the teacher has 5 classes, the student 3"):
        ckpt.load_teacher_state(p, 3, "vggf-tiny")


# --------------------------------------------------------------------------------------- the objective
def _numpy_objective(z, u, y, alpha, T, cw=None, eps=0.0, soft=None):
    """(1 - a) F.cross_entropy + a T^2 F.kl_div(batchmean, log_target) written out with scipy's log_softmax."""
    z, u = np.asarray(z, np.float64), np.asarray(u, np.float64)
    B, C = z.shape
    q = np.eye(C)[np.asarray(y)] if soft is None else np.asarray(soft, np.float64)
    q = q * (1 - eps) + eps / C
    w = np.ones(C) if cw is None else np.asarray(cw, np.float64)
    nll = -(q * w[None, :] * log_softmax(z, axis=1)).sum(1)
    denom = w[np.asarray(y)].sum() if (cw is not None and soft is None) else B
    ce = nll.sum() / denom
    lt, ls = log_softmax(u / T, axis=1), log_softmax(z / T, axis=1)
    kl = (np.exp(lt) * (lt - ls)).sum() / B
    return (1 - alpha) * ce + alpha * T * T * kl


def _case(form, weighted, B=6, C=5, seed=0):
    from distributed_vgg_f_b200.data import transforms as T

    g = torch.Generator().manual_seed(seed)
    z, u = torch.randn(B, C, generator=g, dtype=torch.float64) * 2, torch.randn(B, C, generator=g, dtype=torch.float64) * 2
    y = torch.randint(0, C, (B,), generator=g)
    cw = torch.rand(C, generator=g, dtype=torch.float64) + 0.5 if weighted else None
    eps, soft = (0.1 if "smooth" in form else 0.0), None
    if form in ("mixup", "cutmix"):
        mix = T.MixDraw("mixup", 0.35, (0, 0, 0, 0)) if form == "mixup" else T.MixDraw("cutmix", 0.75, (0, 0, 4, 4))
        soft = T.mixed_targets(y, C, mix).double()
    return z, u, y, cw, eps, soft


FORMS = ["plain", "smooth", "mixup", "cutmix"]


@pytest.mark.parametrize("alpha", [0.25, 1.0])
@pytest.mark.parametrize("T", [1.0, 4.0])
@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("weighted", [False, True])
def test_oracle_objective_matches_the_numpy_formula(alpha, T, form, weighted):
    from distributed_vgg_f_b200.ops import ref as R
    from distributed_vgg_f_b200.trainer import distill_loss

    z, u, y, cw, eps, soft = _case(form, weighted)
    want = _numpy_objective(z.numpy(), u.numpy(), y.numpy(), alpha, T, None if cw is None else cw.numpy(), eps,
                            None if soft is None else soft.numpy())
    ce = F.cross_entropy(z, y if soft is None else soft, weight=cw, label_smoothing=eps)
    got = float(distill_loss(z, u, ce, alpha, T))               # what the torch-op trainer optimises
    assert abs(got - want) <= 1e-12 * max(1.0, abs(want))
    ref = R.kd_cross_entropy64(z, u, y, alpha=alpha, temperature=T, class_weights=cw, label_smoothing=eps,
                               soft_target=soft)
    assert abs(float(ref["loss"]) - want) <= 1e-12 * max(1.0, abs(want))


@pytest.mark.parametrize("alpha", [0.25, 1.0])
@pytest.mark.parametrize("T", [1.0, 4.0])
@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("weighted", [False, True])
def test_closed_form_gradient_is_autograds(alpha, T, form, weighted):
    from distributed_vgg_f_b200.ops import ref as R
    from distributed_vgg_f_b200.trainer import distill_loss

    z, u, y, cw, eps, soft = _case(form, weighted, seed=3)
    zz = z.clone().requires_grad_(True)
    ce = F.cross_entropy(zz, y if soft is None else soft, weight=cw, label_smoothing=eps)
    distill_loss(zz, u, ce, alpha, T).backward()
    ref = R.kd_cross_entropy64(z, u, y, alpha=alpha, temperature=T, class_weights=cw, label_smoothing=eps,
                               soft_target=soft, ldd=8)
    assert torch.allclose(ref["dlogits"][:, :z.shape[1]], zz.grad, rtol=1e-10, atol=1e-13)
    assert torch.count_nonzero(ref["dlogits"][:, z.shape[1]:]) == 0


@pytest.mark.parametrize("T", [1.0, 4.0])
def test_a_teacher_equal_to_the_student_at_alpha_one_gives_zero(T):
    from distributed_vgg_f_b200.ops import ref as R

    z, _, y, _, _, _ = _case("plain", False)
    ref = R.kd_cross_entropy64(z, z.clone(), y, alpha=1.0, temperature=T)
    assert float(ref["loss"]) == 0.0 and float(ref["dlogits"].abs().max()) == 0.0


def test_emulated_step_with_a_teacher_uses_the_objective():
    """emulated_step's teacher arguments give the objective and its gradient at the logits; off by default."""
    from distributed_vgg_f_b200.models.vggf import build_oracle, vggf_tiny_spec
    from distributed_vgg_f_b200.ops import ref as R

    spec = vggf_tiny_spec(3)
    state = build_oracle(spec, seed=0).state_dict()
    g = torch.Generator().manual_seed(1)
    x, y = torch.randn(4, 3, 64, 64, generator=g), torch.randint(0, 3, (4,), generator=g)
    logits, loss0, _ = R.emulated_step(spec, state, x, y)
    u = torch.randn(4, 3, generator=g)
    _, loss, _, inter = R.emulated_step(spec, state, x, y, teacher_logits=u, distill_alpha=0.3, distill_temperature=2.0,
                                        return_intermediates=True)
    ref = R.kd_cross_entropy64(logits, u, y, alpha=0.3, temperature=2.0)
    assert abs(float(loss) - float(ref["loss"])) < 1e-5 and float(loss) != float(loss0)
    dz = inter["fc_dz"][len(spec.fcs) - 1]
    assert float((dz.double() - ref["dlogits"]).abs().max()) <= 2.0 ** -8 * float(ref["dlogits"].abs().max()) + 1e-9


# ------------------------------------------------------------------------------------------------ CLI runs
LINE = re.compile(r"^\[Info\] Epoch: (\d+)/\d+, train loss: ([\d.]+), train acc: [\d.]+%, test loss: ([\d.]+), "
                  r"test acc: [\d.]+%\.$", re.M)
BANNER = re.compile(r"^\[Info\] distillation: teacher vggf-mini from \S+ \(alpha 0\.7, temperature 2\.0\): "
                    r"test loss [\d.]+, test acc [\d.]+%\.$", re.M)


def _main(argv):
    from distributed_vgg_f_b200 import cli

    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        assert cli.main(argv) == 0
    return buf.getvalue()


@pytest.fixture(scope="module")
def runs(tmp_path_factory, synth_root):
    """A vggf-mini teacher (--save), then a vggf-tiny student distilled from it for two epochs, and its --eval-only."""
    d = tmp_path_factory.mktemp("distill_runs")
    teacher = str(d / "teacher.pt")
    common = ["-rd", synth_root, "--train-crop-size", "64", "--val-crop-size", "64", "--train-resize-size", "72",
              "--val-resize-size", "72", "--seed", "3"]
    _main(BASE[:-4] + ["--model", "vggf-mini", "--engine", "oracle", "-ep", "1", "--save", teacher] + common)
    before = torch.load(teacher, weights_only=True)
    kd = ["--distill-teacher", teacher, "--distill-alpha", "0.7", "--distill-temperature", "2.0",
          "--mixup-alpha", "0.2"] + common
    out = {"teacher": teacher, "teacher_before": before}
    full = (str(d / "full.pt"), str(d / "full.jsonl"))
    out["full"] = (_main(BASE + ["-ep", "2", "--save", full[0], "--log-jsonl", full[1]] + kd),) + full
    out["eval"] = _main(BASE + ["--eval-only", "--resume", full[0]] + common)
    return out


def test_cli_distillation_run_reports_and_logs(runs):
    text, ck, log = runs["full"]
    assert len(BANNER.findall(text)) == 1
    lines = text.splitlines()
    assert next(k for k, s in enumerate(lines) if BANNER.match(s)) < next(k for k, s in enumerate(lines)
                                                                         if s.startswith("[Info] Epoch: 1/2"))
    recs = [json.loads(s) for s in open(log).read().splitlines()]
    assert len(recs) == 2
    for rec in recs:
        assert rec["distill"] == {"path": runs["teacher"], "model": "vggf-mini", "alpha": 0.7, "temperature": 2.0}
        assert 0.0 <= rec["teacher_test_acc"] <= 1.0


def test_the_teacher_is_unchanged_and_not_in_the_checkpoint(runs):
    after = torch.load(runs["teacher"], weights_only=True)
    before = runs["teacher_before"]
    assert all(torch.equal(after["model"][k], before["model"][k]) for k in before["model"])
    _, ck, _ = runs["full"]
    payload = torch.load(ck, weights_only=True)
    from distributed_vgg_f_b200.models.vggf import vggf_tiny_spec
    assert set(payload["model"]) == {"module." + n for n in vggf_tiny_spec(3).param_names}
    assert payload["args"]["distill_teacher"] == runs["teacher"] and payload["args"]["distill_alpha"] == 0.7


def test_train_line_reports_the_objective_and_test_line_cross_entropy(runs, synth_root):
    """Re-derive epoch 2's test loss (plain CE of the saved student) and check the train loss is not CE-sized alone:
    with a teacher far from the student the objective differs from the student's cross-entropy."""
    from distributed_vgg_f_b200.data.loader import DataManager
    from distributed_vgg_f_b200.models.vggf import build_oracle, vggf_tiny_spec
    from distributed_vgg_f_b200.utils import checkpoint as ckpt

    text, ck, _ = runs["full"]
    epochs = LINE.findall(text)
    assert [e[0] for e in epochs] == ["1", "2"]
    model = build_oracle(vggf_tiny_spec(3))
    ckpt.load_checkpoint(ck, model)
    model.eval()
    dm = DataManager(synth_root, 4, train=False, world_size=1, rank=0, pipeline="auto", seed=3, reference_order=False,
                     resize_size=72, crop_size=64)
    tot, n = 0.0, 0
    with torch.no_grad():
        for bt in dm.get_loader():
            x, y = (bt.to_float("cpu", out_hw=64) if hasattr(bt, "to_float") else (bt[0], bt[1]))
            tot += float(F.cross_entropy(model(x), y)) * y.shape[0]
            n += y.shape[0]
    assert abs(float(epochs[1][2]) - tot / n) < 1e-4


def test_resume_continues_identically(tmp_path):
    """Two epochs with a teacher against one epoch, a checkpoint, and a resumed second epoch with the teacher loaded
    again (it is not in the checkpoint).  Dropout off: the torch path draws its masks from the global generator,
    which a checkpoint does not hold."""
    from distributed_vgg_f_b200.models.vggf import build_oracle, vggf_mini_spec, vggf_tiny_spec
    from distributed_vgg_f_b200.trainer import Trainer
    from distributed_vgg_f_b200.utils import checkpoint as ckpt

    g = torch.Generator().manual_seed(2)
    batches = [(torch.randn(4, 3, 64, 64, generator=g), torch.randint(0, 3, (4,), generator=g)) for _ in range(3)]

    def setup():
        model = build_oracle(vggf_tiny_spec(3), seed=0)
        for m in model.modules():
            if isinstance(m, torch.nn.Dropout):
                m.p = 0.0
        teacher = build_oracle(vggf_mini_spec(3), seed=4).eval().requires_grad_(False)
        opt = torch.optim.Adam(model.parameters(), lr=1e-3)
        return model, opt, Trainer(model, opt, batches, batches[:1], "cpu", verbose_throughput=False, teacher=teacher,
                                   distill_alpha=0.7, distill_temperature=2.0)

    m1, _, t1 = setup()
    t1.fit(2)
    m2, o2, t2 = setup()
    path = str(tmp_path / "ck.pt")
    t2.on_epoch_end = lambda epoch, tr: ckpt.save_checkpoint(path, m2, o2, epoch, {})
    t2.fit(1)
    m3, o3, t3 = setup()
    t3.fit(2, start_epoch=ckpt.load_checkpoint(path, m3, o3) + 1)
    assert t1.history[1] == t3.history[0]
    assert all(torch.equal(a, b) for a, b in zip(m1.state_dict().values(), m3.state_dict().values()))


def test_eval_only_of_the_student_works(runs):
    assert re.search(r"^\[Info\] Evaluation: test loss: [\d.]+, test acc: [\d.]+%\.$", runs["eval"], re.M)
    assert "distillation" not in runs["eval"]


def test_a_teacher_the_native_engine_cannot_run_is_named(monkeypatch):
    """vggf-tiny's 16-channel convolutions: refused when the native teacher is built, naming the model."""
    import argparse

    from distributed_vgg_f_b200 import train
    from distributed_vgg_f_b200.engine import native_engine as ne
    from distributed_vgg_f_b200.models.vggf import get_spec
    from distributed_vgg_f_b200.utils import checkpoint as ckpt

    monkeypatch.setattr(ckpt, "load_teacher_state", lambda *a: ("vggf-tiny", _state()))
    monkeypatch.setattr(ne.ops, "require", lambda: None)
    args = argparse.Namespace(distill_teacher="t.pt", distill_teacher_model=None, model="vggf", distill_alpha=0.5,
                              distill_temperature=4.0, mini_batch=4, deterministic=False)
    with pytest.raises(ValueError, match="--distill-teacher-model vggf-tiny: the native engine cannot run it"):
        train.build_teacher(args, get_spec("vggf", 3), torch.device("cpu"), True, 224, 224)


# ------------------------------------------------------------------------------------------- two gloo ranks
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _rank_main(rank, world, port, batches, out):
    import argparse

    import torch.distributed as dist

    from distributed_vgg_f_b200.models.vggf import build_oracle, get_spec
    from distributed_vgg_f_b200.parallel.ddp import FlatDDP
    from distributed_vgg_f_b200.train import build_optimizer
    from distributed_vgg_f_b200.trainer import Trainer

    torch.set_num_threads(2)
    dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%d" % port, rank=rank, world_size=world)
    model = build_oracle(get_spec("vggf-tiny", 3), seed=0).eval()       # no dropout: the same function on every rank
    teacher = build_oracle(get_spec("vggf-tiny", 3), seed=9).eval().requires_grad_(False)
    ddp = FlatDDP(model, bucket_cap_mb=1.0)
    opt = build_optimizer(model, argparse.Namespace(optimizer="sgd", learning_rate=0.05, momentum=0.9,
                                                    weight_decay=0.0, bias_weight_decay=None))
    per = batches[0][0].shape[0] // world
    mine = [(x[rank * per:(rank + 1) * per], y[rank * per:(rank + 1) * per]) for x, y in batches]
    tr = Trainer(ddp, opt, mine, mine[:1], "cpu", verbose_throughput=False, teacher=teacher, distill_alpha=0.6,
                 distill_temperature=3.0)
    model.train = lambda mode=True: model           # keep dropout off: Trainer switches to train mode
    tr._train()
    torch.save({k: v.detach().clone() for k, v in model.state_dict().items()}, "%s.%d" % (out, rank))
    dist.destroy_process_group()


def test_two_gloo_ranks_with_a_teacher_equal_one_process_with_the_doubled_batch(tmp_path):
    import torch.multiprocessing as mp

    g = torch.Generator().manual_seed(5)
    batches = [(torch.randn(8, 3, 64, 64, generator=g), torch.randint(0, 3, (8,), generator=g)) for _ in range(3)]
    mp.spawn(_rank_main, args=(2, _free_port(), batches, str(tmp_path / "two")), nprocs=2, join=True)
    mp.spawn(_rank_main, args=(1, _free_port(), batches, str(tmp_path / "one")), nprocs=1, join=True)
    r0, r1 = torch.load(str(tmp_path / "two.0")), torch.load(str(tmp_path / "two.1"))
    one = torch.load(str(tmp_path / "one.0"))
    from distributed_vgg_f_b200.models.vggf import build_oracle, get_spec
    init = build_oracle(get_spec("vggf-tiny", 3), seed=0).state_dict()
    for k in r0:
        assert torch.equal(r0[k], r1[k]), "replicas differ in %s" % k
        moved = float((one[k] - init[k]).abs().max())
        err = float((r0[k] - one[k]).abs().max())
        assert err <= 1e-3 * moved + 1e-6, "%s: two ranks %.3g from one process (moved %.3g)" % (k, err, moved)
