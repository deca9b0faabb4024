"""The moving average of the weights (--model-ema) without a GPU: the flags, torchvision's adjusted decay,
which updates take the EMA, the torch-op trainer against torchvision's AveragedModel stepped by hand,
the checkpoint entry, resume, the report line, --eval-only, predict --ema and two gloo ranks."""
import json
import os
import re
import socket
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BASE = ["-iu", "tcp://127.0.0.1:29999", "-rn", "0", "-ws", "1", "-nc", "-mb", "4", "--model", "vggf-tiny",
        "--engine", "oracle"]


# ---------------------------------------------------------------------------------------------- CLI
@pytest.mark.parametrize("flag,value,ok", [("--model-ema-steps", "1", True), ("--model-ema-steps", "0", False),
                                           ("--model-ema-steps", "-3", False), ("--model-ema-decay", "0", True),
                                           ("--model-ema-decay", "0.999", True), ("--model-ema-decay", "1.0", False),
                                           ("--model-ema-decay", "-0.1", False)])
def test_cli_validates_the_flags(flag, value, ok):
    from distributed_vgg_f_b200 import cli

    argv = ["-iu", "tcp://127.0.0.1:1", "-rn", "0", "-ws", "1", "-rd", "/nonexistent", "--model-ema", flag, value]
    if ok:
        args = cli.parse_command_line(argv, init=False)
        assert args.model_ema and float(getattr(args, flag[2:].replace("-", "_"))) == float(value)
    else:
        with pytest.raises(SystemExit):
            cli.parse_command_line(argv, init=False)


def test_cli_defaults_are_torchvisions():
    from distributed_vgg_f_b200 import cli

    args = cli.build_parser().parse_args(["-iu", "x", "-rn", "0", "-ws", "1", "-rd", "/r"])
    assert (args.model_ema, args.model_ema_steps, args.model_ema_decay) == (False, 32, 0.99998)


# ---------------------------------------------------------------------------------------- decay
def test_adjusted_decay_is_torchvisions_formula_with_the_accumulation_factor():
    from distributed_vgg_f_b200.train import model_ema_decay

    # torchvision's references/classification/train.py, K = 1
    world, mb, steps, epochs, d = 8, 32, 32, 600, 0.99998
    adjust = world * mb * steps / epochs
    want = 1.0 - min(1.0, (1.0 - d) * adjust)
    assert model_ema_decay(d, world, mb, 1, steps, epochs) == want
    # K mini-batches per update: K times the images between two updates
    adjust4 = world * mb * 4 * steps / epochs
    assert model_ema_decay(d, world, mb, 4, steps, epochs) == 1.0 - min(1.0, (1.0 - d) * adjust4)
    assert model_ema_decay(d, world, mb, 4, steps, epochs) < want
    # the clamp: alpha = 1 makes every update a copy of the weights
    assert model_ema_decay(0.5, 2, 64, 1, 32, 1) == 0.0


# ------------------------------------------------------------------------------------- schedule
class _FakeEngine:
    """The native engine as Trainer sees it: records how train_step is called."""

    def __init__(self):
        self.calls, self.ema32 = [], torch.zeros(4)

    def train_step(self, batch, update=True, ema=False):
        self.calls.append((update, ema))

    def eval_step(self, batch, ema=False):
        pass

    def set_meter(self, meter):
        pass

    def sync(self):
        pass

    def prepare_ema(self):
        self.calls.append("prepare_ema")


@pytest.mark.parametrize("n,K,steps", [(10, 1, 1), (10, 1, 3), (10, 3, 1), (11, 3, 2), (7, 4, 2), (5, 2, 32)])
def test_ema_updates_follow_torchvisions_schedule(n, K, steps):
    """The EMA updates after the optimizer updates whose 0-based index u within the epoch has
    u % steps == 0; with accumulation an update ends every group of K and the epoch's short last group."""
    from distributed_vgg_f_b200.trainer import Trainer

    eng = _FakeEngine()
    tr = Trainer(eng, None, list(range(n)), [], "cpu", verbose_throughput=False, accum_steps=K, model_ema=True,
                 model_ema_steps=steps)
    tr._train()
    updates = [k for k in range(n) if (k + 1) % K == 0 or k + 1 == n]
    want = []
    for k in range(n):
        if k in updates:
            u = updates.index(k)
            want.append((True, u % steps == 0))
        else:
            want.append((False, False))
    assert eng.calls == want
    tr._evaluate(ema=True)
    assert eng.calls[-1] == "prepare_ema"


def test_native_trainer_without_ema_makes_the_parents_calls():
    from distributed_vgg_f_b200.trainer import Trainer

    class Plain(_FakeEngine):
        def train_step(self, *a, **k):
            self.calls.append((a[1:], k))

    eng = Plain()
    Trainer(eng, None, list(range(5)), [], "cpu", verbose_throughput=False, accum_steps=2)._train()
    assert eng.calls == [((), {"update": False}), ((), {}), ((), {"update": False}), ((), {}), ((), {})]


def test_native_trainer_refuses_an_engine_without_ema():
    from distributed_vgg_f_b200.trainer import Trainer

    eng = _FakeEngine()
    eng.ema32 = None
    with pytest.raises(ValueError, match="ema_decay"):
        Trainer(eng, None, [], [], "cpu", model_ema=True)


# ------------------------------------------------------------------------------ torch-op trainer
def _tiny(C=3, seed=0):
    from distributed_vgg_f_b200.models.vggf import build_oracle, vggf_tiny_spec

    model = build_oracle(vggf_tiny_spec(C), seed=seed)
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    return model


def _batches(n, b=4, C=3, hw=64, seed=1):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(b, 3, hw, hw, generator=g), torch.randint(0, C, (b,), generator=g)) for _ in range(n)]


def _same(a, b):
    return all(torch.equal(x, y) for x, y in zip(a.values(), b.values())) and list(a) == list(b)


@pytest.mark.parametrize("opt,K,steps", [("adam", 1, 2), ("sgd", 2, 1), ("adam", 3, 1)])
def test_oracle_trainer_ema_is_averaged_model_stepped_by_hand(opt, K, steps):
    from torch.optim.swa_utils import AveragedModel

    from distributed_vgg_f_b200.train import build_model_ema
    from distributed_vgg_f_b200.trainer import Trainer

    decay = 0.8
    batches = _batches(7)
    model = _tiny()
    mk = (lambda p: torch.optim.Adam(p, lr=1e-3)) if opt == "adam" else (lambda p: torch.optim.SGD(p, lr=1e-2,
                                                                                                    momentum=0.9))
    ref_model = _tiny()
    ref_model.load_state_dict(model.state_dict())
    ema = build_model_ema(model, decay)
    tr = Trainer(model, mk(model.parameters()), batches, [], "cpu", verbose_throughput=False, accum_steps=K,
                 model_ema=ema, model_ema_steps=steps)
    tr._train()

    def ema_avg(e, p, n):
        return decay * e + (1 - decay) * p

    ref_ema = AveragedModel(ref_model, avg_fn=ema_avg, use_buffers=True)
    ref_opt = mk(ref_model.parameters())
    u, pending = 0, 0
    for k, (x, y) in enumerate(batches):
        if pending == 0:
            ref_opt.zero_grad()
        F.cross_entropy(ref_model(x), y).backward()
        pending += 1
        if (k + 1) % K == 0 or k + 1 == len(batches):
            if pending > 1:
                for p in ref_model.parameters():
                    p.grad.mul_(1.0 / pending)
            ref_opt.step()
            if u % steps == 0:
                ref_ema.update_parameters(ref_model)
            u += 1
            pending = 0
    assert int(ref_ema.n_averaged) == int(ema.n_averaged) == len(range(0, u, steps))
    assert _same(ema.state_dict(), ref_ema.state_dict())
    assert not _same(ema.module.state_dict(), model.state_dict())


# ---------------------------------------------------------------------------------------- checkpoint
def test_checkpoint_ema_keys_are_averaged_models_and_load_into_it(tmp_path):
    from torch.optim.swa_utils import AveragedModel

    from distributed_vgg_f_b200.models.vggf import vgg_funnel_model
    from distributed_vgg_f_b200.train import build_model_ema
    from distributed_vgg_f_b200.utils import checkpoint as ckpt

    model = _tiny()
    ema = build_model_ema(model, 0.9)
    ema.update_parameters(model)
    path = str(tmp_path / "ck.pt")
    ckpt.save_checkpoint(path, model, None, 1, {}, model_ema=ema)
    payload = torch.load(path, weights_only=True)
    assert set(payload) == {"format", "model", "optimizer", "epoch", "args", "model_ema"}
    assert payload["format"] == ckpt.FORMAT
    tv = AveragedModel(vgg_funnel_model(3))
    assert list(payload["model_ema"]) == list(tv.state_dict())
    assert payload["model_ema"]["n_averaged"].dtype == torch.int64 and int(payload["model_ema"]["n_averaged"]) == 1


def test_native_engine_ema_entry_has_the_same_keys(tmp_path):
    """The native engine's entry (host logic only: an engine assembled without device buffers) has the
    keys of AveragedModel(model).state_dict(), its tensors in torch layout, and loads back."""
    from torch.optim.swa_utils import AveragedModel

    from distributed_vgg_f_b200.engine.native_engine import NativeEngine
    from distributed_vgg_f_b200.models import layout as L
    from distributed_vgg_f_b200.models.vggf import vggf_tiny_spec
    from distributed_vgg_f_b200.parallel.buckets import engine_bucket_plan
    from distributed_vgg_f_b200.utils import checkpoint as ckpt

    spec = vggf_tiny_spec(3)
    eng = NativeEngine.__new__(NativeEngine)
    eng.spec, eng.device = spec, torch.device("cpu")
    eng.plan = engine_bucket_plan(L.ready_order(spec), 32.0, 9.5, 2400.0)
    eng.ema32 = torch.randn(eng.plan.total)
    eng.ema_updates, eng._accum = 5, 0
    entry = {k: v.clone() for k, v in ckpt.ema_state(eng, True).items()}    # on the CPU, biases are views
    model = _tiny()
    tv = AveragedModel(model)
    assert set(entry) == set(tv.state_dict())
    tv.load_state_dict(entry)
    assert int(tv.n_averaged) == 5
    ema32 = eng.ema32.clone()
    eng.ema32.zero_()
    eng.import_ema_state(ckpt.strip_module_prefix({k: v for k, v in entry.items() if k != "n_averaged"}), 7)
    for name in spec.param_names:           # the arena gaps and conv0's zero tail are not part of the state
        assert torch.equal(L.to_torch(spec, name, eng._view(eng.ema32, name)), L.to_torch(spec, name, eng._view(ema32, name)))
    assert eng.ema_updates == 7


def test_resume_continues_the_ema_of_an_uninterrupted_run(tmp_path, capsys):
    from distributed_vgg_f_b200.train import build_model_ema
    from distributed_vgg_f_b200.trainer import Trainer
    from distributed_vgg_f_b200.utils import checkpoint as ckpt

    batches = _batches(5)

    def setup():
        model = _tiny()
        opt = torch.optim.Adam(model.parameters(), lr=1e-3)
        ema = build_model_ema(model, 0.7)
        return model, opt, ema, Trainer(model, opt, batches, batches[:1], "cpu", verbose_throughput=False,
                                        model_ema=ema, model_ema_steps=2)

    m1, o1, e1, t1 = setup()
    t1.fit(2)
    m2, o2, e2, t2 = setup()
    path = str(tmp_path / "ck.pt")
    t2.on_epoch_end = lambda epoch, tr: ckpt.save_checkpoint(path, m2, o2, epoch, {}, model_ema=e2)
    t2.fit(1)
    m3, o3, e3, t3 = setup()
    start = ckpt.load_checkpoint(path, m3, o3, model_ema=e3) + 1
    assert start == 2 and int(e3.n_averaged) == 3
    t3.fit(2, start_epoch=start)
    assert int(e1.n_averaged) == int(e3.n_averaged) == 6
    assert _same(e1.state_dict(), e3.state_dict())
    # a checkpoint without an EMA: the EMA starts fresh, with a note
    capsys.readouterr()
    plain = str(tmp_path / "plain.pt")
    ckpt.save_checkpoint(plain, m1, o1, 1, {})
    m4, o4, e4, _ = setup()
    ckpt.load_checkpoint(plain, m4, o4, model_ema=e4)
    assert int(e4.n_averaged) == 0 and "holds no model EMA: the EMA starts fresh" in capsys.readouterr().out
    with pytest.raises(ValueError, match="no model EMA"):
        ckpt.load_checkpoint(plain, m4, o4, model_ema=e4, ema_required=True)


# ------------------------------------------------------------------------------------------- CLI runs
@pytest.fixture(scope="module")
def runs(tmp_path_factory, synth_root):
    """One epoch of the CLI with --model-ema and one without, each with --save and --log-jsonl."""
    from distributed_vgg_f_b200 import cli

    d = tmp_path_factory.mktemp("ema_runs")
    out = {}
    for name, extra in (("ema", ["--model-ema", "--model-ema-steps", "1", "--model-ema-decay", "0.999"]),
                        ("off", [])):
        ck, log = str(d / (name + ".pt")), str(d / (name + ".jsonl"))
        argv = BASE + ["-rd", synth_root, "-ep", "1", "--save", ck, "--log-jsonl", log] + extra
        import contextlib
        import io
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            assert cli.main(argv) == 0
        out[name] = (ck, log, buf.getvalue())
    return out


EMA_LINE = re.compile(r"^\[Info\] Epoch: 1/1, EMA test loss: [\d.]+, EMA test acc: [\d.]+%\.$", re.M)


def test_cli_run_reports_and_logs_the_ema(runs):
    ck, log, text = runs["ema"]
    assert len(EMA_LINE.findall(text)) == 1
    lines = text.splitlines()
    i = next(k for k, s in enumerate(lines) if s.startswith("[Info] Epoch: 1/1, train loss"))
    assert EMA_LINE.match(lines[i + 1])
    rec = json.loads(open(log).read().splitlines()[-1])
    assert {"ema_test_loss", "ema_test_acc"} <= set(rec)
    payload = torch.load(ck, weights_only=True)
    n_updates = -(-24 // 4)                       # synth_root: 3 classes x 8 training images, batch 4
    assert int(payload["model_ema"]["n_averaged"]) == n_updates


def test_flags_off_keep_the_parents_checkpoint_and_output(runs):
    ck, log, text = runs["off"]
    assert "EMA" not in text
    payload = torch.load(ck, weights_only=True)
    assert set(payload) == {"format", "model", "optimizer", "epoch", "args"}
    rec = json.loads(open(log).read().splitlines()[-1])
    assert not {k for k in rec if "ema" in k}
    assert set(rec) == {"epoch", "train_loss", "train_acc", "test_loss", "test_acc", "time", "world_size"}


def test_eval_only_scores_the_checkpoints_ema(runs, synth_root, capsys):
    from distributed_vgg_f_b200 import cli

    ck = runs["ema"][0]
    capsys.readouterr()
    assert cli.main(BASE + ["-rd", synth_root, "--eval-only", "--resume", ck, "--model-ema"]) == 0
    out = capsys.readouterr().out
    assert re.search(r"^\[Info\] Evaluation: test loss: [\d.]+, test acc: [\d.]+%\.$", out, re.M)
    assert re.search(r"^\[Info\] Evaluation: EMA test loss: [\d.]+, EMA test acc: [\d.]+%\.$", out, re.M)
    with pytest.raises(ValueError, match="no model EMA"):
        cli.main(BASE + ["-rd", synth_root, "--eval-only", "--resume", runs["off"][0], "--model-ema"])
    assert cli.main(BASE + ["-rd", synth_root, "--eval-only", "--resume", runs["off"][0]]) == 0
    assert "EMA" not in capsys.readouterr().out


def test_predict_with_the_ema_weights(runs, synth_root):
    from distributed_vgg_f_b200.tools import predict as P
    from distributed_vgg_f_b200.utils.checkpoint import strip_module_prefix

    img = os.path.join(synth_root, "ValidationData")
    ck = runs["ema"][0]
    raw, files = P.predict(ck, [img], engine="oracle")
    ema, files2 = P.predict(ck, [img], engine="oracle", ema=True)
    assert files == files2 and len(files) > 0
    payload = torch.load(ck, weights_only=True)
    model = _tiny()
    model.load_state_dict(strip_module_prefix({k: v for k, v in payload["model_ema"].items() if k != "n_averaged"}))
    model.eval()
    from PIL import Image

    from distributed_vgg_f_b200.data.transforms import reference_transforms
    tf = reference_transforms(train=False)
    with torch.no_grad():
        want = model(torch.stack([tf(Image.open(f).convert("RGB")) for f in files]))
    assert torch.equal(ema, want) and not torch.equal(raw, ema)
    with pytest.raises(ValueError, match="no model EMA"):
        P.predict(runs["off"][0], [img], engine="oracle", ema=True)


# ------------------------------------------------------------------------------------- 2 gloo ranks
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def test_two_gloo_ranks_end_with_identical_emas(synth_root):
    port = _free_port()
    procs = []
    for r in range(2):
        cmd = [sys.executable, "-m", "distributed_vgg_f_b200", "-iu", "tcp://127.0.0.1:%d" % port, "-rn", str(r),
               "-ws", "2", "-rd", synth_root, "-ep", "1", "-nc", "-lr", "0.001", "-mb", "4", "--model", "vggf-tiny",
               "--engine", "oracle", "--model-ema", "--model-ema-steps", "1", "--model-ema-decay", "0.99"]
        env = dict(os.environ, PYTHONPATH=ROOT, OMP_NUM_THREADS="2")
        procs.append(subprocess.Popen(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                                      text=True))
    outs = [p.communicate(timeout=600)[0] for p in procs]
    assert all(p.returncode == 0 for p in procs), outs
    pat = re.compile(r"\[Info\] Epoch: 1/1, EMA test loss: ([\d.]+), EMA test acc: ([\d.]+)%\.")
    lines = [pat.findall(o) for o in outs]
    assert all(len(l) == 1 for l in lines), outs
    # unsharded validation of the EMA: replicas whose EMAs are identical score identically
    assert lines[0] == lines[1]
