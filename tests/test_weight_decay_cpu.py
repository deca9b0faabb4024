"""Weight decay, AdamW and the learning-rate schedule without a GPU: the schedule against torch's
schedulers, the torch-op engine's parameter groups, resume, a gloo run and the flags' validation."""
import itertools
import json
import math
import os
import socket
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BASE = ["-iu", "tcp://127.0.0.1:29999", "-rn", "0", "-ws", "1", "-nc", "-mb", "4", "--model", "vggf-tiny",
        "--engine", "oracle"]
RECIPE = ["--optimizer", "adamw", "--weight-decay", "0.05", "--bias-weight-decay", "0", "--lr-scheduler", "cosine",
          "--lr-warmup-epochs", "1", "--lr-warmup-method", "linear", "--lr-warmup-decay", "0.1", "--lr-min", "1e-5"]


# ------------------------------------------------------------------------------------------ schedule
def _torch_rates(base_lr, epochs, scheduler, step, gamma, lr_min, W, method, decay):
    """The rate of every epoch from torchvision's recipe of schedulers, stepped once per epoch."""
    p = torch.nn.Parameter(torch.zeros(1))
    opt = torch.optim.SGD([p], lr=base_lr)
    S = torch.optim.lr_scheduler
    if scheduler == "cosine":
        main = S.CosineAnnealingLR(opt, T_max=epochs - W, eta_min=lr_min)
    else:
        main = S.StepLR(opt, step_size=step, gamma=gamma) if step else S.ConstantLR(opt, factor=1.0, total_iters=0)
    if W:
        warm = (S.LinearLR(opt, start_factor=decay, total_iters=W) if method == "linear"
                else S.ConstantLR(opt, factor=decay, total_iters=W))
        sched = S.SequentialLR(opt, schedulers=[warm, main], milestones=[W])
    else:
        sched = main
    rates = []
    for _ in range(epochs):
        rates.append(opt.param_groups[0]["lr"])
        opt.step()
        sched.step()
    return rates


GRID = list(itertools.product([0, 1, 3], ["linear", "constant"], [5, 12], [0.0, 1e-4]))


@pytest.mark.parametrize("W,method,epochs,lr_min", GRID)
@pytest.mark.parametrize("scheduler,step,gamma", [("cosine", 0, 0.1), ("step", 2, 0.5), ("step", 3, 0.1),
                                                  ("step", 0, 0.1)])
def test_schedule_matches_torchs_schedulers(W, method, epochs, lr_min, scheduler, step, gamma):
    import warnings

    from distributed_vgg_f_b200.utils.lr_schedule import LRSchedule

    base = 0.02
    sch = LRSchedule(base_lr=base, epochs=epochs, scheduler=scheduler, step=step, gamma=gamma, lr_min=lr_min,
                     warmup_epochs=W, warmup_method=method, warmup_decay=0.1)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        want = _torch_rates(base, epochs, scheduler, step, gamma, lr_min, W, method, 0.1)
    got = [sch.lr_at(k) for k in range(epochs)]
    for k, (a, b) in enumerate(zip(got, want)):
        assert abs(a - b) <= 1e-12 * abs(b) + 1e-18, (k, a, b)


@pytest.mark.parametrize("step,gamma", [(1, 0.1), (2, 0.5), (3, 0.7), (7, 0.3)])
def test_step_schedule_is_the_parents_closed_form_bit_for_bit(step, gamma):
    from distributed_vgg_f_b200.utils.lr_schedule import LRSchedule

    base = 0.0123
    sch = LRSchedule(base_lr=base, epochs=40, step=step, gamma=gamma)
    assert not sch.constant
    for e in range(40):
        assert sch.lr_at(e) == base * gamma ** (e // step)
    assert LRSchedule(base_lr=base, epochs=40).constant


# ------------------------------------------------------------------------------------ optimizer groups
def _tiny():
    from distributed_vgg_f_b200.models.vggf import build_oracle, vggf_tiny_spec

    return build_oracle(vggf_tiny_spec(3), seed=0)


@pytest.mark.parametrize("opt,cls", [("adam", torch.optim.Adam), ("adamw", torch.optim.AdamW),
                                     ("sgd", torch.optim.SGD)])
def test_bias_tensors_take_the_bias_decay(opt, cls):
    import argparse

    from distributed_vgg_f_b200.train import build_optimizer

    model = _tiny()
    args = argparse.Namespace(optimizer=opt, learning_rate=1e-3, momentum=0.9, weight_decay=0.05,
                              bias_weight_decay=0.0)
    o = build_optimizer(model, args)
    assert isinstance(o, cls)
    names = {id(p): n for n, p in model.named_parameters()}
    seen = set()
    for g in o.param_groups:
        for p in g["params"]:
            n = names[id(p)]
            seen.add(n)
            assert g["weight_decay"] == (0.0 if n.endswith(".bias") else 0.05), n
    assert seen == set(names.values())
    # without a bias decay: one group, every tensor at the decay -- AdamW's own default (0.01) never applies
    args.bias_weight_decay, args.weight_decay = None, 0.0
    o = build_optimizer(model, args)
    assert len(o.param_groups) == 1 and o.param_groups[0]["weight_decay"] == 0.0


# --------------------------------------------------------------------------------------------- runs
def _run(argv):
    from distributed_vgg_f_b200.cli import parse_command_line
    from distributed_vgg_f_b200.train import manage_training

    return manage_training(parse_command_line(argv))


@pytest.fixture
def no_dropout(monkeypatch):
    """The oracle without dropout, so that runs compare bit for bit whatever the global RNG holds."""
    from distributed_vgg_f_b200 import train

    real = train.build_oracle

    def build(*a, **k):
        model = real(*a, **k)
        for m in model.modules():
            if isinstance(m, torch.nn.Dropout):
                m.p = 0.0
        return model
    monkeypatch.setattr(train, "build_oracle", build)


def test_recipe_run_resumes_and_equals_a_plain_torch_loop(synth_root, tmp_path, monkeypatch, no_dropout):
    """4 epochs of AdamW (decay, biases at 0) with cosine after a linear warmup: equal bit for bit to 2
    epochs resumed for 2 more, and to a plain loop of torch.optim.AdamW with torchvision's parameter groups
    and SequentialLR(LinearLR, CosineAnnealingLR) stepped per epoch.  The JSONL records each epoch's rate."""
    import torch.nn.functional as F

    from distributed_vgg_f_b200.models.vggf import build_oracle, vggf_tiny_spec
    from distributed_vgg_f_b200.trainer import Trainer

    full, half, log = str(tmp_path / "full.pt"), str(tmp_path / "half.pt"), str(tmp_path / "full.jsonl")
    common = BASE + ["-rd", synth_root, "-lr", "0.01", "-ep", "4"] + RECIPE
    seen_batches = []
    real_to_device = Trainer._mixed_to_device

    def record(self, batch):
        out = real_to_device(self, batch)
        seen_batches.append((out[0].clone(), out[1].clone()))
        return out
    monkeypatch.setattr(Trainer, "_mixed_to_device", record)
    _run(common + ["--save", full, "--log-jsonl", log])
    monkeypatch.setattr(Trainer, "_mixed_to_device", real_to_device)
    real_fit = Trainer.fit
    monkeypatch.setattr(Trainer, "fit", lambda self, epochs, start_epoch=1: real_fit(self, 2, start_epoch))
    _run(common + ["--save", half])
    monkeypatch.setattr(Trainer, "fit", real_fit)
    assert torch.load(half, weights_only=True)["epoch"] == 2
    _run(common + ["--resume", half, "--save", half])
    a, b = torch.load(full, weights_only=True), torch.load(half, weights_only=True)
    assert b["epoch"] == 4
    for k in a["model"]:
        assert torch.equal(a["model"][k], b["model"][k]), k
    assert a["optimizer"]["param_groups"][0]["lr"] == b["optimizer"]["param_groups"][0]["lr"]

    recs = [json.loads(s) for s in open(log).read().splitlines()]
    rates = [r["lr"] for r in recs]
    assert rates == [0.01 * (0.1 + 0.9 * 0 / 1)] + [1e-5 + (0.01 - 1e-5) * (1 + math.cos(math.pi * k / 3)) / 2
                                                   for k in range(3)]

    # the plain torch loop, on the batches the trainer drew
    model = build_oracle(vggf_tiny_spec(3), seed=0)
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    named = list(model.named_parameters())
    opt = torch.optim.AdamW([{"params": [p for n, p in named if not n.endswith(".bias")], "weight_decay": 0.05},
                             {"params": [p for n, p in named if n.endswith(".bias")], "weight_decay": 0.0}],
                            lr=0.01, weight_decay=0.05)
    S = torch.optim.lr_scheduler
    sched = S.SequentialLR(opt, [S.LinearLR(opt, start_factor=0.1, total_iters=1),
                                 S.CosineAnnealingLR(opt, T_max=3, eta_min=1e-5)], milestones=[1])
    per_epoch = len(seen_batches) // 4
    seen = []
    for epoch in range(4):
        seen.append(opt.param_groups[0]["lr"])
        model.train()
        for x, y in seen_batches[epoch * per_epoch:(epoch + 1) * per_epoch]:
            loss = F.cross_entropy(model(x), y)
            opt.zero_grad()
            loss.backward()
            opt.step()
        sched.step()
    for r, t in zip(rates, seen):
        assert abs(r - t) <= 1e-12 * t
    state = model.state_dict()
    for k, v in a["model"].items():
        assert torch.equal(v, state[k[len("module."):]]), k


def test_two_gloo_ranks_run_the_recipe(synth_root):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    procs = []
    for r in range(2):
        cmd = [sys.executable, "-m", "distributed_vgg_f_b200", "-iu", "tcp://127.0.0.1:%d" % port, "-rn", str(r),
               "-ws", "2", "-rd", synth_root, "-ep", "2", "-nc", "-lr", "0.001", "-mb", "4", "--model", "vggf-tiny",
               "--engine", "oracle"] + RECIPE
        env = dict(os.environ, PYTHONPATH=ROOT, OMP_NUM_THREADS="2")
        procs.append(subprocess.Popen(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                                      text=True))
    outs = [p.communicate(timeout=600)[0] for p in procs]
    assert all(p.returncode == 0 for p in procs), outs
    assert all("Epoch: 2/2" in o for o in outs), outs


# ------------------------------------------------------------------------------------------- flags
@pytest.mark.parametrize("extra", [["--weight-decay", "-0.1"], ["--bias-weight-decay", "-1"],
                                   ["--lr-scheduler", "cosine", "--lr-warmup-epochs", "5", "-ep", "5"],
                                   ["--lr-warmup-decay", "0"], ["--lr-warmup-decay", "1.5"],
                                   ["--lr-warmup-epochs", "-1"], ["--lr-min", "-1"], ["--optimizer", "lamb"],
                                   ["--lr-scheduler", "poly"], ["--lr-warmup-method", "exp"]])
def test_bad_flag_values_are_refused(extra):
    from distributed_vgg_f_b200 import cli

    with pytest.raises(SystemExit):
        cli.parse_command_line(["-iu", "x", "-rn", "0", "-ws", "1", "-rd", "/r"] + extra, init=False)


def test_flag_defaults_are_the_parents_behaviour():
    from distributed_vgg_f_b200 import cli
    from distributed_vgg_f_b200.utils.lr_schedule import LRSchedule

    args = cli.parse_command_line(["-iu", "x", "-rn", "0", "-ws", "1", "-rd", "/r"], init=False)
    assert (args.optimizer, args.weight_decay, args.bias_weight_decay, args.lr_scheduler) == ("adam", 0.0, None, "step")
    assert LRSchedule.from_args(args).constant
    ok = cli.parse_command_line(["-iu", "x", "-rn", "0", "-ws", "1", "-rd", "/r", "-ep", "6"] + RECIPE, init=False)
    assert ok.optimizer == "adamw" and ok.bias_weight_decay == 0.0 and ok.lr_warmup_epochs == 1
