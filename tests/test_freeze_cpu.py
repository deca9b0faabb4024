"""--freeze-layers without a GPU: the flag's range, the bucket plan over the trainable prefix of the arena,
tools.plan, the torch-op engine against a plain torch loop with requires_grad_(False), two gloo ranks,
checkpoints and --pretrained from this project's own checkpoint, and the deterministic split-K rows."""
import contextlib
import io
import os
import socket
import subprocess
import sys

import pytest
import torch

from distributed_vgg_f_b200 import cli, ops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ARGV = ["-iu", "x", "-rn", "0", "-ws", "1", "-rd", "/r"]
BASE = ["-iu", "tcp://127.0.0.1:29999", "-rn", "0", "-ws", "1", "-nc", "-mb", "4", "--model", "vggf-tiny",
        "--engine", "oracle"]
needs_ext = pytest.mark.skipif(not ops.available(), reason="needs the built extension (host code only)")


# ------------------------------------------------------------------------------------------------ flag
@pytest.mark.parametrize("model,layers", [("vggf", 17), ("vgg16", 16), ("vgg11", 11), ("vggf-tiny", 17),
                                          ("vggf19", 20)])
def test_flag_range_follows_the_model(model, layers):
    assert cli.parse_command_line(ARGV + ["--model", model], init=False).freeze_layers == 0
    for n in (1, layers - 4, layers - 1):
        assert cli.parse_command_line(ARGV + ["--model", model, "--freeze-layers", str(n)], init=False).freeze_layers == n
    for n in (-1, layers, layers + 3):
        with pytest.raises(SystemExit):
            cli.parse_command_line(ARGV + ["--model", model, "--freeze-layers", str(n)], init=False)


def test_flag_reaches_the_native_engine(monkeypatch, tmp_path, capsys):
    """manage_training passes freeze_layers= to NativeEngine (stopped at construction: no GPU here) and prints
    one [Info] line naming the frozen layers, only when some are frozen."""
    from distributed_vgg_f_b200 import train
    from distributed_vgg_f_b200.engine import native_engine

    seen = {}

    class Stop(Exception):
        pass

    def fake(*a, **k):
        seen.update(k)
        raise Stop

    monkeypatch.setattr(native_engine, "NativeEngine", fake)
    monkeypatch.setattr(train, "_want_native", lambda args, device: True)
    for extra, want in (([], 0), (["--freeze-layers", "13"], 13)):
        argv = ["-iu", "x", "-rn", "0", "-ws", "1", "-rd", str(tmp_path / "s"), "-nc", "-mb", "4", "--model",
                "vggf-tiny", "--synthetic", "2"] + extra
        capsys.readouterr()
        with pytest.raises(Stop):
            train.manage_training(cli.parse_command_line(argv))
        assert seen["freeze_layers"] == want
        info = [s for s in capsys.readouterr().out.splitlines() if s.startswith("[Info] frozen layers")]
        if want:
            from distributed_vgg_f_b200.models.vggf import vggf_tiny_spec

            spec = vggf_tiny_spec(3)
            count = sum(torch.Size(spec.param_shape(t)).numel() for t in spec.frozen_param_names(13))
            assert info == ["[Info] frozen layers: features.0 .. features.28 (13 layers, %d parameters)" % count]
        else:
            assert info == []


# ----------------------------------------------------------------------------------------- bucket plan
def _ready(model="vggf"):
    from distributed_vgg_f_b200.models import layout as L
    from distributed_vgg_f_b200.models.vggf import get_spec

    spec = get_spec(model, 3)
    return spec, L.ready_order(spec)


def _parents_plan(ready, bucket_mb=32.0, conv_bucket_mb=9.5, tail_bucket_kb=2400.0):
    """engine_bucket_plan as it was before trainable= existed."""
    from distributed_vgg_f_b200.parallel.buckets import make_bucket_plan

    cap = int(bucket_mb * 1024 * 1024 / 4)
    first_conv = next((n for n, _ in ready if n.startswith("features.")), "")
    return make_bucket_plan(ready, cap_elems=cap, late_cap_elems=min(cap, int(conv_bucket_mb * 1024 * 1024 / 4)),
                            late_from=first_conv, tail_elems=int(tail_bucket_kb * 1024 / 4))


@pytest.mark.parametrize("model", ["vggf", "vgg16", "vggf-tiny", "vggf-mini"])
@pytest.mark.parametrize("sizes", [(32.0, 9.5, 2400.0), (8.0, 2.0, 300.0)])
def test_no_frozen_layer_is_the_parents_plan_field_by_field(model, sizes):
    from distributed_vgg_f_b200.parallel.buckets import engine_bucket_plan

    _, ready = _ready(model)
    want = _parents_plan(ready, *sizes)
    for got in (engine_bucket_plan(ready, *sizes), engine_bucket_plan(ready, *sizes, trainable=len(ready))):
        assert got.offsets == want.offsets and got.numels == want.numels and got.order == want.order
        assert got.total == want.total and got.align == want.align and got.buckets == want.buckets
        assert got.grad_total == got.total


@pytest.mark.parametrize("model,n", [("vggf", 1), ("vggf", 7), ("vggf", 10), ("vggf", 13), ("vggf", 16),
                                     ("vgg16", 13), ("vgg16", 15), ("vggf-mini", 12)])
def test_frozen_layers_keep_their_offsets_and_leave_the_buckets(model, n):
    from distributed_vgg_f_b200.parallel.buckets import engine_bucket_plan

    spec, ready = _ready(model)
    full = engine_bucket_plan(ready)
    frozen = spec.frozen_param_names(n)
    plan = engine_bucket_plan(ready, trainable=len(ready) - len(frozen))
    assert plan.offsets == full.offsets and plan.numels == full.numels and plan.order == full.order
    assert plan.total == full.total
    T = min(full.offsets[t] for t in frozen)
    assert plan.grad_total == T
    # the buckets tile [0, T) exactly, hold every trainable tensor and no frozen one
    assert plan.buckets[0].start == 0 and plan.buckets[-1].end == T
    assert all(a.end == b.start for a, b in zip(plan.buckets, plan.buckets[1:]))
    assert all(b.start % plan.align == 0 for b in plan.buckets)
    inside = {t for b in plan.buckets for t in b.tensors}
    assert inside == {t for t, _ in ready} - set(frozen)
    for t in frozen:
        assert plan.bucket_of(t) == [] and plan.offsets[t] >= T
    # the tail rule holds for the last trainable layers: the final bucket is the longest suffix of the
    # trainable ready order within 2400 KB (or the one tensor that is larger)
    trainable = [t for t, _ in ready if t not in frozen]
    limit = 2400 * 1024 // 4
    suffix = [t for t in trainable if T - full.offsets[t] <= limit]
    assert suffix == trainable[len(trainable) - len(suffix):]
    tail = plan.buckets[-1]
    if suffix:
        assert tail.tensors == tuple(suffix) and tail.start == full.offsets[suffix[0]]
    else:                                    # the last trainable tensor alone is larger than the tail
        assert tail.tensors == (trainable[-1],)


def test_bucket_plan_refuses_an_empty_trainable_set():
    from distributed_vgg_f_b200.parallel.buckets import engine_bucket_plan

    _, ready = _ready()
    for bad in (0, len(ready) + 1):
        with pytest.raises(ValueError):
            engine_bucket_plan(ready, trainable=bad)


def test_tools_plan_prints_the_frozen_layers_T_and_the_buckets():
    from distributed_vgg_f_b200.parallel.buckets import engine_bucket_plan
    from distributed_vgg_f_b200.tools import plan

    spec, ready = _ready()
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        assert plan.main(["--freeze-layers", "13", "--world", "8"]) == 0
    out = buf.getvalue().splitlines()
    T = engine_bucket_plan(ready, trainable=8).grad_total
    frozen = [s for s in out if s.startswith("frozen:")]
    assert len(frozen) == 1 and "13 layers, features.0 .. features.28" in frozen[0] and "T = %d" % T in frozen[0]
    rows = [s for s in out if s[:3].strip().isdigit()]
    assert rows and not any("features." in s for s in rows)
    # without the flag: no frozen line, and the conv buckets are there
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        assert plan.main([]) == 0
    assert "frozen:" not in buf.getvalue() and "features.28" in buf.getvalue()
    with pytest.raises(SystemExit):
        plan.main(["--freeze-layers", "17"])


# ------------------------------------------------------------------------------------ torch-op engine
def _run(argv):
    from distributed_vgg_f_b200.train import manage_training

    return manage_training(cli.parse_command_line(argv))


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


def _plain_optimizer(params, opt, wd, bwd):
    named = list(params)
    if bwd is None:
        groups = [{"params": [p for _, p in named], "weight_decay": wd}]
    else:
        groups = [{"params": [p for n, p in named if not n.endswith(".bias")], "weight_decay": wd},
                  {"params": [p for n, p in named if n.endswith(".bias")], "weight_decay": bwd}]
    if opt == "sgd":
        return torch.optim.SGD(groups, lr=0.01, momentum=0.9, weight_decay=wd)
    if opt == "adamw":
        return torch.optim.AdamW(groups, lr=0.01, weight_decay=wd)
    return torch.optim.Adam(groups, lr=0.01, weight_decay=wd)


@pytest.mark.parametrize("opt,n,wd,bwd", [("adam", 13, 0.0, None), ("adamw", 7, 0.05, 0.01), ("sgd", 16, 1e-3, None)])
def test_torch_op_trainer_matches_a_plain_loop_with_requires_grad_off(synth_root, tmp_path, monkeypatch, no_dropout,
                                                                     opt, n, wd, bwd):
    import torch.nn.functional as F

    from distributed_vgg_f_b200.models.vggf import build_oracle, vggf_tiny_spec
    from distributed_vgg_f_b200.trainer import Trainer

    seen = []
    real = Trainer._mixed_to_device

    def record(self, batch):
        out = real(self, batch)
        seen.append((out[0].clone(), out[1].clone()))
        return out
    monkeypatch.setattr(Trainer, "_mixed_to_device", record)
    path = str(tmp_path / "c.pt")
    extra = ["--optimizer", opt, "--weight-decay", str(wd), "--freeze-layers", str(n)]
    if bwd is not None:
        extra += ["--bias-weight-decay", str(bwd)]
    _run(BASE + ["-rd", synth_root, "-lr", "0.01", "-ep", "1", "--save", path] + extra)
    got = torch.load(path, weights_only=True)

    spec = vggf_tiny_spec(3)
    start = build_oracle(spec, seed=0).state_dict()
    frozen = set(spec.frozen_param_names(n))
    model = build_oracle(spec, seed=0)
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    for name, p in model.named_parameters():
        if name in frozen:
            p.requires_grad_(False)
    o = _plain_optimizer([(k, p) for k, p in model.named_parameters() if p.requires_grad], opt, wd, bwd)
    model.train()
    for x, y in seen:
        loss = F.cross_entropy(model(x), y)
        o.zero_grad()
        loss.backward()
        o.step()
    want = model.state_dict()
    assert len(got["model"]) == 34 and set(got["model"]) == {"module." + k for k in spec.param_names}
    for name in spec.param_names:
        g = got["model"]["module." + name]
        if name in frozen:
            assert torch.equal(g, start[name]), name              # untouched, bit for bit
        else:
            assert not torch.equal(g, start[name]), name
            assert torch.equal(g, want[name]), name               # the plain loop, bit for bit
    st = got["optimizer"]
    assert st["frozen_layers"] == n
    assert len(st["state"]) == len(spec.param_names) - 2 * n      # state for the trainable tensors only
    assert sum(len(g["params"]) for g in st["param_groups"]) == len(spec.param_names) - 2 * n


def test_default_torch_op_checkpoint_has_no_frozen_key(synth_root, tmp_path):
    path = str(tmp_path / "c.pt")
    _run(BASE + ["-rd", synth_root, "-ep", "1", "--save", path])
    st = torch.load(path, weights_only=True)["optimizer"]
    assert "frozen_layers" not in st and len(st["state"]) == 34


def test_resume_with_another_frozen_count_is_refused_and_eval_only_is_not(synth_root, tmp_path):
    path = str(tmp_path / "c.pt")
    _run(BASE + ["-rd", synth_root, "-ep", "1", "--freeze-layers", "13", "--save", path])
    for other in ("0", "10"):
        with pytest.raises(ValueError, match=r"--freeze-layers 13, this run has --freeze-layers %s" % other):
            _run(BASE + ["-rd", synth_root, "-ep", "2", "--freeze-layers", other, "--resume", path])
    _run(BASE + ["-rd", synth_root, "-ep", "2", "--freeze-layers", "13", "--resume", path])     # same count: fine
    for other in ("0", "10", "13"):
        t = _run(BASE + ["-rd", synth_root, "--freeze-layers", other, "--resume", path, "--eval-only"])
        assert len(t.history) == 1


def test_native_engine_refuses_optimizer_state_of_another_frozen_count():
    """import_optimizer_state is host code: an engine shell without buffers is enough."""
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine

    eng = NativeEngine.__new__(NativeEngine)
    eng.freeze_layers = 0
    with pytest.raises(ValueError, match="--freeze-layers 13, this run has --freeze-layers 0"):
        eng.import_optimizer_state({"name": "adam", "step": 3, "frozen_layers": 13})
    eng.freeze_layers = 13
    with pytest.raises(ValueError, match="--freeze-layers 0, this run has --freeze-layers 13"):
        eng.import_optimizer_state({"name": "adam", "step": 3})


def test_two_gloo_ranks_stay_identical(synth_root, tmp_path):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    code = ("import sys, torch\n"
            "from distributed_vgg_f_b200.cli import parse_command_line\n"
            "from distributed_vgg_f_b200.train import manage_training\n"
            "a = parse_command_line(sys.argv[2:])\n"
            "t = manage_training(a)\n"
            "torch.save(t.model.state_dict(), sys.argv[1])\n")
    procs = []
    for r in range(2):
        cmd = [sys.executable, "-c", code, str(tmp_path / ("r%d.pt" % r)), "-iu", "tcp://127.0.0.1:%d" % port,
               "-rn", str(r), "-ws", "2", "-rd", synth_root, "-ep", "2", "-nc", "-lr", "0.001", "-mb", "4",
               "--model", "vggf-tiny", "--engine", "oracle", "--freeze-layers", "13", "--optimizer", "adamw",
               "--weight-decay", "0.05"]
        env = dict(os.environ, PYTHONPATH=ROOT, OMP_NUM_THREADS="2")
        procs.append(subprocess.Popen(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                                      text=True))
    outs = [p.communicate(timeout=600)[0] for p in procs]
    assert all(p.returncode == 0 for p in procs), outs
    from distributed_vgg_f_b200.models.vggf import build_oracle, vggf_tiny_spec

    spec = vggf_tiny_spec(3)
    start = build_oracle(spec, seed=0).state_dict()
    a, b = (torch.load(str(tmp_path / ("r%d.pt" % r)), weights_only=True) for r in range(2))
    frozen = set(spec.frozen_param_names(13))
    for name in spec.param_names:
        k = "module." + name
        assert torch.equal(a[k], b[k]), name
        assert torch.equal(a[k], start[name]) == (name in frozen), name


# ----------------------------------------------------------------------------------------- --pretrained
def test_pretrained_takes_this_projects_checkpoint_whole(tmp_path):
    from distributed_vgg_f_b200.models.vggf import build_oracle, load_pretrained_vgg16_, vggf_tiny_spec
    from distributed_vgg_f_b200.utils import checkpoint as ckpt

    spec = vggf_tiny_spec(3)
    src = build_oracle(spec, seed=7)
    path = str(tmp_path / "stage1.pt")
    ckpt.save_checkpoint(path, src, None, 3, {"freeze_layers": 13})
    state = torch.load(path, map_location="cpu")            # what --pretrained loads
    dst = build_oracle(spec, seed=0)
    loaded = load_pretrained_vgg16_(dst, state)
    assert sorted(loaded) == sorted(spec.param_names) and len(loaded) == 34
    for k, v in src.state_dict().items():
        assert torch.equal(dst.state_dict()[k], v), k


def test_pretrained_torchvision_state_dict_loads_what_it_loaded_before():
    from distributed_vgg_f_b200.models.vggf import build_oracle, load_pretrained_vgg16_, vggf_tiny_spec

    spec = vggf_tiny_spec(3)
    tv = {k: v for k, v in build_oracle(spec, seed=7).state_dict().items() if not k.startswith("classifier.6.")}
    tv["classifier.6.weight"], tv["classifier.6.bias"] = torch.randn(1000, 128), torch.randn(1000)
    dst = build_oracle(spec, seed=0)
    funnel = {k: v.clone() for k, v in dst.state_dict().items() if k.startswith("classifier.6.")}
    loaded = load_pretrained_vgg16_(dst, tv)
    assert sorted(loaded) == sorted(k for k in tv if not k.startswith("classifier.6."))     # 30: no funnel
    for k, v in dst.state_dict().items():
        assert torch.equal(v, funnel[k] if k in funnel else tv[k]), k


def test_stage_two_run_starts_from_the_stage_one_checkpoint(synth_root, tmp_path):
    """The fine-tune recipe: the head with features frozen, then everything from that result."""
    stage1 = str(tmp_path / "stage1.pt")
    _run(BASE + ["-rd", synth_root, "-ep", "1", "--freeze-layers", "13", "--save", stage1])
    t = _run(BASE + ["-rd", synth_root, "-ep", "0", "--pretrained", stage1])
    want = torch.load(stage1, weights_only=True)["model"]
    got = t.model.state_dict()
    assert len(want) == 34
    for k, v in want.items():
        assert torch.equal(got[k[len("module."):]], v), k


# ---------------------------------------------------------------------------------- --deterministic
@needs_ext
@pytest.mark.parametrize("model,fused,n", [("vggf", True, 7), ("vggf", True, 8), ("vggf", True, 13),
                                           ("vggf", True, 16), ("vgg16", False, 15), ("vggf-mini", True, 3)])
def test_deterministic_rows_keep_the_forward_and_drop_the_frozen_backward(model, fused, n):
    from distributed_vgg_f_b200.engine.native_engine import deterministic_plan
    from distributed_vgg_f_b200.models.vggf import get_spec

    spec = get_spec(model, 1000 if model == "vgg16" else 3)
    index = {l.name: i for i, l in enumerate(list(spec.convs) + list(spec.fcs))}
    full = deterministic_plan(spec, 64, 224 if model != "vggf-mini" else 64, 132, fused)
    got = deterministic_plan(spec, 64, 224 if model != "vggf-mini" else 64, 132, fused, freeze_layers=n)
    want = [r for r in full if r[1] == "fprop" or (r[1] in ("bias", "wgrad") and index[r[0]] >= n)
            or (r[1] == "dgrad" and index[r[0]] > n)]
    assert got == want
    assert not any(index[name] < n and what != "fprop" for name, what, _, _ in got)


def _flat_ddp_frozen_worker(rank, world, port):
    import torch.distributed as dist

    from distributed_vgg_f_b200.models.vggf import build_oracle, freeze_leading_layers_, vggf_tiny_spec
    from distributed_vgg_f_b200.parallel.ddp import FlatDDP

    dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%d" % port, rank=rank, world_size=world)
    try:
        spec = vggf_tiny_spec(3)
        model = build_oracle(spec, seed=rank)            # every rank starts from different weights
        frozen = set(freeze_leading_layers_(model, 13))
        ddp = FlatDDP(model)
        want = build_oracle(spec, seed=0).state_dict()
        for name, p in model.named_parameters():         # rank 0's, frozen tensors included (as DDP does)
            assert torch.equal(p.detach(), want[name]), (rank, name)
        assert set(ddp.plan.order) == set(spec.param_names) - frozen     # only trainable tensors are bucketed
    finally:
        dist.destroy_process_group()


def test_flat_ddp_broadcasts_frozen_tensors_too():
    import torch.multiprocessing as mp

    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    mp.spawn(_flat_ddp_frozen_worker, args=(2, port), nprocs=2, join=True)
