"""Gradient accumulation (``--accum-steps`` / ``Trainer(accum_steps=K)``) on the torch-op path, without a GPU:
one update per group of K mini-batches with the mean of their gradients, the epoch's last group shorter,
FlatDDP's all-reduce once per bucket per update, and the update counter across a checkpoint."""
import os
import socket

import pytest
import torch
from torch import nn

from distributed_vgg_f_b200 import cli
from distributed_vgg_f_b200.models.vggf import build_oracle, vggf_tiny_spec
from distributed_vgg_f_b200.trainer import Trainer

CPU = torch.device("cpu")
REQUIRED = ["-iu", "tcp://127.0.0.1:29999", "-rn", "0", "-ws", "1", "-rd", "/nonexistent"]


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _model(seed=0):
    """vggf-tiny with dropout off (p = 0), so that micro-batches and big batches see the same network."""
    m = build_oracle(vggf_tiny_spec(3), seed=seed)
    for mod in m.modules():
        if isinstance(mod, nn.Dropout):
            mod.p = 0.0
    return m


def _data(n, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, 3, 64, 64, generator=g), torch.randint(0, 3, (n,), generator=g)


def _split(x, y, b):
    return [(x[i:i + b], y[i:i + b]) for i in range(0, x.shape[0], b)]


def _flat(model):
    return torch.cat([p.detach().flatten() for p in model.parameters()])


class _CountingSGD(torch.optim.SGD):
    """SGD that keeps a copy of the gradients it was stepped with."""

    def __init__(self, params, **kw):
        super().__init__(params, **kw)
        self.seen = []

    def step(self, closure=None):
        self.seen.append([p.grad.clone() for g in self.param_groups for p in g["params"]])
        return super().step(closure)


# ------------------------------------------------------------------------------------------- CLI
def test_cli_accum_steps_default_and_validation(capsys):
    assert cli.parse_command_line(REQUIRED, init=False).accum_steps == 1
    assert cli.parse_command_line(REQUIRED + ["--accum-steps", "4"], init=False).accum_steps == 4
    for bad in ("0", "-2"):
        with pytest.raises(SystemExit):
            cli.parse_command_line(REQUIRED + ["--accum-steps", bad], init=False)
    assert "--accum-steps must be >= 1" in capsys.readouterr().err


def test_trainer_refuses_bad_accum_steps():
    with pytest.raises(ValueError):
        Trainer(_model(), None, [], [], CPU, accum_steps=0)
    with pytest.raises(ValueError, match="__len__"):
        Trainer(_model(), None, iter([]), [], CPU, accum_steps=2)
    Trainer(_model(), None, iter([]), [], CPU, accum_steps=1)      # K = 1 needs no length


# ------------------------------------------------------------------------------- equivalence
@pytest.mark.parametrize("optimizer", ["sgd", "adam"])
def test_four_micro_batches_equal_one_big_batch(optimizer):
    """K = 4 x mb 4 against K = 1 x mb 16, two updates: the same weights up to fp32 rounding."""
    x, y = _data(32)
    out = {}
    for K, b in ((1, 16), (4, 4)):
        model = _model()
        # Adam with eps = 1: the update is smooth in g (with eps = 1e-8 the first steps are ~lr * sign(g),
        # and a near-zero gradient whose rounding differs would flip a weight by 2 lr)
        opt = torch.optim.SGD(model.parameters(), lr=0.05, momentum=0.9) if optimizer == "sgd" else \
            torch.optim.Adam(model.parameters(), lr=1e-3, eps=1.0)
        tr = Trainer(model, opt, _split(x, y, b), [], CPU, verbose_throughput=False, accum_steps=K)
        loss, acc = tr._train()
        assert acc.count == 32                       # metrics count every micro-batch
        out[K] = (_flat(model), opt.state_dict()["state"][0]["step"] if optimizer == "adam" else None)
    p0 = _flat(_model())
    assert not torch.allclose(out[1][0], p0), "the weights did not move"
    assert torch.allclose(out[4][0], out[1][0], rtol=1e-5, atol=1e-6), float((out[4][0] - out[1][0]).abs().max())
    if optimizer == "adam":
        assert int(out[4][1]) == int(out[1][1]) == 2         # Adam's step counts updates


def test_tail_group_is_shorter_and_scaled_by_its_own_size():
    """5 batches with K = 2: updates after batches 2, 4 and 5; the last one is batch 5's gradient x 1.
    lr = 0 keeps the weights fixed, so every gradient is taken at the same point."""
    x, y = _data(10, seed=3)
    batches = _split(x, y, 2)
    model = _model()
    opt = _CountingSGD(model.parameters(), lr=0.0)
    Trainer(model, opt, batches, [], CPU, verbose_throughput=False, accum_steps=2)._train()
    assert len(opt.seen) == 3
    ref = []
    for bx, by in batches:
        model.zero_grad()
        nn.functional.cross_entropy(model(bx), by).backward()
        ref.append([p.grad.clone() for p in model.parameters()])
    want = [[(a + b) / 2 for a, b in zip(ref[0], ref[1])], [(a + b) / 2 for a, b in zip(ref[2], ref[3])], ref[4]]
    for u, (got, exp) in enumerate(zip(opt.seen, want)):
        for a, b in zip(got, exp):
            assert torch.allclose(a, b, rtol=1e-5, atol=1e-7), u


# ---------------------------------------------------------------------------- FlatDDP, gloo ws 2
class _CountingCollective:
    """TorchCollective that counts the bucket all-reduces it is asked for."""

    def __init__(self):
        from distributed_vgg_f_b200.parallel.ddp import TorchCollective

        self.inner = TorchCollective()
        self.calls = []

    def allocate(self, numel, dtype, device):
        return self.inner.allocate(numel, dtype, device)

    def broadcast_(self, flat, src=0):
        self.inner.broadcast_(flat, src)

    def allreduce_range_async(self, flat, start, end):
        self.calls.append((start, end))
        return self.inner.allreduce_range_async(flat, start, end)


def _ddp_accum_worker(rank, world, port):
    import torch.distributed as dist

    from distributed_vgg_f_b200.parallel.ddp import FlatDDP

    torch.set_num_threads(2)
    dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%d" % port, rank=rank, world_size=world)
    x, y = _data(16, seed=5)
    # per update: rank r takes micro-batches of 2 at [8u + 4r, 8u + 4r + 2) and [8u + 4r + 2, 8u + 4r + 4)
    mine = [(x[8 * u + 4 * rank + 2 * j:8 * u + 4 * rank + 2 * j + 2], y[8 * u + 4 * rank + 2 * j:8 * u + 4 * rank + 2 * j + 2])
            for u in range(2) for j in range(2)]
    coll = _CountingCollective()
    ddp = FlatDDP(_model(seed=rank), collective=coll, bucket_cap_mb=0.05)      # rank 1's init is replaced
    n_buckets = len(ddp.plan.buckets)
    assert n_buckets > 3
    opt = torch.optim.SGD(ddp.parameters(), lr=0.05, momentum=0.9)
    Trainer(ddp, opt, mine, [], CPU, verbose_throughput=False, accum_steps=2)._train()
    assert sorted(coll.calls) == sorted([(b.start, b.end) for b in ddp.plan.buckets] * 2), \
        "expected one all-reduce per bucket per update"
    flat = _flat(ddp.module)
    ref = flat.clone()
    dist.broadcast(ref, 0)
    assert torch.equal(flat, ref), "replicas diverged"
    single = _model()
    sopt = torch.optim.SGD(single.parameters(), lr=0.05, momentum=0.9)
    Trainer(single, sopt, _split(x, y, 8), [], CPU, verbose_throughput=False)._train()
    assert torch.allclose(flat, _flat(single), rtol=1e-5, atol=1e-6), float((flat - _flat(single)).abs().max())
    dist.destroy_process_group()


def test_flat_ddp_accumulation_two_ranks_gloo():
    import torch.multiprocessing as mp

    mp.spawn(_ddp_accum_worker, args=(2, _free_port()), nprocs=2, join=True)


# ------------------------------------------------------------------------------ checkpoint
def test_checkpoint_resume_keeps_the_update_count(synth_root, tmp_path, capsys):
    """24 training images at mb 4 = 6 batches per epoch; --accum-steps 4 -> groups of 4 and 2 = 2 updates.
    The checkpoint's optimizer step counts updates, and a resumed run continues from it."""
    ck = str(tmp_path / "ck.pt")
    base = REQUIRED[:-1] + [synth_root, "-nc", "-mb", "4", "--model", "vggf-tiny", "--engine", "oracle",
                            "--accum-steps", "4", "--save", ck]
    assert cli.main(base + ["-ep", "1"]) == 0
    step = torch.load(ck, weights_only=False)["optimizer"]["state"][0]["step"]
    assert int(step) == 2
    assert cli.main(base + ["-ep", "2", "--resume", ck]) == 0
    out = capsys.readouterr().out
    assert "resumed from" in out and "[Info] Epoch: 2/2," in out
    payload = torch.load(ck, weights_only=False)
    assert payload["epoch"] == 2 and int(payload["optimizer"]["state"][0]["step"]) == 4


def test_native_engine_counters_round_trip_and_pending_refusal():
    """The native engine's optimizer state carries both counters (updates: Adam / SGD step, micro-batches:
    the dropout offset), and export refuses while a group has pending gradients.  Host logic only: the
    engine is assembled without its device buffers."""
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine
    from distributed_vgg_f_b200.models import layout as L
    from distributed_vgg_f_b200.parallel.buckets import engine_bucket_plan

    spec = vggf_tiny_spec(3)
    eng = NativeEngine.__new__(NativeEngine)
    eng.spec, eng.device, eng.opt_name, eng.lr = spec, CPU, "sgd", 1e-3
    eng.plan = engine_bucket_plan(L.ready_order(spec), 32.0, 9.5, 2400.0)
    eng.m32, eng.v32 = torch.zeros(eng.plan.total), None
    eng.p32 = torch.zeros(eng.plan.total)
    eng._zero1_buckets = set()
    eng.step_count, eng.micro_count, eng._accum = 3, 11, 0
    st = eng.export_optimizer_state()
    assert (st["step"], st["micro_step"]) == (3, 11)
    eng.step_count = eng.micro_count = 0
    eng.import_optimizer_state(st)
    assert (eng.step_count, eng.micro_count) == (3, 11)
    eng.import_optimizer_state({"name": "sgd", "step": 5})      # a checkpoint written before accumulation
    assert (eng.step_count, eng.micro_count) == (5, 5)
    eng._accum = 2
    for call in (eng.export_state, eng.prepare_export):
        with pytest.raises(RuntimeError, match="await an update"):
            call()


@pytest.mark.skipif(os.environ.get("B200_SKIP_SLOW", "0") == "1", reason="B200_SKIP_SLOW=1")
def test_cli_accum_steps_trains_on_cpu(tmp_path, capsys):
    """``--accum-steps 4 -nc`` end to end on a --synthetic set (torch-op engine)."""
    root = str(tmp_path / "synth")
    argv = ["-iu", "tcp://127.0.0.1:29999", "-rn", "0", "-ws", "1", "-rd", root, "-ep", "1", "-nc", "-mb", "4",
            "--model", "vggf-tiny", "--synthetic", "6", "--accum-steps", "4"]
    assert cli.main(argv) == 0
    out = capsys.readouterr().out
    assert "accum_steps=4" in out and "[Info] Epoch: 1/1, train loss:" in out
