"""PowerSGD (--powersgd-rank) without a GPU: the compression rule, the initial Q draws, the exchange plan, the
refusals, the CLI, and the torch-op engine (FlatDDP(powersgd=...)) against torch's DistributedDataParallel with
powerSGD_hook on a spawned gloo world of two."""
import json
import os
import socket
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


# ------------------------------------------------------------------------------------------ host logic
def test_compression_rule_is_torchs():
    from torch.distributed.algorithms.ddp_comm_hooks.powerSGD_hook import _should_compress

    from distributed_vgg_f_b200.parallel import powersgd

    for n, m in ((4096, 25088), (512, 4608), (64, 27), (3, 512), (512, 1), (8, 8), (6, 10), (2, 64)):
        for r in (1, 2, 4, 8):
            rr = min(n, m, r)
            assert powersgd.should_compress(n, m, rr) == _should_compress(n, m, rr, 2)[0], (n, m, r)


def test_vggf_plan_counts():
    from distributed_vgg_f_b200.models.vggf import vggf_spec
    from distributed_vgg_f_b200.parallel import powersgd

    spec = vggf_spec(3)
    rows = powersgd.plan(spec, 4)
    comp = [t for t in rows if t.compressed]
    assert len(rows) == 34 and len(comp) == 16
    assert {t.name for t in rows if not t.compressed} == \
        {n for n in spec.param_names if n.endswith(".bias")} | {"classifier.6.3.weight"}
    assert sum(t.n * t.m for t in comp) == 136_345_280
    assert sum(t.pq_elems for t in rows) == 318_572
    assert sum(t.n * t.m for t in rows if not t.compressed) == 14_467
    b = powersgd.exchange_bytes(rows)
    assert b["compressed"] == 4 * 318_572 and b["uncompressed"] == 2 * 14_467
    assert b["without_powersgd"] == 2 * spec.num_params
    assert powersgd.exchange_bytes(powersgd.plan(spec, 1))["total"] < 0.36e6
    # frozen layers are no bucket of DDP's: they leave the plan
    assert [t.name for t in powersgd.plan(spec, 4, freeze_layers=13)] == [t.name for t in rows][:8]


class _OneRank:
    """The process group of a world of one: what powerSGD_hook asks of it."""

    def size(self) -> int:
        return 1


class _Done:
    """A finished all-reduce over a world of one: the tensor is its own sum."""

    def __init__(self, t):
        self.t = t

    def get_future(self):
        f = torch.futures.Future()
        f.set_result([self.t])
        return f


def test_initial_q_matches_the_hooks_draws(monkeypatch):
    """Run torch's powerSGD_hook itself over one-tensor buckets in DDP's order, at its first compressed iteration,
    and capture each bucket's Q as drawn (the argument of its first orthogonalisation, before it is used)."""
    import torch.distributed as dist
    from torch.distributed.algorithms.ddp_comm_hooks import powerSGD_hook as H

    from distributed_vgg_f_b200.models.vggf import vggf_tiny_spec
    from distributed_vgg_f_b200.parallel import powersgd

    spec = vggf_tiny_spec(3)
    rows = powersgd.plan(spec, 2)
    drawn, current = {}, [None]
    real = H._orthogonalize

    def capture(matrices, epsilon=0):
        if current[0] not in drawn:                  # the first call of a bucket orthogonalises the fresh draw
            drawn[current[0]] = matrices[0].clone()
        real(matrices, epsilon)
    monkeypatch.setattr(H, "_orthogonalize", capture)
    monkeypatch.setattr(dist, "all_reduce", lambda t, group=None, async_op=False: _Done(t))
    state = powersgd.make_state(2, 2, seed=7, process_group=_OneRank())
    state.iter = state.start_powerSGD_iter           # the hook's first compressed iteration
    g = torch.Generator().manual_seed(0)
    for j, t in enumerate(rows):
        current[0] = t.name
        flat = torch.randn(t.n * t.m, generator=g)
        H.powerSGD_hook(state, powersgd.HookBucket(j, flat, spec.param_shape(t.name), j == len(rows) - 1)).wait()
    got = powersgd.initial_q_torch(rows, seed=7)
    assert set(got) == set(drawn) == {t.name for t in rows if t.compressed}
    for name, q in got.items():
        assert torch.equal(q, drawn[name]), name


def test_native_column_order_round_trips():
    from distributed_vgg_f_b200.models import layout as L
    from distributed_vgg_f_b200.models.vggf import vggf_tiny_spec
    from distributed_vgg_f_b200.parallel import powersgd

    spec = vggf_tiny_spec(3)
    g = torch.Generator().manual_seed(0)
    for name in ("features.0.weight", "features.2.weight", "classifier.0.weight", "classifier.3.weight"):
        shape = spec.param_shape(name)
        w = torch.randn(*shape, generator=g)
        nat = L.to_native(spec, name, w).reshape(shape[0], -1)
        cols = powersgd.native_columns(spec, name)
        wt = w.reshape(shape[0], -1)
        for j, c in enumerate(cols.tolist()):
            assert torch.equal(nat[:, j], wt[:, c] if c >= 0 else torch.zeros(shape[0])), (name, j)
        q = torch.randn(wt.shape[1], 2, generator=g)
        qn = powersgd.q_to_native(spec, name, q)
        assert torch.equal(powersgd.q_to_torch(spec, name, qn), q)
        assert torch.allclose(nat.double() @ qn.double(), wt.double() @ q.double())   # P is the same in both orders


def test_bucket_plan_without_compressed_tensors_keeps_every_offset():
    from distributed_vgg_f_b200.models import layout as L
    from distributed_vgg_f_b200.models.vggf import vggf_spec
    from distributed_vgg_f_b200.parallel import powersgd
    from distributed_vgg_f_b200.parallel.buckets import engine_bucket_plan

    spec = vggf_spec(3)
    ready = L.ready_order(spec)
    comp = [t.name for t in powersgd.plan(spec, 4) if t.compressed]
    a, b = engine_bucket_plan(ready), engine_bucket_plan(ready, exclude=comp)
    assert a.offsets == b.offsets and a.total == b.total and a.order == b.order
    covered = set()
    for bk in b.buckets:
        assert not set(bk.tensors) & set(comp)
        covered |= set(bk.tensors)
    assert covered == {n for n, _ in ready} - set(comp)
    for name in comp:                            # no bucket range overlaps a compressed tensor's range
        s0, s1 = b.offsets[name], b.offsets[name] + b.numels[name]
        assert all(bk.end <= s0 or bk.start >= s1 for bk in b.buckets), name
    assert engine_bucket_plan(ready, exclude=()).buckets == a.buckets


def test_plan_tool_prints_the_exchange(capsys):
    from distributed_vgg_f_b200.tools import plan

    plan.main(["--model", "vggf", "--powersgd-rank", "4"])
    out = capsys.readouterr().out
    assert "16 of 34 tensors compressed" in out
    assert "318572 P + Q elements" in out
    assert "classifier.0.weight" in out and "4096" in out and "25088" in out


def test_refusals():
    from distributed_vgg_f_b200.parallel import powersgd

    with pytest.raises(ValueError, match="register budget"):
        powersgd.check_config(9, 1000)
    with pytest.raises(ValueError, match=">= 2"):
        powersgd.check_config(4, 1)
    powersgd.check_config(0, 0)                  # off: the start iteration does not matter
    with pytest.raises(ValueError, match="ZeRO-1 shards"):
        powersgd.resolve_zero1(True, 4)
    assert powersgd.resolve_zero1("auto", 4) is False and powersgd.resolve_zero1("auto", 0) == "auto"
    with pytest.raises(ValueError, match="summation order"):
        powersgd.check_deterministic(4, True, 2)
    powersgd.check_deterministic(4, True, 1)


CLI = ["-iu", "tcp://127.0.0.1:1", "-rn", "0", "-ws", "1", "-rd", "/nonexistent"]


@pytest.mark.parametrize("argv,msg", [
    (["--powersgd-rank", "9"], "register budget"),
    (["--powersgd-rank", "2", "--powersgd-start-iter", "1"], ">= 2"),
    (["--powersgd-rank", "2", "--zero1", "on"], "ZeRO-1"),
    (["--powersgd-rank", "2", "--deterministic", "-ws", "2"], "summation order"),
])
def test_cli_refusals(argv, msg, capsys):
    from distributed_vgg_f_b200 import cli

    with pytest.raises(SystemExit):
        cli.parse_command_line(CLI + argv, init=False)
    assert msg in capsys.readouterr().err


def test_cli_round_trip():
    from distributed_vgg_f_b200 import cli

    a = cli.parse_command_line(CLI + ["--powersgd-rank", "4", "--powersgd-start-iter", "10"], init=False)
    assert (a.powersgd_rank, a.powersgd_start_iter) == (4, 10)
    a = cli.parse_command_line(CLI, init=False)
    assert (a.powersgd_rank, a.powersgd_start_iter) == (0, 1000)


def test_native_engine_checkpoint_records_rank_and_start():
    """export_optimizer_state is host code: an engine shell with empty arenas is enough."""
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine
    from distributed_vgg_f_b200.models.vggf import vggf_tiny_spec

    eng = NativeEngine.__new__(NativeEngine)
    eng.spec, eng.opt_name, eng.step_count, eng.micro_count, eng.lr = vggf_tiny_spec(3), "sgd", 5, 5, 0.1
    eng._frozen = set(eng.spec.param_names)      # no tensor state to export
    eng.powersgd_rank, eng.powersgd_start_iter = 4, 10
    st = eng.export_optimizer_state()
    assert st["powersgd"] == {"rank": 4, "start_iter": 10}
    eng.powersgd_rank = 0
    assert "powersgd" not in eng.export_optimizer_state()


# ------------------------------------------------------------------------------- gloo world of two
S = 2           # start iteration: updates 1..S uncompressed


def _worker(rank: int, port: int, r: int, accum: int, out: str) -> None:
    import torch.distributed as dist
    import torch.nn.functional as F
    from torch.distributed.algorithms.ddp_comm_hooks.powerSGD_hook import powerSGD_hook

    from distributed_vgg_f_b200.models.vggf import build_oracle, vggf_tiny_spec
    from distributed_vgg_f_b200.parallel import powersgd
    from distributed_vgg_f_b200.parallel.ddp import FlatDDP

    torch.set_num_threads(2)
    dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%d" % port, rank=rank, world_size=2)
    spec = vggf_tiny_spec(3)

    def model():
        m = build_oracle(spec, seed=0)
        for mod in m.modules():
            if isinstance(mod, torch.nn.Dropout):
                mod.p = 0.0
        return m

    ours = FlatDDP(model(), powersgd=powersgd.make_state(r, S, seed=3))
    plain = FlatDDP(model())
    ddp = torch.nn.parallel.DistributedDataParallel(model(), bucket_cap_mb=1e-7)
    def serial_hook(state, bucket):
        # gloo needs every rank to issue its collectives in one order; the hook issues P's and Q's all-reduces from
        # future callbacks, which would race the next bucket's: finish each bucket before DDP launches the next
        fut = powerSGD_hook(state, bucket)
        fut.wait()
        return fut
    ddp.register_comm_hook(powersgd.make_state(r, S, seed=3), serial_hook)
    opts = [torch.optim.SGD(w.module.parameters(), lr=0.05, momentum=0.9) for w in (ours, plain, ddp)]
    g = torch.Generator().manual_seed(100 + rank)        # each rank its own data
    rec = {"max_rel": [], "plain_equal": [], "buckets": None, "order": None}
    for u in range(S + 4):
        batches = [(torch.randn(4, 3, 32, 32, generator=g), torch.randint(0, 3, (4,), generator=g))
                   for _ in range(accum)]
        for w in (ours, plain):
            w.zero_grad()
            for k, (x, y) in enumerate(batches):
                w._require_sync = k == accum - 1
                F.cross_entropy(w(x), y).backward()
                w.finish_backward()
        for p in plain.module.parameters():              # the trainer's group mean for the plain wrapper
            p.grad.mul_(1.0 / accum)
        opts[2].zero_grad()
        for k, (x, y) in enumerate(batches):
            if k < accum - 1:
                with ddp.no_sync():
                    (F.cross_entropy(ddp(x), y) / accum).backward()
            else:
                (F.cross_entropy(ddp(x), y) / accum).backward()
        for o in opts:
            o.step()
        a, b, c = ours.module.state_dict(), plain.module.state_dict(), ddp.module.state_dict()
        rec["max_rel"].append(max(((a[n] - c[n]).abs().max() / c[n].abs().max().clamp_min(1e-30)).item()
                                  for n in spec.param_names))
        rec["plain_equal"].append(all(torch.equal(a[n], b[n]) for n in spec.param_names))
    # DDP's buckets after its rebuild: one parameter each, in this project's gradient-ready order
    rec["buckets"] = len(ddp.reducer._get_zeros_like_grad_buckets())
    rec["order"] = ours._ready_order == powersgd.hook_order(spec)
    with open(out, "w") as f:
        json.dump(rec, f)
    dist.destroy_process_group()


@pytest.mark.parametrize("r,accum", [(2, 1), (4, 1), (2, 2)])
def test_flat_ddp_matches_ddp_with_powersgd_hook_on_two_gloo_ranks(tmp_path, r, accum):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    env = dict(os.environ, PYTHONPATH=ROOT, OMP_NUM_THREADS="2")
    procs = [subprocess.Popen([sys.executable, __file__, str(k), str(port), str(r), str(accum),
                               str(tmp_path / ("r%d.json" % k))], cwd=ROOT, env=env, stdout=subprocess.PIPE,
                              stderr=subprocess.STDOUT, text=True) for k in range(2)]
    outs = [p.communicate(timeout=600)[0] for p in procs]
    assert all(p.returncode == 0 for p in procs), outs
    for k in range(2):
        rec = json.load(open(tmp_path / ("r%d.json" % k)))
        assert rec["buckets"] == 34 and rec["order"]
        assert all(rec["plain_equal"][:S]), rec               # updates <= S: the uncompressed exchange, bit for bit
        assert not any(rec["plain_equal"][S:]), rec           # then compression changes the update
        assert max(rec["max_rel"]) <= 1e-6, rec


if __name__ == "__main__":
    _worker(int(sys.argv[1]), int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4]), sys.argv[5])
