"""LAMB and LARS without a GPU: the package's optimizer classes against a float64 NumPy transcription of the
formulas, the flags and their refusals, the phase-1 / phase-2 launch plan over the engine's buckets, a two-rank gloo
run against one process with the doubled batch, and a torch-op engine checkpoint round trip."""
import os
import socket

import numpy as np
import pytest
import torch

from distributed_vgg_f_b200.config import TRAIN
from distributed_vgg_f_b200.utils.optim import Lamb, Lars

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------ the formulas
def _lamb64(p, g, m, v, t, lr, wd):
    b1, b2, eps = TRAIN.lamb_beta1, TRAIN.lamb_beta2, TRAIN.lamb_eps
    m = b1 * m + (1 - b1) * g
    v = b2 * v + (1 - b2) * g * g
    u = (m / (1 - b1 ** t)) / (np.sqrt(v) / np.sqrt(1 - b2 ** t) + eps) + wd * p
    pn, un = np.linalg.norm(p), np.linalg.norm(u)
    r = pn / un if (wd != 0 and pn > 0 and un > 0) else 1.0
    return p - lr * r * u, m, v


def _lars64(p, g, buf, first, lr, wd, momentum):
    pn, gn = np.linalg.norm(p), np.linalg.norm(g)
    r = TRAIN.lars_trust_coeff * pn / (gn + wd * pn + TRAIN.lars_eps) if (wd != 0 and pn > 0 and gn > 0) else 1.0
    d = r * (g + wd * p)
    buf = d if first else momentum * buf + d
    return p - lr * buf, buf


@pytest.mark.parametrize("kind", ["lamb", "lars"])
def test_package_optimizers_match_the_float64_formulas(kind):
    """Four steps over two parameter groups (weights at a decay, biases at 0), a tensor of zero weights (ratio 1) and
    a frozen tensor without a gradient that must not move and keep no state."""
    rng = np.random.default_rng(3)
    shapes = {"w1": (7, 5), "w0": (6,), "b1": (5,), "frozen": (4, 4)}
    init = {n: rng.standard_normal(s) * 0.1 for n, s in shapes.items()}
    init["w0"][:] = 0.0
    params = {n: torch.tensor(v, dtype=torch.float64, requires_grad=n != "frozen") for n, v in init.items()}
    wd, lr = 0.3, 0.05
    groups = [{"params": [params["w1"], params["w0"], params["frozen"]], "weight_decay": wd},
              {"params": [params["b1"]], "weight_decay": 0.0}]
    opt = Lamb(groups, lr=lr) if kind == "lamb" else Lars(groups, lr=lr, momentum=0.9)
    ref = {n: v.copy() for n, v in init.items()}
    st = {n: (np.zeros(s), np.zeros(s)) for n, s in shapes.items()}
    for t in range(1, 5):
        grads = {n: rng.standard_normal(s) * 10.0 ** rng.uniform(-3, 0) for n, s in shapes.items()}
        for n, p in params.items():
            p.grad = None if n == "frozen" else torch.tensor(grads[n])
        opt.step()
        for n in shapes:
            if n == "frozen":
                continue
            d = wd if n != "b1" else 0.0
            if kind == "lamb":
                ref[n], m, v = _lamb64(ref[n], grads[n], *st[n], t, lr, d)
                st[n] = (m, v)
            else:
                ref[n], buf = _lars64(ref[n], grads[n], st[n][0], t == 1, lr, d, 0.9)
                st[n] = (buf, None)
        for n in shapes:
            np.testing.assert_allclose(params[n].detach().numpy(), ref[n], rtol=1e-12, atol=1e-14, err_msg=n)
    assert params["frozen"] not in opt.state
    assert np.array_equal(params["frozen"].detach().numpy(), init["frozen"])


# ------------------------------------------------------------------------------------ flags
def _parse(extra, ws="1"):
    from distributed_vgg_f_b200 import cli
    return cli.parse_command_line(["-iu", "x", "-rn", "0", "-ws", ws, "-rd", "/r"] + extra, init=False)


@pytest.mark.parametrize("kind", ["lamb", "lars"])
def test_flags_take_the_new_optimizers_and_refuse_what_would_not_adapt(kind):
    from distributed_vgg_f_b200.parallel import powersgd

    args = _parse(["--optimizer", kind, "--weight-decay", "0.01", "--bias-weight-decay", "0"])
    assert (args.optimizer, args.weight_decay, args.bias_weight_decay) == (kind, 0.01, 0.0)
    for extra, ws in ((["--optimizer", kind], "1"), (["--optimizer", kind, "--weight-decay", "0"], "1"),
                      (["--optimizer", kind, "--weight-decay", "0.01", "--zero1", "on"], "2")):
        with pytest.raises(SystemExit):
            _parse(extra, ws)
    assert _parse(["--optimizer", kind, "--weight-decay", "0.01", "--zero1", "on"]).zero1 == "on"   # one rank
    # auto: ZeRO-1 is for Adam / AdamW only; the engine resolves it off (z1_ok) and refuses "on" at world > 1
    assert _parse(["--optimizer", kind, "--weight-decay", "0.01", "--zero1", "auto"], "2").zero1 == "auto"
    assert powersgd.resolve_zero1("auto", 0) == "auto"


def test_build_optimizer_gives_the_package_classes_with_torchvisions_groups():
    import argparse

    from distributed_vgg_f_b200.models.vggf import build_oracle, get_spec
    from distributed_vgg_f_b200.train import build_optimizer

    model = build_oracle(get_spec("vggf-tiny", 3), seed=0)
    for kind, cls in (("lamb", Lamb), ("lars", Lars)):
        a = argparse.Namespace(optimizer=kind, learning_rate=0.1, momentum=0.8, weight_decay=0.02,
                               bias_weight_decay=0.0)
        opt = build_optimizer(model, a)
        assert isinstance(opt, cls) and [g["weight_decay"] for g in opt.param_groups] == [0.02, 0.0]
        with pytest.raises(ValueError):
            build_optimizer(model, argparse.Namespace(**dict(vars(a), weight_decay=0.0)))


# ------------------------------------------------------------------------------------ the launch plan
@pytest.mark.parametrize("model", ["vggf", "vgg16", "vggf-mini"])
@pytest.mark.parametrize("freeze", [0, 13])
@pytest.mark.parametrize("psgd", [0, 2])
def test_layerwise_plan_covers_every_tensor_once(model, freeze, psgd):
    """Every trainable tensor gets exactly one phase 2, issued after the phase 1 of its last piece; the slots of all
    tensors are dense and disjoint, a tensor's slots are exactly its phase-1 CTAs; no phase-1 segment spans two
    tensors, and no launch exceeds the segment or grid cap."""
    from distributed_vgg_f_b200.models.vggf import get_spec
    from distributed_vgg_f_b200.parallel import layerwise as lw

    spec = get_spec(model, 3)
    plans = lw.engine_layerwise_plans(spec, 132, freeze_layers=freeze, powersgd_rank=psgd)
    assert set(plans) == ({False, True} if psgd else {False})
    trainable = [n for n in spec.param_names if n not in set(spec.frozen_param_names(freeze))]
    for plan in plans.values():
        assert sorted(plan.tensors) == sorted(trainable)
        seen_p2, issued, slot_owner = {}, set(), {}
        for u, (s, e) in enumerate(plan.units):
            for L in plan.phase1[s]:
                assert s <= L.start < L.end <= e and len(L.segments) <= lw.MAX_SEGMENTS and L.grid <= 4 * 132
                bounds = [L.start + g.start for g in L.segments] + [L.end]
                for g, a, b in zip(L.segments, bounds, bounds[1:]):
                    name = plan.tensors[g.tensor]
                    lo, hi = plan.ranges[name]
                    assert lo <= a < b <= hi, "a phase-1 segment spans two tensors"
                    for k in range(g.slot, g.slot + g.ctas):
                        assert k not in slot_owner
                        slot_owner[k] = name
                    issued.add(name)
            for L in plan.phase2[s]:
                assert len(L.segments) <= lw.MAX_SEGMENTS and L.grid <= 4 * 132
                bounds = [L.start + g.start for g in L.segments] + [L.end]
                for g, a, b in zip(L.segments, bounds, bounds[1:]):
                    name = plan.tensors[g.tensor]
                    assert (a, b) == plan.ranges[name]
                    assert name not in seen_p2
                    seen_p2[name] = u
                    assert (g.slot, g.nslots) == plan.slots[name]
            # a tensor's phase 2 comes after the unit holding its last piece
            for name, uu in seen_p2.items():
                if uu == u:
                    lo, hi = plan.ranges[name]
                    assert all(not (a < hi and b > lo) for a, b in plan.units[u + 1:])
        assert sorted(seen_p2) == sorted(trainable)
        assert sorted(slot_owner) == list(range(plan.total_slots))
        for name, (base, count) in plan.slots.items():
            assert all(slot_owner[k] == name for k in range(base, base + count))


def test_plan_caps_are_the_kernels():
    from distributed_vgg_f_b200 import ops
    from distributed_vgg_f_b200.parallel import layerwise as lw

    if not ops.available():
        pytest.skip("needs the built extension")
    assert ops.require().layerwise_max_segments() == lw.MAX_SEGMENTS


def test_vggf_plan_runs_fc1_in_13_pieces_and_one_phase2():
    from distributed_vgg_f_b200.models.vggf import get_spec
    from distributed_vgg_f_b200.parallel import layerwise as lw

    plan = lw.engine_layerwise_plans(get_spec("vggf", 3), 132)[False]
    pieces = [s for s in plan.phase1 for L in plan.phase1[s] for g in L.segments
              if plan.tensors[g.tensor] == "classifier.0.weight"]
    assert len(pieces) == 13
    after = [s for s in plan.phase2 for L in plan.phase2[s] for g in L.segments
             if plan.tensors[g.tensor] == "classifier.0.weight"]
    assert after == [pieces[-1]] and plan.units.index((pieces[-1], plan.units[16][1])) == 16


def test_tools_plan_prints_the_layerwise_plan(capsys):
    from distributed_vgg_f_b200.tools import plan

    assert plan.main(["--optimizer", "lars", "--model", "vggf-mini", "--freeze-layers", "2", "--powersgd-rank", "2"]) == 0
    out = capsys.readouterr().out
    assert "phase-2 launches" in out and "updates PowerSGD compresses" in out


# ------------------------------------------------------------------------------------ torch-op engine
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _rank_main(rank, world, port, kind, batches, out):
    import argparse

    import torch.distributed as dist

    from distributed_vgg_f_b200.models.vggf import build_oracle, get_spec
    from distributed_vgg_f_b200.parallel.ddp import FlatDDP
    from distributed_vgg_f_b200.train import build_optimizer

    torch.set_num_threads(2)
    dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%d" % port, rank=rank, world_size=world)
    model = build_oracle(get_spec("vggf-tiny", 3), seed=0).eval()       # no dropout: the same function on every rank
    ddp = FlatDDP(model, bucket_cap_mb=1.0)
    opt = build_optimizer(model, argparse.Namespace(optimizer=kind, learning_rate=0.01, momentum=0.9,
                                                    weight_decay=0.05, bias_weight_decay=0.0))
    for x, y in batches:
        per = x.shape[0] // world
        out_ = ddp(x[rank * per:(rank + 1) * per])
        loss = torch.nn.functional.cross_entropy(out_, y[rank * per:(rank + 1) * per])
        ddp.zero_grad()                  # the gradients are views of its arena
        loss.backward()
        ddp.finish_backward()
        opt.step()
    torch.save({k: v.detach().clone() for k, v in model.state_dict().items()}, "%s.%d" % (out, rank))
    dist.destroy_process_group()


@pytest.mark.parametrize("kind", ["lamb"])
def test_two_gloo_ranks_equal_one_process_with_the_doubled_batch(tmp_path, kind):
    import torch.multiprocessing as mp

    g = torch.Generator().manual_seed(5)
    batches = [(torch.randn(8, 3, 64, 64, generator=g), torch.randint(0, 3, (8,), generator=g)) for _ in range(3)]
    mp.spawn(_rank_main, args=(2, _free_port(), kind, batches, str(tmp_path / "two")), nprocs=2, join=True)
    mp.spawn(_rank_main, args=(1, _free_port(), kind, batches, str(tmp_path / "one")), nprocs=1, join=True)
    r0, r1 = torch.load(str(tmp_path / "two.0")), torch.load(str(tmp_path / "two.1"))
    one = torch.load(str(tmp_path / "one.0"))
    from distributed_vgg_f_b200.models.vggf import build_oracle, get_spec
    init = build_oracle(get_spec("vggf-tiny", 3), seed=0).state_dict()
    for k in r0:
        assert torch.equal(r0[k], r1[k]), "replicas differ in %s" % k
        moved = float((one[k] - init[k]).abs().max())
        err = float((r0[k] - one[k]).abs().max())
        assert err <= 1e-3 * moved + 1e-6, "%s: two ranks %.3g from one process (moved %.3g)" % (k, err, moved)


@pytest.mark.parametrize("kind", ["lamb", "lars"])
def test_oracle_checkpoint_round_trip(tmp_path, kind):
    """The torch-op engine saves the optimizer class's own state dict and a resumed run continues exactly."""
    import argparse

    from distributed_vgg_f_b200.models.vggf import build_oracle, get_spec
    from distributed_vgg_f_b200.train import build_optimizer
    from distributed_vgg_f_b200.utils import checkpoint as ckpt

    args = argparse.Namespace(optimizer=kind, learning_rate=0.01, momentum=0.9, weight_decay=0.05,
                              bias_weight_decay=0.0)
    g = torch.Generator().manual_seed(1)
    batches = [(torch.randn(4, 3, 64, 64, generator=g), torch.randint(0, 3, (4,), generator=g)) for _ in range(3)]

    def step(model, opt, b):
        opt.zero_grad()
        torch.nn.functional.cross_entropy(model(b[0]), b[1]).backward()
        opt.step()

    spec = get_spec("vggf-tiny", 3)
    a = build_oracle(spec, seed=0).eval()
    oa = build_optimizer(a, args)
    step(a, oa, batches[0])
    step(a, oa, batches[1])
    ckpt.save_checkpoint(str(tmp_path / "c.pt"), a, oa, 1, {})
    step(a, oa, batches[2])
    b = build_oracle(spec, seed=7).eval()
    ob = build_optimizer(b, args)
    ckpt.load_checkpoint(str(tmp_path / "c.pt"), b, ob)
    step(b, ob, batches[2])
    for k, v in a.state_dict().items():
        assert torch.equal(v, b.state_dict()[k]), k
