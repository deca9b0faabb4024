"""Gradient accumulation on the native engine: ``train_step(batch, update=False)`` adds a micro-batch's
gradients to the arena; the updating micro-batch reduces and applies their mean.

* head_ce's accumulate mode against float64 on guarded operands: dW is added to, nothing else changes;
* the other launch signatures of an accumulating step, replayed on guarded operands (launch_replay.py);
* K micro-batches of b against one batch of K b on the gradient arena and after Adam / SGD updates;
* dropout draws a fresh mask per micro-batch; the counters survive export / import;
* with >= 2 GPUs: ws 2 x K 2 x b 4 against one process at b 16 on every reduction path.
"""
import os
import socket

import pytest
import torch

import guarded as G
import kernel_check as KC
from distributed_vgg_f_b200.ops import ref as R
from launch_replay import _batch, _Recorder, replay_all

pytestmark = pytest.mark.gpu
DEV = "cuda"
F64 = torch.float64


def _C():
    from distributed_vgg_f_b200 import ops
    return ops.require()


# --------------------------------------------------------------------------- head_ce accumulate
@pytest.mark.parametrize("B,C,K,weighted", [(64, 3, 512, False), (37, 3, 512, True), (16, 8, 1024, False),
                                            (4, 1, 96, True)])
def test_head_ce_accumulate_mode(B, C, K, weighted):
    """The same guarded launch in both modes: with accumulate dW = prefill + the batch's gradient; every
    other output (logits, dlogits, db, dh, meter, loss) is bit-identical to the storing launch, and
    nothing outside the written regions changes."""
    Cx = _C()
    g = torch.Generator(device=DEV).manual_seed(B * 100 + C + K)
    h = torch.relu(torch.randn(B, K, device=DEV, generator=g)).to(torch.bfloat16)
    W = (torch.randn(C, K, device=DEV, generator=g) * 0.1).to(torch.bfloat16)
    bias = torch.randn(C, device=DEV, generator=g) * 0.1
    t = torch.randint(0, C, (B,), device=DEV, generator=g)
    cw = torch.rand(C, device=DEV, generator=g) + 0.5 if weighted else None
    dW0 = torch.randint(-8, 9, (C, K), device=DEV, generator=g).float()
    db0 = torch.randint(-8, 9, (C,), device=DEV, generator=g).float()
    m0 = torch.randint(0, 9, (4,), device=DEV, generator=g).float()
    ldd = 8
    out = {}
    for acc in (False, True):
        ops = {
            "h": G.guarded((B, K), (K, 1), torch.bfloat16, 3, G.NAN, DEV, h),
            "W": G.guarded((C, K), (K, 1), torch.bfloat16, 0, G.NAN, DEV, W),
            "bias": G.guarded((C,), (1,), torch.float32, 0, G.NAN, DEV, bias),
            "target": G.guarded((B,), (1,), torch.int64, 0, C - 1, DEV, t),
            "logits": G.guarded((B, C), (C, 1), torch.float32, 0, G.NAN, DEV),
            "dlogits": G.guarded((B, ldd), (ldd, 1), torch.bfloat16, 0, G.NAN, DEV),
            "dW": G.guarded((C, K), (K, 1), torch.float32, 4, G.NAN, DEV, dW0),
            "db": G.guarded((C,), (1,), torch.float32, 0, G.NAN, DEV, db0),
            "dh": G.guarded((B, K), (K, 1), torch.bfloat16, 0, G.NAN, DEV),
            "meter": G.guarded((4,), (1,), torch.float32, 0, G.NAN, DEV, m0),
            "loss": G.guarded((1,), (1,), torch.float32, 0, G.NAN, DEV),
        }
        if cw is not None:
            ops["cw"] = G.guarded((C,), (1,), torch.float32, 0, G.NAN, DEV, cw)
        for op in ops.values():
            op.seal()
        T = {k: v.t for k, v in ops.items()}
        args = (T["h"], T["W"], T["bias"], T["target"], T["logits"], T["dlogits"], ldd, T["dW"], T["db"], T["dh"],
                2.0, True, T["meter"], T["loss"], T.get("cw"))
        if acc:
            Cx.head_ce(*args, True)
        else:
            Cx.head_ce(*args)
        torch.cuda.synchronize()
        written = {"logits": T["logits"], "dlogits": T["dlogits"], "dW": T["dW"], "db": T["db"], "dh": T["dh"],
                   "meter": T["meter"][:3], "loss": T["loss"]}
        for k, op in ops.items():
            op.check((written[k],) if k in written else (), what="head_ce accumulate=%s %s" % (acc, k))
        out[acc] = {k: v.clone() for k, v in T.items()}
    for k in ("logits", "dlogits", "db", "dh", "meter", "loss"):
        assert torch.equal(out[True][k].view(torch.int8), out[False][k].view(torch.int8)), k
    # the storing launch's dW is the batch's gradient; the accumulating one adds exactly that to the prefill
    ref = R.head_ce64(h, W, bias, dl_used=out[True]["dlogits"][:, :C], drop_scale=2.0, relu=True)
    chain = KC.head_chain(K, B)
    KC.check(out[False]["dW"], *ref["dW"], chain=chain["dW"], exact=False, family="head_dW")
    want, mag = ref["dW"][0] + dW0.double(), ref["dW"][1] + dW0.double().abs()
    KC.check(out[True]["dW"], want, mag, chain=chain["dW"] + 1, exact=False, family="head_dW")
    assert torch.equal(out[True]["dW"], dW0 + out[False]["dW"])       # one fp32 add onto the stored value


# ------------------------------------------------------------------------------------- replay
def _record_groups(configs):
    """Launch signatures of training steps, each config's steps given as (batch size, update)."""
    from distributed_vgg_f_b200 import ops
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine

    real = ops.require()
    rec = _Recorder(real)
    for spec, batch, steps, env, kw in configs:
        saved = {k: os.environ.get(k) for k in env}
        os.environ.update(env)
        try:
            eng = NativeEngine(spec, device=torch.device(DEV), batch=batch, seed=0, distributed=False, **kw)
            ops._C = rec
            try:
                for b, update in steps:
                    eng.train_step(_batch(spec, eng, b, False), update=update)
                eng.sync()
            finally:
                ops._C = real
        finally:
            for k, v in saved.items():
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = v
        del eng
        torch.cuda.empty_cache()
    return real, list(rec.sigs)


def test_replay_the_new_launches_of_an_accumulating_step(capsys):
    """Every launch signature an accumulating group makes that a K = 1 step does not (FC wgrad with the
    red.add epilogue, the optimizers' 1/k' gradient scale, ...), replayed on guarded operands.  head_ce's
    accumulate mode is covered by test_head_ce_accumulate_mode."""
    from distributed_vgg_f_b200.models.vggf import vggf_spec

    base = [(vggf_spec(3), 64, ((64, True), (64, True)), {}, {}),
            (vggf_spec(3), 16, ((16, True), (16, True)), {"B200_FUSED_HEAD": "0"}, {"optimizer": "sgd"})]
    accum = [(vggf_spec(3), 64, ((64, False), (64, True)), {}, {}),
             (vggf_spec(3), 64, ((64, False), (64, False), (37, True)), {}, {}),      # k' = 3, ragged last batch
             (vggf_spec(3), 16, ((16, False), (16, True)), {"B200_FUSED_HEAD": "0"}, {"optimizer": "sgd"})]
    _, old = _record_groups(base)
    C, sigs = _record_groups(accum)
    head_acc = [s for s in sigs if s[0] == "head_ce" and len(s) == 17]
    assert head_acc and all(s[-1] is True for s in head_acc)
    old = set(old)
    new = [s for s in sigs if s not in old and s not in head_acc]
    kinds = {s[0] for s in new}
    assert {"gemm", "adam", "sgd"} <= kinds, kinds
    codes = {s[10] for s in new if s[0] == "gemm"}
    assert C.EPI_F32_ATOMIC in codes                     # FC wgrad of a later micro-batch
    scales = {round(s[13], 6) for s in new if s[0] == "adam"}
    assert {0.5, round(1 / 3, 6)} <= scales, scales
    g = torch.Generator(device=DEV).manual_seed(1)
    done = replay_all(C, new, g, KC.sm_count())
    with capsys.disabled():
        print("\n[replay accum] %d new launch signatures replayed: %s" % (len(new), ", ".join(
            "%s=%d" % kv for kv in sorted(done.items()))))


# ------------------------------------------------------------------------ engine equivalence
def _engines(classes, optimizer="adam", fuse_pool=True, lr=1e-3):
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine
    from distributed_vgg_f_b200.models.vggf import build_oracle, vggf_mini_spec

    if fuse_pool:
        os.environ.pop("B200_FUSE_POOL", None)
    else:
        os.environ["B200_FUSE_POOL"] = "0"
    try:
        spec = vggf_mini_spec(classes)
        init = build_oracle(spec, seed=0).state_dict()
        kw = dict(device=torch.device(DEV), lr=lr, seed=0, input_hw=64, init_state=init, optimizer=optimizer,
                  distributed=False)
        small, big = NativeEngine(spec, batch=4, **kw), NativeEngine(spec, batch=16, **kw)
    finally:
        os.environ.pop("B200_FUSE_POOL", None)
    for e in (small, big):
        e.train_dropout = False
    return spec, small, big


def _data(n, classes, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, 3, 64, 64, generator=g).to(torch.bfloat16).float()
    return x, torch.randint(0, classes, (n,), generator=g)


def _rel(a, b):
    return float((a - b).norm() / (b.norm() + 1e-30))


@pytest.mark.parametrize("classes,fuse_pool", [(3, True), (10, True), (3, False)])
def test_four_micro_batches_equal_one_batch_on_the_arena(classes, fuse_pool, capsys):
    """K = 4 x b = 4 against K = 1 x b = 16 with updates off: the arena holds the sum of the four micro-batch
    means = 4 x the big batch's mean gradient.  Fused head (3 classes), unfused head (10), unfused pool."""
    spec, small, big = _engines(classes, fuse_pool=fuse_pool)
    assert small.fused_head == (classes <= 8)
    assert fuse_pool or not any(m is not None for m in small.pool_masks)
    for e in (small, big):
        e.apply_updates = False
    x, y = _data(16, classes, seed=11)
    for i in range(4):
        small.train_step((x[4 * i:4 * i + 4], y[4 * i:4 * i + 4]), update=i == 3)
    big.train_step((x, y))
    small.sync()
    assert small.step_count == 1 and small.micro_count == 4 and small._accum == 0
    worst = {}
    for name in spec.param_names:
        a, r = small._view(small.g32, name), 4 * big._view(big.g32, name)
        worst[name] = _rel(a, r)
    with capsys.disabled():
        print("\n[accum arena rel L2, %d classes, fused pool %s] max %.2e (%s)" % (
            classes, fuse_pool, max(worst.values()), max(worst, key=worst.get)))
    # only fp32 summation orders differ (1/4 and 1/16 scale the bf16 dlogits exactly); a micro-batch
    # stored instead of added would be off by ~75 %
    bad = {k: v for k, v in worst.items() if v > 1e-3}
    assert not bad, bad
    assert _rel(small.g32, 4 * big.g32) < 1e-4


@pytest.mark.parametrize("optimizer", ["adam", "sgd"])
def test_accumulated_updates_match_big_batch_updates(optimizer):
    """Three updates of K = 4 x b = 4 against three steps at b = 16: the same weights.  Adam runs with
    eps = 1 so that its update is smooth in g (see test_multigpu.py::_zero1_worker)."""
    spec, small, big = _engines(3, optimizer=optimizer, lr=5e-2 if optimizer == "adam" else 1e-2)
    if optimizer == "adam":
        small.eps = big.eps = 1.0
    p0 = big.p32.clone()
    for u in range(3):
        x, y = _data(16, 3, seed=20 + u)
        for i in range(4):
            small.train_step((x[4 * i:4 * i + 4], y[4 * i:4 * i + 4]), update=i == 3)
        big.train_step((x, y))
    small.sync()
    assert (small.step_count, small.micro_count, big.step_count) == (3, 12, 3)
    moved = _rel(big.p32, p0)
    assert moved > 1e-4, "the optimizer did not move the weights (%g)" % moved
    r = _rel(small.p32 - p0, big.p32 - p0)
    assert r < 1e-2, r
    assert torch.equal(small.w16, small.p32.to(torch.bfloat16))
    # the ranges the optimizer re-zeroes are clean for the next group
    assert torch.count_nonzero(small._view(small.g32, "features.2.weight")) == 0


def test_dropout_masks_differ_between_micro_batches():
    spec, small, _ = _engines(3)
    small.train_dropout = True
    assert spec.fcs[0].dropout > 0
    x, y = _data(4, 3, seed=5)
    masks = []
    for update in (False, False, True):              # no update in between: only the dropout draw differs
        small.train_step((x, y), update=update)
        small.sync()
        masks.append(small.fc_y[0][:4] == 0)
    assert not torch.equal(masks[0], masks[1]) and not torch.equal(masks[1], masks[2])
    assert (small.micro_count, small.step_count) == (3, 1)


def test_counters_survive_export_and_pending_groups_refuse_export():
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine

    spec, small, _ = _engines(3, optimizer="sgd")
    x, y = _data(4, 3, seed=6)
    small.train_step((x, y), update=False)
    with pytest.raises(RuntimeError, match="await an update"):
        small.export_state()
    small.train_step((x, y), update=True)
    small.train_step((x, y), update=True)
    small.sync()
    st, params = small.export_optimizer_state(), small.export_state()
    assert (st["step"], st["micro_step"]) == (2, 3)
    fresh = NativeEngine(spec, device=torch.device(DEV), batch=4, seed=0, input_hw=64, init_state=params,
                         optimizer="sgd", distributed=False)
    fresh.import_optimizer_state(st)
    assert (fresh.step_count, fresh.micro_count) == (2, 3)
    assert torch.equal(fresh.m32, small.m32) and torch.equal(fresh.p32, small.p32)


# --------------------------------------------------------------------------------- >= 2 GPUs
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _entry(rank, world, port, fn, args):
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        fn(rank, world, *args)
    finally:
        dist.barrier()
        dist.destroy_process_group()


def _dp_accum_worker(rank, world, algo, zero1, env):
    import torch.distributed as dist

    from distributed_vgg_f_b200.engine.native_engine import NativeEngine
    from distributed_vgg_f_b200.models.vggf import build_oracle, vggf_mini_spec

    os.environ.update(env)
    dev = torch.device("cuda", rank)
    spec = vggf_mini_spec(3)
    init = build_oracle(spec, seed=0).state_dict()
    eng = NativeEngine(spec, device=dev, batch=4, lr=1e-3, seed=0, input_hw=64, init_state=init, allreduce=algo,
                       bucket_mb=0.25, zero1=zero1)
    single = NativeEngine(spec, device=dev, batch=16, lr=1e-3, seed=0, input_hw=64, init_state=init,
                          distributed=False)
    if env.get("B200_FORCE_HIERARCHICAL") == "1":
        assert eng.comm_mode == "hierarchical"
    if algo == "nccl":
        assert eng.use_nccl
    for e in (eng, single):
        e.train_dropout = False
        e.apply_updates = False
    x, y = _data(16, 3, seed=9)
    # one update = 2 ranks x 2 micro-batches x 4 images: rank r's micro-batch j is images [8j + 4r, 8j + 4r + 4)
    mine = [(x[8 * j + 4 * rank:8 * j + 4 * rank + 4], y[8 * j + 4 * rank:8 * j + 4 * rank + 4]) for j in range(2)]
    for j, mb in enumerate(mine):
        eng.train_step(mb, update=j == 1)
    single.train_step((x, y))
    eng.sync()
    a, r = eng.g32, single.g32                   # reduced and scaled by 1 / (world k') = the big batch's mean
    assert _rel(a, r) < 2e-2, _rel(a, r)
    eng.apply_updates = True
    eng.g32.zero_()
    for j, mb in enumerate(mine):
        eng.train_step(mb, update=j == 1)
    eng.sync()
    if zero1:
        assert eng._zero1_buckets, "no bucket took the fused ZeRO-1 path"
    w = eng.w16.clone()
    dist.broadcast(w, src=0)
    assert torch.equal(w, eng.w16), "replicas diverged after an accumulated update (bf16 weights)"
    eng.prepare_export()
    p = eng.p32.clone()
    dist.broadcast(p, src=0)
    assert torch.equal(p, eng.p32), "replicas diverged after an accumulated update (fp32 master)"


@pytest.mark.multigpu
@pytest.mark.parametrize("algo,zero1,env", [("auto", False, {}), ("twoshot", False, {}), ("nccl", False, {}),
                                            ("twoshot", True, {}), ("auto", False, {"B200_FORCE_HIERARCHICAL": "1"})])
def test_two_ranks_accumulate_like_one_big_batch(algo, zero1, env):
    import torch.multiprocessing as mp

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    mp.spawn(_entry, args=(2, _free_port(), _dp_accum_worker, (algo, zero1, env)), nprocs=2, join=True)
