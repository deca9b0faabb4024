"""--freeze-layers across GPUs (>= 2 devices of one node; skipped otherwise): data-parallel equivalence with
features frozen against one process at the world-fold batch, with every rank starting from different weights
(the constructor broadcast covers the frozen range, which lies outside the shorter wire), and the fused ZeRO-1
step with classifier.0 frozen against replicated Adam."""
import pytest
import torch

import test_multigpu as TM

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]


def _dp_worker(rank, world, n):
    import torch.distributed as dist

    from distributed_vgg_f_b200.engine.native_engine import NativeEngine
    from distributed_vgg_f_b200.models.vggf import build_oracle, vggf_mini_spec

    dev = torch.device("cuda", rank)
    spec = vggf_mini_spec(3)
    init = build_oracle(spec, seed=rank).state_dict()          # different on every rank: the broadcast fixes it
    eng = NativeEngine(spec, device=dev, batch=4, lr=1e-3, seed=0, input_hw=64, init_state=init, bucket_mb=0.25,
                       freeze_layers=n)
    single = NativeEngine(spec, device=dev, batch=4 * world, lr=1e-3, seed=0, input_hw=64,
                          init_state=build_oracle(spec, seed=0).state_dict(), distributed=False, freeze_layers=n)
    assert eng.arena is not None and eng.arena.wire.numel() == eng.n_grad < eng.p32.numel()
    assert torch.equal(eng.p32, single.p32), "rank-0 weights (frozen range included) were not broadcast"
    start = eng.p32.clone()
    for e in (eng, single):
        e.train_dropout = False
        e.apply_updates = False
    g = torch.Generator().manual_seed(7)
    x = torch.randn(4 * world, 3, 64, 64, generator=g).to(torch.bfloat16).float()
    y = torch.randint(0, 3, (4 * world,), generator=g)
    eng.train_step((x[4 * rank:4 * rank + 4], y[4 * rank:4 * rank + 4]))
    single.train_step((x, y))
    eng.sync()
    single.sync()
    a, r = eng.g32, single.g32
    cos = float(torch.dot(a, r) / (a.norm() * r.norm()))
    assert cos > 0.995, cos          # bf16 wire + a different batch split of the bf16 activations
    eng.apply_updates = True
    eng.g32.zero_()
    for k in range(3):
        eng.train_step((x[4 * rank:4 * rank + 4], y[4 * rank:4 * rank + 4]), ema=False)
    eng.sync()
    for arena in (eng.w16, eng.p32):
        ref = arena.clone()
        dist.broadcast(ref, src=0)
        assert torch.equal(ref, arena), "replicas diverged"
    assert torch.equal(eng.p32[eng.n_grad:], start[eng.n_grad:]), "a frozen weight moved"
    assert not torch.equal(eng.p32[:eng.n_grad], start[:eng.n_grad]), "nothing trained"


@pytest.mark.parametrize("n", [13, 16])
def test_data_parallel_equivalence_with_frozen_layers(n):
    TM._run(_dp_worker, 2, n)


def _zero1_worker(rank, world):
    """As test_multigpu.py's ZeRO-1 worker (eps = 1 so that the comparison is smooth in the gradient), with
    classifier.0 frozen: the fused path keeps the buckets that hold one big FC weight alone, fewer of them."""
    import torch.distributed as dist

    from distributed_vgg_f_b200.engine.native_engine import NativeEngine
    from distributed_vgg_f_b200.models.vggf import build_oracle, vggf_mini_spec

    dev = torch.device("cuda", rank)
    spec = vggf_mini_spec(3)
    n = len(spec.convs) + 1                                     # features and classifier.0 frozen
    kw = dict(zero1=False, device=dev, batch=4, lr=5e-2, seed=0, input_hw=64, init_state=build_oracle(spec, seed=0)
              .state_dict(), allreduce="twoshot", bucket_mb=0.25, freeze_layers=n)
    ref = NativeEngine(spec, **kw)
    z = NativeEngine(spec, **dict(kw, zero1=True))
    full = NativeEngine(spec, **dict(kw, zero1=True, freeze_layers=0))
    assert z.zero1 and z._bucket_prepacked.count(True) < full._bucket_prepacked.count(True)
    assert not any("classifier.0.weight" in bk.tensors for bk in z.plan.buckets)
    del full
    p0 = ref.p32.clone()
    for e in (ref, z):
        e.train_dropout = False
        e.eps = 1.0
    g = torch.Generator().manual_seed(7 + rank)
    for _ in range(3):
        x = torch.randn(4, 3, 64, 64, generator=g).to(torch.bfloat16).float()
        y = torch.randint(0, 3, (4,), generator=g)
        for e in (ref, z):
            e.train_step((x, y))
            e.sync()
            dist.barrier()
    assert z._zero1_buckets, "no bucket took the fused path"
    w = z.w16.clone()
    dist.broadcast(w, src=0)
    assert torch.equal(w, z.w16), "replicas diverged"
    z.prepare_export()
    T = z.n_grad
    assert torch.equal(z.p32[T:], p0[T:]) and torch.equal(ref.p32[T:], p0[T:]), "a frozen weight moved"

    def rel(a, b):
        return float((a - b).norm() / (b.norm() + 1e-30))

    assert rel(ref.p32, p0) > 1e-4, "the optimizer did not move the weights: vacuous test"
    for name, a, b in (("update", z.p32 - p0, ref.p32 - p0), ("exp_avg", z.m32, ref.m32), ("exp_avg_sq", z.v32, ref.v32)):
        for bi, bk in enumerate(z.plan.buckets):
            r = rel(a[bk.start:bk.end], b[bk.start:bk.end])
            assert r < 2e-2, "%s of bucket %d (zero1=%s) differs: rel %g" % (name, bi, bi in z._zero1_buckets, r)


def test_zero1_with_classifier0_frozen_matches_replicated_adam():
    TM._run(_zero1_worker, 2)
