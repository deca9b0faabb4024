"""Knowledge distillation across GPUs (>= 2 devices of one node; skipped otherwise): every rank loads the same teacher
and runs it on its own shard; the gradient of two ranks against one process at the doubled batch, then updates that
leave the replicas bit-identical."""
import pytest
import torch

import test_multigpu as TM

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]


def _dp_worker(rank, world):
    import torch.distributed as dist

    from distributed_vgg_f_b200.engine.native_engine import NativeEngine, TeacherEngine
    from distributed_vgg_f_b200.models.vggf import build_oracle, vggf_mini_spec

    dev = torch.device("cuda", rank)
    spec = vggf_mini_spec(3)
    kw = dict(lr=1e-3, seed=0, input_hw=64)
    teacher_state = build_oracle(spec, seed=11).state_dict()
    eng = NativeEngine(spec, device=dev, batch=4, init_state=build_oracle(spec, seed=rank).state_dict(),
                       bucket_mb=0.25, **kw)
    single = NativeEngine(spec, device=dev, batch=4 * world, init_state=build_oracle(spec, seed=0).state_dict(),
                          distributed=False, **kw)
    eng.set_distillation(TeacherEngine(spec, dev, 4, teacher_state, input_hw=64), 0.5, 4.0)
    single.set_distillation(TeacherEngine(spec, dev, 4 * world, teacher_state, input_hw=64), 0.5, 4.0)
    for e in (eng, single):
        e.train_dropout = False
        e.apply_updates = False
    g = torch.Generator().manual_seed(7)
    x = torch.randn(4 * world, 3, 64, 64, generator=g).to(torch.bfloat16).float()
    y = torch.randint(0, 3, (4 * world,), generator=g)
    mine = (x[4 * rank:4 * rank + 4], y[4 * rank:4 * rank + 4])
    eng.train_step(mine)
    single.train_step((x, y))
    eng.sync()
    single.sync()
    a, r = eng.g32, single.g32
    cos = float(torch.dot(a, r) / (a.norm() * r.norm()))
    assert cos > 0.995, cos          # bf16 wire + a different batch split of the bf16 activations
    eng.apply_updates = single.apply_updates = True
    eng.g32.zero_()
    single.g32.zero_()
    eng.step_count = single.step_count = 0
    start = eng.p32.clone()
    for _ in range(3):
        eng.train_step(mine)
        single.train_step((x, y))
    eng.sync()
    single.sync()
    for arena in (eng.w16, eng.p32, eng.m32):
        ref = arena.clone()
        dist.broadcast(ref, src=0)
        assert torch.equal(ref, arena), "replicas diverged"
    moved = float((single.p32 - start).norm())
    assert moved > 0 and float((eng.p32 - single.p32).norm()) <= 0.05 * moved, "two ranks differ from one process"


def test_data_parallel_equivalence_and_identical_replicas():
    TM._run(_dp_worker, 2)
