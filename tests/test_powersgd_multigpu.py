"""--powersgd-rank across GPUs (>= 2 devices of one node; skipped otherwise): world 2 on vggf-mini under the default
arena all-reduce and under --allreduce nccl.  P and Q go through dist.all_reduce from the comm stream, between the
uncompressed buckets' reductions.  After the compressed updates both replicas hold the same bits, and every
compressed update agrees with torch's hook applied in float64 to both ranks' pre-exchange gradients (each from a
deterministic single-process twin on the replica's weights and the rank's batch)."""
import pytest
import torch

import test_multigpu as TM
import test_powersgd_gpu as TP

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]
S = 2


def _gathered(t: torch.Tensor, world: int) -> list:
    import torch.distributed as dist

    out = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(out, t.contiguous())
    return out


def _worker(rank, world, allreduce):
    import torch.distributed as dist

    from distributed_vgg_f_b200 import ops
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine
    from distributed_vgg_f_b200.models.vggf import build_oracle, vggf_mini_spec
    from distributed_vgg_f_b200.parallel import powersgd

    dev = torch.device("cuda", rank)
    spec = vggf_mini_spec(TP.CLASSES)
    init = build_oracle(spec, seed=1).state_dict()
    eng = NativeEngine(spec, device=dev, batch=TP.B, lr=1e-3, seed=5, input_hw=64, init_state=init, bucket_mb=0.25,
                       allreduce=allreduce, powersgd_rank=4, powersgd_start_iter=S)
    twin = NativeEngine(spec, device=dev, batch=TP.B, lr=1e-3, seed=5, input_hw=64, init_state=init, distributed=False,
                        deterministic=True)
    assert eng.world == world and eng.use_nccl == (allreduce == "nccl")
    for e in (eng, twin):
        e.train_dropout = False
    twin.apply_updates = False
    seen = {}
    real = ops.psgd_decompress

    def record(p, q, g, e, **kw):
        real(p, q, g, e, **kw)
        seen[g.data_ptr()] = g.clone()
    projected = {}
    real_project = ops.psgd_project

    def record_project(g, e, q, p, **kw):
        real_project(g, e, q, p, **kw)
        projected[g.data_ptr()] = e.clone()              # M = g + e, the matrix this rank compresses
    ops.psgd_decompress = record
    ops.psgd_project = record_project
    try:
        batches = TP.TD._batches(S + 2, TP.B, TP.CLASSES, hw=128, mix=False, seed=31 + 100 * rank)     # each rank its own data
        p0 = eng.p32.clone()
        for u in range(1, S + 3):
            if u > S:
                eng.sync()
                e_prev, q_prev = eng._psgd_e.clone(), eng._psgd_q.clone()
                twin.import_state(eng.export_state())
                twin.g32.zero_()
                twin.train_step(batches[u - 1])
                twin.sync()
            seen.clear()
            projected.clear()
            eng.train_step(batches[u - 1])
            eng.sync()
            if u <= S:
                assert not seen, "compressed before the start iteration"
                continue
            assert len(seen) == len(eng._psgd)
            first = powersgd.initial_q_torch(eng._psgd_rows, eng.seed) if u == S + 1 else None
            for name, (n, m, r, eo, po, qo) in eng._psgd.items():
                what = "%s update %d rank %d (%s)" % (name, u, rank, allreduce)
                # the engine's gradient comes from atomics, the twin's from ordered partial sums: fp32 rounding apart.
                # The hook is then applied to the engine's own M of every rank: an ill-conditioned power step would
                # turn that rounding into a different P
                M = projected[eng._view(eng.g32, name).data_ptr()].view(n, m)
                M_twin = twin._view(twin.g32, name).reshape(n, m) + e_prev[eo:eo + n * m].view(n, m)
                assert TP.rel(M, M_twin) < 1e-4, what
                Ms = _gathered(M, world)
                q0 = powersgd.q_to_native(spec, name, first[name]).to(dev) if first else q_prev[qo:qo + m * r].view(m, r)
                G = seen[eng._view(eng.g32, name).data_ptr()].view(n, m)
                P = eng._psgd_p[po:po + n * r].view(n, r).to(TP.F64)
                Q = eng._psgd_q[qo:qo + m * r].view(m, r).to(TP.F64)
                assert TP.rel(Q, sum(x.to(TP.F64).t() @ P for x in Ms)) < 1e-5, what          # Q keeps the sum
                assert TP.rel(G, P @ Q.t() / world, scale=M) < 1e-5, what
                e = eng._psgd_e[eo:eo + n * m].view(n, m)
                assert TP.rel(e, M.to(TP.F64) - G.to(TP.F64), scale=M) < 1e-6, what
                _, _, q64, G64 = TP.hook64(Ms, q0)            # every tensor: see test_powersgd_gpu.CLASSES
                assert TP.rel(G, G64, scale=M) < 1e-3, what
                assert TP.rel(Q / world, q64) < 1e-3, what
            # both replicas apply the same G (the same P and Q) and the same reduced uncompressed buckets
            for arena in (eng.p32, eng.w16):
                ref = arena.clone()
                dist.broadcast(ref, src=0)
                assert torch.equal(ref, arena), "replicas diverged at update %d (%s)" % (u, allreduce)
        assert not torch.equal(eng.p32, p0), "nothing trained"
    finally:
        ops.psgd_decompress = real
        ops.psgd_project = real_project


@pytest.mark.parametrize("allreduce", ["auto", "nccl"])
def test_world2_replicas_agree_and_match_the_hook(allreduce):
    TM._run(_worker, 2, allreduce)
