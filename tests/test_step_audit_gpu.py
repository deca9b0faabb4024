"""Every launch of full-size training steps audited on the engine's own tensors (step_audit.py).

Each configuration runs real steps of ``NativeEngine`` at world size 1 with ``ops._C`` replaced by
the auditing proxy: every launch is checked against its float64 reference on the snapshots of its
own arguments, for overlapping arguments, and for the links to the launches that produced what it
reads.  The streams are serialised in enqueue order; cross-stream event waits are not checked.
"""
import os
import time

import pytest
import torch

import kernel_check as KC
import launch_replay as LR
import step_audit as SA

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _audit(spec, batch, steps, env=None, fused=True, class_weights=None, **kw):
    """steps: ("train", b, update) / ("eval", b, None).  Returns (engine, auditor)."""
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine

    env = env or {}
    saved = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        eng = NativeEngine(spec, device=torch.device(DEV), batch=batch, seed=0, distributed=False, **kw)
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    if class_weights is not None:
        eng.set_class_weights(torch.tensor(class_weights))
    with SA.audit_engine(eng) as aud:
        for n, (kind, b, update) in enumerate(steps):
            data = LR._batch(spec, eng, b, fused, seed=1000 + n)
            if kind == "train":
                eng.train_step(data, update=update)
            else:
                eng.eval_step(data)
        eng.sync()
    return eng, aud


def _report(capsys, what, aud, t0):
    with capsys.disabled():
        print("\n[audit] %s: %d launches (%s), %d links, %.1f s, max_memory_allocated %.1f GiB" % (
            what, sum(aud.counts.values()), ", ".join("%s=%d" % kv for kv in sorted(aud.counts.items())), aud.links,
            time.time() - t0, torch.cuda.max_memory_allocated() / 2 ** 30))
        print("[audit] worst err/bound: " + ", ".join("%s %.3g" % kv for kv in sorted(KC.worst_ratio.items())))


def _pooled(spec):
    return [i for i, c in enumerate(spec.convs) if c.pool_after and i > 0]


def _run(capsys, what, *args, **kw):
    KC.worst_ratio.clear()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    eng, aud = _audit(*args, **kw)
    _report(capsys, what, aud, t0)
    return eng, aud


def test_audit_vggf_fused_pool_fused_head(capsys):
    """The default step at 224^2, batch 64: uint8 images through augment, fused pool and head, Adam;
    two steps (links across the update), an evaluation step and a ragged training batch of 37."""
    from distributed_vgg_f_b200.models.vggf import vggf_spec

    spec = vggf_spec(3)
    steps = [("train", 64, True), ("train", 64, True), ("eval", 64, None), ("train", 37, True)]
    eng, aud = _run(capsys, "vggf 224 b64 fused", spec, 64, steps)
    assert all(eng.pool_masks[i] is not None for i in _pooled(spec)), "a pooled layer took the unfused route"
    assert eng.fused_head
    assert aud.counts["conv_fprop_pool"] == len(_pooled(spec)) * len(steps)
    assert "maxpool_fwd" not in aud.counts and "cross_entropy" not in aud.counts
    assert aud.counts["augment"] == len(steps)


def test_audit_vgg16_gemm_head(capsys):
    """VGG-16 / 1000 classes, batch 32: the head as GEMM + fc_bias_act + cross_entropy, float images."""
    from distributed_vgg_f_b200.models.vggf import vgg16_spec

    eng, aud = _run(capsys, "vgg16 224 b32", vgg16_spec(1000), 32, [("train", 32, True), ("eval", 32, None)],
                    fused=False)
    assert not eng.fused_head and aud.counts["cross_entropy"] == 2 and "head_ce" not in aud.counts


def test_audit_vggf_separate_pool(capsys):
    """B200_FUSE_POOL=0: conv_fprop + maxpool_fwd forward, maxpool_relu_bwd backward."""
    from distributed_vgg_f_b200.models.vggf import vggf_spec

    spec = vggf_spec(3)
    eng, aud = _run(capsys, "vggf 224 b64 separate pool", spec, 64, [("train", 64, True), ("train", 64, True)],
                    env={"B200_FUSE_POOL": "0"})
    assert "conv_fprop_pool" not in aud.counts
    assert aud.counts["maxpool_relu_bwd"] == 2 * (len(_pooled(spec)) + spec.convs[0].pool_after)


def test_audit_accumulation_group(capsys):
    """Two micro-batches per update: FC wgrad and head_ce store, then add; the optimizer scales by 1/2."""
    from distributed_vgg_f_b200.models.vggf import vggf_spec

    eng, aud = _run(capsys, "vggf 224 b64 accumulate 2", vggf_spec(3), 64,
                    [("train", 64, False), ("train", 64, True), ("train", 64, True)])
    assert aud.counts["head_ce"] == 3


def test_audit_sgd_class_weights_small_input(capsys):
    """SGD with weight decay and class weights at 128^2 (a 4 x 4 feature map: adaptive average pool)."""
    from distributed_vgg_f_b200.models.vggf import vggf_spec

    eng, aud = _run(capsys, "vggf 128 b8 sgd", vggf_spec(3), 8, [("train", 8, True), ("train", 8, True),
                                                               ("eval", 8, None)],
                    env={"B200_FUSE_POOL": "0"}, fused=False, class_weights=[0.5, 1.0, 2.0], input_hw=128,
                    optimizer="sgd", weight_decay=1e-4)
    assert aud.counts["sgd"] > 0 and aud.counts["avgpool_fwd"] == 3 and aud.counts["avgpool_bwd"] == 2
