"""NativeEngine (sm_90a kernels end to end) against the torch oracle on the same weights."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _mk(batch=4, hw=64, classes=3, seed=0, fuse_pool=None, **kw):
    import os

    from distributed_vgg_f_b200.engine.native_engine import NativeEngine
    from distributed_vgg_f_b200.models.vggf import build_oracle, vggf_mini_spec

    if fuse_pool is not None:            # read once, when the engine lays out its buffers
        os.environ["B200_FUSE_POOL"] = "1" if fuse_pool else "0"
    else:
        os.environ.pop("B200_FUSE_POOL", None)

    spec = vggf_mini_spec(classes)
    oracle = build_oracle(spec, seed=seed)
    # the engine computes with bf16 weights: give the oracle the same rounded values
    with torch.no_grad():
        for p in oracle.parameters():
            if p.dim() > 1:
                p.copy_(p.to(torch.bfloat16).float())
    eng = NativeEngine(spec, device=torch.device(DEV), batch=batch, lr=1e-3, seed=seed, input_hw=hw,
                       init_state=oracle.state_dict(), **kw)
    return spec, oracle.to(DEV), eng


def _rel(a, b):
    return float((a.float() - b.float()).abs().max() / (b.float().abs().max() + 1e-12))


def test_forward_matches_oracle():
    spec, oracle, eng = _mk()
    torch.manual_seed(1)
    x = torch.randn(4, 3, 64, 64, device=DEV).to(torch.bfloat16).float()
    y = torch.randint(0, 3, (4,), device=DEV)
    oracle.eval()
    with torch.no_grad():
        ref = oracle(x)
    got = eng.forward_logits((x, y))
    assert _rel(got, ref) < 3e-2


def test_ragged_batch_and_eval_step():
    spec, oracle, eng = _mk(batch=8)
    from distributed_vgg_f_b200.utils.metrics import DeviceMeter

    torch.manual_seed(2)
    x = torch.randn(5, 3, 64, 64, device=DEV).to(torch.bfloat16).float()
    y = torch.randint(0, 3, (5,), device=DEV)
    meter = DeviceMeter(DEV)
    eng.set_meter(meter)
    eng.eval_step((x, y))
    avg, acc = meter.snapshot()
    oracle.eval()
    with torch.no_grad():
        ref = oracle(x)
    assert acc.count == 5 and abs(avg.average - float(F.cross_entropy(ref, y))) < 3e-2


def _l2(a, b):
    return float((a.float() - b.float()).norm() / (b.float().norm() + 1e-20))


def test_backward_matches_reference_on_same_forward(capsys):
    """Backward pass vs a torch fp32 chain with the engine's bf16 rounding points
    (ops.ref.emulated_step), gated on the engine's own forward activations: ReLU / pool routing is
    then identical on both sides and only accumulation order differs."""
    _backward_on_same_forward(capsys, classes=3, batch=4, b=4)


@pytest.mark.parametrize("classes,batch,b", [(10, 4, 4),     # > 8 classes: unfused head (GEMM + epilogue + CE)
                                             (3, 4, 3)])     # ragged training batch
def test_backward_matches_reference_unfused_head_and_ragged_batch(capsys, classes, batch, b):
    """The same check on the paths the default mini model does not take."""
    _backward_on_same_forward(capsys, classes=classes, batch=batch, b=b)


def _backward_on_same_forward(capsys, classes, batch, b):
    from distributed_vgg_f_b200.models import layout as L
    from distributed_vgg_f_b200.ops import ref as R

    # the un-pooled activations this check gates on only exist when the pool is NOT fused into the conv
    # epilogue (the default fuses it: test_fused_pool_step_matches_unfused_step covers that path)
    spec, oracle, eng = _mk(batch=batch, classes=classes, fuse_pool=False)
    assert eng.fused_head == (classes <= 8)
    eng.train_dropout = False
    eng.apply_updates = False
    torch.manual_seed(3)
    x = torch.randn(b, 3, 64, 64, device=DEV).to(torch.bfloat16).float()
    y = torch.randint(0, classes, (b,), device=DEV)
    got_loss = float(eng.train_step((x, y)))
    eng.sync()
    override = {
        "acts": [a[:b].permute(0, 3, 1, 2).float() for a in eng.acts],
        "feat": eng.feat.permute(0, 3, 1, 2).float(),
        "fc_y": [t[:b].float() if t is not None else None for t in eng.fc_y],
        "logits": eng.logits[:b].clone(),
    }
    state = {k: v.detach() for k, v in oracle.state_dict().items()}
    logits, loss, grads = R.emulated_step(spec, state, x, y, override=override)
    assert abs(got_loss - float(loss)) < 1e-4
    worst = {}
    for name in spec.param_names:
        ref = L.to_native(spec, name, grads[name])
        worst[name] = max(_rel(eng._view(eng.g32, name), ref), _l2(eng._view(eng.g32, name), ref))
    with capsys.disabled():
        print("\n[grad err, same forward] " + ", ".join("%s=%.1e" % kv for kv in worst.items()))
    bad = {k: v for k, v in worst.items() if v > 2e-2}
    assert not bad, bad


def test_fused_pool_step_matches_unfused_step():
    """The default step (2x2 max-pool inside the conv epilogue, argmax bit masks, unpool backward) against the
    same step with separate pool kernels: same loss, same logits, same gradients (only the order of the
    fp32 split-K red.adds may differ)."""
    from distributed_vgg_f_b200.models import layout as L

    torch.manual_seed(5)
    x = torch.randn(4, 3, 64, 64, device=DEV).to(torch.bfloat16).float()
    y = torch.randint(0, 3, (4,), device=DEV)
    out = {}
    for fused in (False, True):
        spec, _, eng = _mk(fuse_pool=fused)
        if fused and not any(m is not None for m in eng.pool_masks):
            pytest.skip("no pooled layer of the mini model has a fusable tile shape")
        assert fused or not any(m is not None for m in eng.pool_masks)
        eng.train_dropout = False
        eng.apply_updates = False
        loss = float(eng.train_step((x, y)))
        eng.sync()
        out[fused] = (loss, eng.logits[:4].clone(), eng.g32.clone())
    assert abs(out[True][0] - out[False][0]) < 1e-5
    assert torch.equal(out[True][1], out[False][1])
    a, r = out[True][2], out[False][2]
    assert float((a - r).norm() / r.norm()) < 1e-3 and float((a - r).abs().max() / r.abs().max()) < 1e-2


def test_forward_and_gradients_close_to_fp32_autograd(capsys):
    """End-to-end sanity against plain fp32 autograd (no emulation): forward tight; gradients in
    L2 / cosine terms (mask flips at near-zero activations make max-norm meaningless here)."""
    from distributed_vgg_f_b200.models import layout as L

    spec, oracle, eng = _mk()
    eng.train_dropout = False
    eng.apply_updates = False
    torch.manual_seed(3)
    x = torch.randn(4, 3, 64, 64, device=DEV).to(torch.bfloat16).float()
    y = torch.randint(0, 3, (4,), device=DEV)
    oracle.eval()
    loss = F.cross_entropy(oracle(x), y)
    loss.backward()
    got_loss = float(eng.train_step((x, y)))
    assert abs(got_loss - float(loss.detach())) < 3e-2
    cos = {}
    for name, p in oracle.named_parameters():
        a, r = eng._view(eng.g32, name).flatten().float(), L.to_native(spec, name, p.grad).flatten().float()
        cos[name] = float(torch.dot(a, r) / (a.norm() * r.norm() + 1e-30))
    with capsys.disabled():
        print("\n[grad cosine vs fp32 autograd] " + ", ".join("%s=%.4f" % kv for kv in cos.items()))
    assert min(cos.values()) > 0.9, cos      # bf16 storage + batch of 4: drift, not a defect


def test_training_reduces_loss_and_updates_shadow():
    spec, oracle, eng = _mk(batch=8)
    from distributed_vgg_f_b200.data import transforms as T
    from distributed_vgg_f_b200.data.loader import FusedBatch
    from distributed_vgg_f_b200.data.synthetic import synthetic_uint8_batch

    imgs, labels = synthetic_uint8_batch(8, 128, 3, seed=0)
    batch = FusedBatch(torch.from_numpy(imgs).pin_memory(), T.val_params(8, 128, 128).pin_memory(),
                       torch.from_numpy(labels).pin_memory(), (73, 73), None)   # 64x64 centre crop of a 73x73 resize
    eng.train_dropout = False
    losses = [float(eng.train_step(batch)) for _ in range(40)]
    assert all(math.isfinite(v) for v in losses)
    assert min(losses[-10:]) < 0.5 * losses[0], losses[::4]      # Adam at lr 1e-3 on 8 images is bouncy
    assert torch.equal(eng.w16.float(), eng.p32.to(torch.bfloat16).float())     # shadow follows master
    assert torch.count_nonzero(eng._view(eng.g32, 'features.2.weight')) == 0    # red.add targets are re-zeroed


def test_fused_input_path_equals_float_path():
    spec, oracle, eng = _mk()
    from distributed_vgg_f_b200.data import transforms as T
    from distributed_vgg_f_b200.data.loader import FusedBatch
    from distributed_vgg_f_b200.data.synthetic import synthetic_uint8_batch

    imgs, labels = synthetic_uint8_batch(4, 128, 3, seed=5)
    src = torch.from_numpy(imgs)
    params = T.sample_train_params(4, 128, 128, torch.Generator().manual_seed(1))
    batch = FusedBatch(src, params, torch.from_numpy(labels), (80, 80), None)
    a = eng.forward_logits(batch)
    x = T.augment_reference(src.to(DEV), params, (80, 80), out_hw=64)
    b = eng.forward_logits((x, torch.from_numpy(labels).to(DEV)))
    assert _rel(a, b) < 2e-2


def test_checkpoint_roundtrip_with_oracle(tmp_path):
    from distributed_vgg_f_b200.models.vggf import build_oracle
    from distributed_vgg_f_b200.utils import checkpoint as ck

    spec, oracle, eng = _mk()
    path = str(tmp_path / "e.pt")
    ck.save_checkpoint(path, eng, None, epoch=1)
    payload = torch.load(path, weights_only=False)
    assert list(payload["model"].keys())[0] == "module.features.0.weight"
    fresh = build_oracle(spec, seed=123)
    fresh.load_state_dict(ck.strip_module_prefix(payload["model"]))          # reference-style consumer
    for (k, a), (_, b) in zip(fresh.state_dict().items(), oracle.state_dict().items()):
        assert torch.allclose(a, b.cpu(), atol=0, rtol=0), k
    spec2, _, eng2 = _mk(seed=7)
    assert ck.load_checkpoint(path, eng2, None) == 1
    assert torch.equal(eng2.p32, eng.p32)


def test_full_vggf_smoke():
    import __graft_entry__ as g
    g.smoke()


def test_cli_native_end_to_end(tmp_path, capsys):
    """The reference-compatible CLI on the native engine: banner, per-epoch report line, checkpoint,
    resume, sharded-eval flag parsing, class weights -- on a generated ImageFolder."""
    import re

    from distributed_vgg_f_b200 import cli
    from distributed_vgg_f_b200.data.synthetic import make_synthetic_imagefolder

    root = str(tmp_path / "data")
    make_synthetic_imagefolder(root, train_per_class=16, val_per_class=4, size=128, seed=3)
    ck = str(tmp_path / "ck.pt")
    base = ["-iu", "tcp://127.0.0.1:29999", "-rn", "0", "-ws", "1", "-rd", root, "-lr", "0.0005", "-mb", "8",
            "--model", "vggf-mini", "--save", ck, "--class-weights", "1.0,1.0,1.0", "--profile", "events"]
    assert cli.main(base + ["-ep", "2"]) == 0
    out = capsys.readouterr().out
    assert "[Info] number of classes: 3" in out and "[Info] Running instance 0 using NVIDIA" in out
    pat = re.compile(r"\[Info\] Epoch: (\d)/2, train loss: [\d.]+, train acc: [\d.]+%, test loss: [\d.]+, test acc: [\d.]+%\.")
    assert len(pat.findall(out)) == 2, out
    payload = torch.load(ck, weights_only=False)
    assert payload["epoch"] == 2 and payload["optimizer"]["name"] == "adam" and payload["optimizer"]["step"] == 12
    assert cli.main(base + ["-ep", "3", "--resume", ck]) == 0
    out = capsys.readouterr().out
    assert "resumed from" in out and "[Info] Epoch: 3/3," in out and "Epoch: 1/3" not in out


def test_pretrained_state_reaches_the_native_arenas(tmp_path):
    """--pretrained on the native path: a torchvision VGG-16 state dict lands in the engine's arenas
    (OHWI conv weights, NHWC-ordered FC-1 columns) and comes back out in torch layout unchanged, while
    the funnel keeps its fresh init (distributedVggf.py:46-57)."""
    import torchvision

    from distributed_vgg_f_b200.engine.native_engine import NativeEngine
    from distributed_vgg_f_b200.models.vggf import build_oracle, vggf_spec

    tv = torchvision.models.vgg16(weights=None).state_dict()
    spec = vggf_spec(3)
    eng = NativeEngine(spec, device=torch.device(DEV), batch=2, seed=4, pretrained_state=tv, distributed=False)
    out = eng.export_state()
    fresh = build_oracle(spec, seed=4).state_dict()
    for k, v in out.items():
        if k.startswith("classifier.6."):
            assert torch.equal(v, fresh[k]), k
        else:
            assert torch.equal(v, tv[k].float()), k
    # and the bf16 shadow the kernels read is the rounded master
    assert torch.equal(eng.w16, eng.p32.to(torch.bfloat16))
