"""Training and evaluation at input sizes other than 224 (--train-crop-size, --val-crop-size, FixRes) on the
native engine: floor-mode max-pool at odd maps, the convolutions at 11^2 and 25^2, whole steps at 128, 176 and
200 against the emulated reference, an evaluation size other than the training size, and the augment kernels at
the new (resize, crop) pairs."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import kernel_check as KC
from distributed_vgg_f_b200.ops import ref as R
from guarded import NAN, fmax, guarded

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _ops():
    from distributed_vgg_f_b200 import ops

    ops.require()
    return ops


def _rel(a, b):
    return float((a.float() - b.float()).abs().max() / (b.float().abs().max() + 1e-12))


def _l2(a, b):
    return float((a.float() - b.float()).norm() / (b.float().norm() + 1e-20))


# ------------------------------------------------------------------------------ floor-mode max-pool
ODD_POOLS = [(64, 11, 11, 512), (37, 25, 25, 512), (3, 13, 9, 64), (5, 7, 7, 128), (2, 8, 8, 64)]


@pytest.mark.parametrize("colsum", [False, True])
@pytest.mark.parametrize("N,H,W,C", ODD_POOLS)
def test_maxpool_floor_mode_on_guarded_operands(N, H, W, C, colsum):
    """Forward against float64 F.max_pool2d, ReLU backward against autograd (the dropped last row / column
    gets dz = 0, as torch's gradient), the column sum against the sum of dz; nothing outside the operands
    changes, y is never modified, and every element of dz is written."""
    ops = _ops()
    g = torch.Generator(device=DEV).manual_seed(N * 100 + H * 10 + W + C)
    # post-ReLU integers: frequent ties and zeros, exact in bf16 and in every sum
    vals = torch.relu(torch.randint(-2, 3, (N, H, W, C), device=DEV, generator=g)).to(torch.bfloat16)
    OH, OW = H // 2, W // 2
    y = guarded((N, H, W, C), (H * W * C, W * C, C, 1), torch.bfloat16, 0, fmax(torch.bfloat16), DEV, vals)
    p = guarded((N, OH, OW, C), (OH * OW * C, OW * C, C, 1), torch.bfloat16, 0, NAN, DEV)
    y.seal()
    p.seal()
    ops.maxpool2x2(y.t, out=p.t)
    torch.cuda.synchronize()
    y.check(what="maxpool_fwd y")
    p.check(written=[p.t], what="maxpool_fwd out")
    ref = F.max_pool2d(vals.double().permute(0, 3, 1, 2), 2, 2).permute(0, 2, 3, 1)
    assert torch.equal(p.t.double(), ref)

    dpv = torch.randint(-3, 4, (N, OH, OW, C), device=DEV, generator=g).to(torch.bfloat16)
    dp = guarded((N, OH, OW, C), (OH * OW * C, OW * C, C, 1), torch.bfloat16, 0, NAN, DEV, dpv)
    dz = guarded((N, H, W, C), (H * W * C, W * C, C, 1), torch.bfloat16, 0, NAN, DEV)
    cs = torch.zeros(C, device=DEV) if colsum else None
    for t in (y, dp, dz):
        t.seal()
    ops.maxpool2x2_relu_bwd(y.t, dp.t, out=dz.t, colsum=cs)
    torch.cuda.synchronize()
    y.check(what="maxpool_relu_bwd y")
    dp.check(what="maxpool_relu_bwd dp")
    dz.check(written=[dz.t], what="maxpool_relu_bwd dz")
    x = vals.double().permute(0, 3, 1, 2).requires_grad_(True)
    F.max_pool2d(x, 2, 2).backward(dpv.double().permute(0, 3, 1, 2))
    want = (x.grad * (x.detach() > 0)).permute(0, 2, 3, 1)
    got = dz.t.double()
    assert not bool(torch.isnan(got).any()), "an element of dz was not written"
    assert torch.equal(got, want)
    if H % 2:
        assert bool((got[:, H - 1] == 0).all())
    if W % 2:
        assert bool((got[:, :, W - 1] == 0).all())
    if colsum:
        assert torch.equal(cs.double(), want.reshape(-1, C).sum(0))


# ------------------------------------------------------------------------------ convolutions at odd maps
ODD_CONVS = [(64, 11, 11, 512, 512), (37, 11, 11, 512, 512), (64, 25, 25, 512, 512), (4, 25, 25, 64, 128),
             (3, 13, 9, 64, 64)]


def test_pixel_boxes_fill_the_tile_only_where_make_tile_does_not():
    """The 224-step shapes at batch 64 keep make_tile's power-of-two boxes (and so their kernels); 11^2 and 25^2
    get boxes that fill the 128-row tile.  (Wb, Hb, Nb, fill)"""
    C = _ops().require()
    for h, box in ((56, (8, 8, 2)), (28, (4, 4, 8)), (14, (2, 2, 32)), (88, (8, 8, 2)), (44, (4, 4, 8)),
                   (22, (2, 2, 32)), (100, (4, 4, 8)), (50, (2, 2, 32))):
        assert tuple(C.conv_pixel_box(64, h, h)) == box + (0,), h
    assert tuple(C.conv_pixel_box(64, 11, 11)) == (11, 11, 1, 1)
    assert tuple(C.conv_pixel_box(64, 25, 25)) == (25, 5, 1, 1)
    for h in (11, 25, 29):
        w, hb, nb, _ = C.conv_pixel_box(64, h, h)
        tiles = -(-h // w) * -(-h // hb) * -(-64 // nb)
        assert tiles <= 1.15 * -(-64 * h * h // 128), (h, tiles)      # within 15 % of ceil(64 h^2 / 128)


@pytest.mark.parametrize("N,H,W,Cin,Cout", ODD_CONVS)
def test_conv_at_odd_maps(N, H, W, Cin, Cout):
    """fprop, dgrad, masked dgrad with its column sum and wgrad at the map sizes of crops 176 and 200, against
    float64, with the outputs inside guarded buffers.  These shapes run the FILL kernels (boxes of any sides)."""
    ops = _ops()
    assert ops.require().conv_pixel_box(N, H, W)[3] == 1
    g = KC.generator(N * 7 + H + Cin * 3 + Cout, DEV)
    x = KC.operand((N, H, W, Cin), "gauss", 9 * Cin, g, DEV)
    w = KC.operand((Cout, 3, 3, Cin), "gauss", 9 * Cin, g, DEV)
    b = KC.bias(Cout, "gauss", g, DEV)
    y = guarded((N, H, W, Cout), (H * W * Cout, W * Cout, Cout, 1), torch.bfloat16, 0, NAN, DEV)
    y.seal()
    ops.require().conv_fprop(x, w, b, y.t, True, 0)
    torch.cuda.synchronize()
    y.check(written=[y.t], what="conv_fprop y")
    ref, mag = R.conv3x3_fprop64(x, w, b, relu=True)
    KC.check(y.t, ref, mag, chain=KC.conv_chain(Cin), exact=False, family="conv_fprop")

    dz = KC.operand((N, H, W, Cout), "gauss", 9 * Cout, g, DEV)
    dx = ops.conv3x3_dgrad(dz, w, Cin)
    ref, mag = R.conv3x3_dgrad64(dz, w)
    KC.check(dx, ref, mag, chain=KC.conv_chain(Cout), exact=False, family="conv_dgrad")
    mask_src = KC.operand((N, H, W, Cin), "gauss", 1, g, DEV)
    dxm = guarded((N, H, W, Cin), (H * W * Cin, W * Cin, Cin, 1), torch.bfloat16, 0, NAN, DEV)
    cs = torch.zeros(Cin, device=DEV)
    dxm.seal()
    ops.require().conv_dgrad(dz, w, mask_src, dxm.t, cs, 0)
    torch.cuda.synchronize()
    dxm.check(written=[dxm.t], what="conv_dgrad dx")
    ref, mag = R.conv3x3_dgrad64(dz, w, mask_src=mask_src)
    KC.check(dxm.t, ref, mag, chain=KC.conv_chain(Cout), exact=False, family="conv_dgrad", what="masked")
    stored = dxm.t.to(torch.float64).reshape(-1, Cin)
    KC.check(cs, stored.sum(0), stored.abs().sum(0), chain=KC.conv_colsum_chain(N * H * W, Cin, KC.sm_count()),
             exact=False, family="conv_colsum")

    dw = torch.zeros(Cout, 3, 3, Cin, device=DEV)
    ops.conv3x3_wgrad(dz, x, dw)
    ref, mag = R.conv3x3_wgrad64(dz, x)
    KC.check(dw, ref, mag, chain=KC.wgrad_chain(N, H, W, Cin, Cout, KC.sm_count()), exact=False, family="conv_wgrad")


# ------------------------------------------------------------------------------ whole steps
def _mk(spec, hw, batch, eval_hw=None, seed=0, fuse_pool=None, **kw):
    import os

    from distributed_vgg_f_b200.engine.native_engine import NativeEngine
    from distributed_vgg_f_b200.models.vggf import build_oracle

    saved = os.environ.get("B200_FUSE_POOL")
    if fuse_pool is not None:            # read once, when the engine lays out its buffers
        os.environ["B200_FUSE_POOL"] = "1" if fuse_pool else "0"
    else:
        os.environ.pop("B200_FUSE_POOL", None)
    oracle = build_oracle(spec, seed=seed)
    with torch.no_grad():                # the engine computes with bf16 weights: give the oracle the same values
        for p in oracle.parameters():
            if p.dim() > 1:
                p.copy_(p.to(torch.bfloat16).float())
    try:
        eng = NativeEngine(spec, device=torch.device(DEV), batch=batch, lr=1e-3, seed=seed, input_hw=hw,
                           eval_hw=eval_hw, init_state=oracle.state_dict(), distributed=False, **kw)
    finally:                             # the caller's setting, as it was
        if saved is None:
            os.environ.pop("B200_FUSE_POOL", None)
        else:
            os.environ["B200_FUSE_POOL"] = saved
    return oracle.to(DEV), eng


def _step_against_emulated(spec, hw, batch, capsys, what):
    """One step with separate pool kernels, gated on the engine's own forward (ops.ref.emulated_step), and the
    default step (pool fused wherever the tile shape allows) against it.  Both deterministic: the fp32 atomics of
    split-K and column sums would otherwise move ReLU / pool routing at near-ties between the two engines."""
    from distributed_vgg_f_b200.models import layout as L

    torch.manual_seed(hw)
    x = torch.randn(batch, 3, hw, hw, device=DEV).to(torch.bfloat16).float()
    y = torch.randint(0, spec.num_classes, (batch,), device=DEV)
    out = {}
    for fused in (False, True):
        oracle, eng = _mk(spec, hw, batch, fuse_pool=fused, deterministic=True)
        eng.train_dropout = False
        eng.apply_updates = False
        loss = float(eng.train_step((x, y)))
        eng.sync()
        out[fused] = (loss, eng.logits[:batch].clone(), eng.g32.clone())
        if fused:
            break
        override = {"acts": [a[:batch].permute(0, 3, 1, 2).float() for a in eng.acts],
                    "feat": eng.feat.permute(0, 3, 1, 2).float(),
                    "fc_y": [t[:batch].float() if t is not None else None for t in eng.fc_y],
                    "logits": eng.logits[:batch].clone()}
        state = {k: v.detach() for k, v in oracle.state_dict().items()}
        _, ref_loss, grads = R.emulated_step(spec, state, x, y, override=override)
        assert abs(loss - float(ref_loss)) < 1e-4
        worst = {}
        for name in spec.param_names:
            ref = L.to_native(spec, name, grads[name])
            worst[name] = max(_rel(eng._view(eng.g32, name), ref), _l2(eng._view(eng.g32, name), ref))
        with capsys.disabled():
            print("\n[%s grad err, same forward] max %.1e" % (what, max(worst.values())))
        bad = {k: v for k, v in worst.items() if v > 2e-2}
        assert not bad, bad
        del eng
    assert out[True][0] == out[False][0]
    assert torch.equal(out[True][1], out[False][1])
    a, r = out[True][2], out[False][2]
    assert _l2(a, r) < 1e-3 and _rel(a, r) < 1e-2


@pytest.mark.parametrize("hw", [176, 200, 128, 64, 504])
def test_mini_step_matches_emulated(hw, capsys):
    """Crops 64 (a 2 x 2 map, upsampled to 7 x 7 by the adaptive pool) and 504 (odd 63^2 and 31^2 maps) are the
    two ends of what the engine takes."""
    from distributed_vgg_f_b200.models.vggf import vggf_mini_spec

    _step_against_emulated(vggf_mini_spec(3), hw, 4, capsys, "vggf-mini %d" % hw)


def test_vggf_b64_step_at_176_matches_emulated(capsys):
    from distributed_vgg_f_b200.models.vggf import vggf_spec

    _step_against_emulated(vggf_spec(3), 176, 64, capsys, "vggf b64 176")


def test_step_audit_vggf_176(capsys):
    """Every launch of a VGG-F step at 176 (odd 11 x 11 maps: separate pool kernels on the last block) and an
    evaluation pass, audited against float64 with their producer-to-consumer links."""
    import launch_replay as LR
    import step_audit as SA
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine
    from distributed_vgg_f_b200.models.vggf import vggf_spec

    spec = vggf_spec(3)
    eng = NativeEngine(spec, device=torch.device(DEV), batch=64, seed=0, distributed=False, input_hw=176)
    assert eng.pool_masks[-1] is None and eng.pool_masks[9] is not None
    with SA.audit_engine(eng) as aud:
        for n, kind in enumerate(("train", "eval")):
            data = LR._batch(spec, eng, 64, False, seed=2000 + n)
            if kind == "train":
                eng.train_step(data)
            else:
                eng.eval_step(data)
        eng.sync()
    assert aud.counts["maxpool_fwd"] == 2 and aud.counts["maxpool_relu_bwd"] == 1


def _uint8_batches(count, b, classes, src=144, seed=7):
    from distributed_vgg_f_b200.data import transforms as T
    from distributed_vgg_f_b200.data.loader import FusedBatch

    out = []
    for k in range(count):
        g = torch.Generator().manual_seed(seed + k)
        img = torch.randint(0, 256, (b, src, src, 3), dtype=torch.uint8, generator=g)
        out.append(FusedBatch(img, T.sample_train_params(b, src, src, g), torch.randint(0, classes, (b,), generator=g),
                              (src, src), None))
    return out


def test_fixres_eval_at_another_size_matches_oracle():
    """Trained at 176, evaluated at 224: the evaluation logits against the fp32 oracle on the same weights."""
    from distributed_vgg_f_b200.models.vggf import vggf_mini_spec

    spec = vggf_mini_spec(3)
    oracle, eng = _mk(spec, 176, 8, eval_hw=224)
    torch.manual_seed(4)
    x = torch.randn(8, 3, 224, 224, device=DEV).to(torch.bfloat16).float()
    y = torch.randint(0, 3, (8,), device=DEV)
    oracle.eval()
    with torch.no_grad():
        ref = oracle(x)
    got = eng.forward_logits((x, y))
    assert _rel(got, ref) < 3e-2
    with pytest.raises(AssertionError, match="input size"):
        eng.train_step((x, y))                    # training passes run at 176


def test_eval_between_steps_changes_no_training_state():
    """train -> eval at 224 -> train gives bit for bit the weights, moments and losses of train -> train
    (--deterministic: without it the fp32 split-K atomics alone make two runs differ in the last bits)."""
    from distributed_vgg_f_b200.models.vggf import vggf_mini_spec
    from distributed_vgg_f_b200.utils.metrics import DeviceMeter

    spec = vggf_mini_spec(3)
    batches = _uint8_batches(2, 8, 3, src=200)
    torch.manual_seed(5)
    xe = torch.randn(8, 3, 224, 224, device=DEV).to(torch.bfloat16).float()
    ye = torch.randint(0, 3, (8,), device=DEV)
    res = []
    for with_eval in (False, True):
        _, eng = _mk(spec, 176, 8, eval_hw=224, deterministic=True)
        meter = DeviceMeter(DEV)
        eng.set_meter(meter)
        losses = [eng.train_step(batches[0]).clone()]
        if with_eval:
            eng.set_meter(DeviceMeter(DEV))
            eng.eval_step((xe, ye))
            eng.set_meter(meter)
        losses.append(eng.train_step(batches[1]).clone())
        eng.sync()
        res.append((eng.p32.clone(), eng.m32.clone(), eng.v32.clone(), torch.cat(losses)))
    for a, b in zip(*res):
        assert torch.equal(a, b)


def test_deterministic_at_176_repeats():
    from distributed_vgg_f_b200.models.vggf import vggf_spec

    spec = vggf_spec(3)
    batches = _uint8_batches(3, 16, 3, src=200)
    out = []
    for _ in range(2):
        _, eng = _mk(spec, 176, 16, deterministic=True)
        losses = [eng.train_step(b).clone() for b in batches]
        eng.sync()
        out.append((eng.p32.clone(), eng.m32.clone(), torch.cat(losses)))
        del eng
    for a, b in zip(*out):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------ input kernels
@pytest.mark.parametrize("resize,crop", [(144, 128), (200, 176), (256, 224)])
def test_augment_uniform_at_new_sizes(resize, crop):
    ops = _ops()
    from distributed_vgg_f_b200.data import transforms as T
    from distributed_vgg_f_b200.data.synthetic import synthetic_uint8_batch

    imgs, _ = synthetic_uint8_batch(4, 128, seed=resize)
    src = torch.from_numpy(imgs).to(DEV)
    params = T.sample_train_params(4, 128, 128, torch.Generator().manual_seed(crop))
    params[0, 6], params[1, 6] = 0.0, 1.0
    ref = T.augment_reference(src, params, (resize, resize), out_hw=crop)
    out = torch.empty(4, crop, crop, 4, dtype=torch.bfloat16, device=DEV)
    ops.augment(src, params.to(DEV), out, (resize, resize), out_hw=crop, mode="nhwc", pad=4)
    diff = (out[..., :3].float().permute(0, 3, 1, 2) - ref).abs()
    assert float(diff.median()) < 5e-3
    assert float((diff > 0.05).float().mean()) < 2e-3


def _ragged(sizes, train, resize, seed=0):
    from distributed_vgg_f_b200.data import transforms as T
    from distributed_vgg_f_b200.data.loader import RaggedBatch

    rng = np.random.default_rng(seed)
    imgs = [rng.integers(0, 256, (h, w, 3)).astype(np.uint8) for h, w in sizes]
    data = torch.from_numpy(np.concatenate([a.reshape(-1) for a in imgs]))
    geom = T.ragged_geometry(sizes, train, resize)
    g = torch.Generator().manual_seed(seed)
    params = torch.cat([T.sample_train_params(1, h, w, g) if train else T.val_params(1, h, w) for h, w in sizes])
    return RaggedBatch(data, geom, params, torch.zeros(len(sizes), dtype=torch.int64), None)


@pytest.mark.parametrize("train,resize,crop", [(True, 144, 128), (True, 200, 176), (True, 256, 224),
                                               (False, 232, 224), (False, 288, 256)])
def test_augment_ragged_at_new_sizes(train, resize, crop):
    """Pillow-exact resize to the split's resize size, then the centre crop at the network's input size."""
    ops = _ops()
    from distributed_vgg_f_b200.data import transforms as T

    batch = _ragged([(97, 161), (300, 240), (128, 128), (500, 375)], train, resize, seed=crop)
    n = batch.geom.shape[0]
    out = torch.full((n, crop, crop, 4), NAN, dtype=torch.bfloat16, device=DEV)
    inter = torch.empty(ops.ragged_inter_bytes(batch.geom), dtype=torch.uint8, device=DEV)
    ops.augment_ragged(batch.data_u8.to(DEV), batch.geom.to(DEV), batch.params.to(DEV), inter, out,
                       batch.geom, batch.params, out_hw=crop)
    ref = T.ragged_reference(batch.data_u8, batch.geom, batch.params, out_hw=crop).permute(0, 2, 3, 1)
    differ = (out[..., :3].cpu() != ref.to(torch.bfloat16)).any(-1)
    assert float(differ.float().mean()) <= 1e-3
