"""The ragged input kernels (``augment_ragged``: Pillow-exact resampling of images of any size) on the
device: against the oracle, on guarded operands, through the engine and through one epoch of
``Trainer.fit``."""
import math
import os
import re

import numpy as np
import pytest
import torch

from distributed_vgg_f_b200 import ops
from distributed_vgg_f_b200.data import transforms as T
from distributed_vgg_f_b200.data.loader import RaggedBatch
from guarded import NAN, guarded

pytestmark = pytest.mark.gpu
DEV = "cuda"

# 1 x N strips up to 3000 x 4000, enlarged and shrunk, both aspect orientations
SIZES = [(1, 300), (300, 1), (37, 53), (128, 128), (256, 256), (480, 640), (1000, 750), (257, 1500),
         (1200, 97), (3000, 4000)]


def _images(sizes, seed=0):
    rng = np.random.default_rng(seed)
    out = []
    for h, w in sizes:
        yy, xx = np.mgrid[0:h, 0:w]
        base = (127 + 100 * np.sin(xx * 1.3) * np.cos(yy * 0.9))[..., None].repeat(3, 2)
        out.append(np.clip(base + rng.integers(-20, 20, (h, w, 3)), 0, 255).astype(np.uint8))
    return out


def _batch(sizes, train, seed=0, labels=None):
    imgs = _images(sizes, seed)
    data = torch.from_numpy(np.concatenate([a.reshape(-1) for a in imgs]))
    geom = T.ragged_geometry(sizes, train)
    g = torch.Generator().manual_seed(seed)
    params = torch.cat([T.sample_train_params(1, h, w, g) if train else T.val_params(1, h, w) for h, w in sizes])
    if train:                                # both flips and both rotation signs
        params[0::2, 6], params[1::2, 6] = 1.0, 0.0
    lab = torch.tensor(labels if labels is not None else [i % 3 for i in range(len(sizes))], dtype=torch.int64)
    return RaggedBatch(data, geom, params, lab, None)


def _run(batch, out_hw=224):
    n = batch.geom.shape[0]
    out = torch.full((n, out_hw, out_hw, 4), NAN, dtype=torch.bfloat16, device=DEV)
    inter = torch.empty(ops.ragged_inter_bytes(batch.geom), dtype=torch.uint8, device=DEV)
    ops.augment_ragged(batch.data_u8.to(DEV), batch.geom.to(DEV), batch.params.to(DEV), inter, out,
                       batch.geom, batch.params, out_hw=out_hw)
    return out


@pytest.mark.parametrize("train", [True, False])
def test_augment_ragged_matches_the_oracle(train):
    """The uint8 stages are exact integer arithmetic and the chain uses the oracle's float operations,
    so the output is bf16 of the oracle; only a nearest-rotation tie could differ."""
    batch = _batch(SIZES, train, seed=3)
    out = _run(batch)
    ref = T.ragged_reference(batch.data_u8, batch.geom, batch.params).permute(0, 2, 3, 1)
    got = out[..., :3].cpu()
    differ = (got != ref.to(torch.bfloat16)).any(-1)
    assert float(differ.float().mean()) <= 1e-3, [int(d.sum()) for d in differ]
    assert bool((out[..., 3].view(torch.int16) == 0).all())         # padding channel is +0


def test_augment_ragged_at_a_small_output_size():
    """The centre crop of a small engine input (input_hw 64) out of the 256-pixel resize."""
    batch = _batch([(90, 120), (700, 500)], True, seed=1)
    out = _run(batch, out_hw=64)
    ref = T.ragged_reference(batch.data_u8, batch.geom, batch.params, out_hw=64).permute(0, 2, 3, 1)
    assert float((out[..., :3].cpu() != ref.to(torch.bfloat16)).any(-1).float().mean()) <= 1e-3


def _guarded_launch(batch, out_hw=64):
    n = batch.geom.shape[0]
    nbytes = batch.data_u8.numel()
    need = ops.ragged_inter_bytes(batch.geom)
    src = guarded((nbytes,), (1,), torch.uint8, 0, 255, DEV, batch.data_u8)
    geom = guarded((n, 5), (5, 1), torch.int64, 0, 0, DEV, batch.geom)
    prm = guarded((n, 8), (8, 1), torch.float32, 0, 0.0, DEV, batch.params)
    inter = guarded((need,), (1,), torch.uint8, 0, 255, DEV)
    out = guarded((n, out_hw, out_hw, 4), (out_hw * out_hw * 4, out_hw * 4, 4, 1), torch.bfloat16, 0, NAN, DEV)
    for g in (src, geom, prm, inter, out):
        g.seal()
    ops.augment_ragged(src.t, geom.t, prm.t, inter.t, out.t, batch.geom, batch.params, out_hw=out_hw)
    torch.cuda.synchronize()
    for g, w, name in ((src, (), "src"), (geom, (), "geom"), (prm, (), "params"), (inter, (inter.t,), "inter"),
                       (out, (out.t,), "out")):
        g.check(w, name)
    return out.t


@pytest.mark.parametrize("train", [True, False])
def test_augment_ragged_stays_inside_its_operands(train):
    batch = _batch([(1, 200), (45, 31), (600, 420), (256, 256), (129, 700)], train, seed=7)
    got = _guarded_launch(batch)
    tight = _run(batch, out_hw=64)
    assert torch.equal(got.view(torch.int16), tight.view(torch.int16))


def test_augment_ragged_refuses_undersized_operands():
    batch = _batch([(40, 50), (70, 30)], True, seed=2)
    n = 2
    data, geom, params = batch.data_u8.to(DEV), batch.geom.to(DEV), batch.params.to(DEV)
    need = ops.ragged_inter_bytes(batch.geom)
    inter = torch.empty(need, dtype=torch.uint8, device=DEV)
    out = torch.empty(n, 64, 64, 4, dtype=torch.bfloat16, device=DEV)
    C = ops.require()

    def call(data=data, geom=geom, params=params, inter=inter, out=out, gh=batch.geom, ph=batch.params):
        C.augment_ragged(data, geom, params, inter, out, gh, ph, 64, 64, [0.5] * 3, [0.25] * 3)

    call()
    past = batch.geom.clone()
    past[1, 0] += 1                                      # row 1 ends one byte past src
    big = batch.geom.clone()
    big[0, 1] = 41                                       # image 0 claims one more row
    rh0 = batch.geom.clone()
    rh0[1, 3] = 0
    box = batch.params.clone()
    box[0, 0] = 40 - box[0, 2] + 1                        # crop box one row past the bottom
    neg = batch.params.clone()
    neg[1, 1] = -1
    cases = {
        "geometry past src": dict(gh=past),
        "size past src": dict(gh=big),
        "short src": dict(data=data[:-1]),
        "short inter": dict(inter=inter[:need - 1]),
        "short out": dict(out=out[:1]),
        "zero RH": dict(gh=rh0),
        "crop past the image": dict(ph=box),
        "negative crop": dict(ph=neg),
        "geom shape": dict(geom=geom[:1]),
        "host geom shape": dict(gh=batch.geom[:1]),
        "params shape": dict(params=params[:, :7].contiguous()),
        "host params on device": dict(ph=params),
    }
    for name, kw in cases.items():
        with pytest.raises(RuntimeError):
            call(**kw)
            torch.cuda.synchronize()
            pytest.fail("accepted: " + name)


def _mk_engine(batch=4, hw=64):
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine
    from distributed_vgg_f_b200.models.vggf import vggf_mini_spec

    os.environ.pop("B200_FUSE_POOL", None)
    return NativeEngine(vggf_mini_spec(3), device=torch.device(DEV), batch=batch, lr=1e-3, seed=0, input_hw=hw)


def _rel(a, b):
    return float((a.float() - b.float()).abs().max() / (b.float().abs().max() + 1e-12))


def test_engine_ragged_batch_equals_float_path():
    """forward_logits and train_step on a RaggedBatch against the same calls on RaggedBatch.to_float()
    (tolerance of test_engine_gpu.py::test_fused_input_path_equals_float_path)."""
    for train in (True, False):
        batch = _batch([(100, 140), (512, 384), (64, 64), (333, 1000)], train, seed=5)
        pinned = RaggedBatch(*(t.pin_memory() for t in batch[:4]), None)
        x = T.ragged_reference(batch.data_u8, batch.geom, batch.params, out_hw=64).to(DEV)
        y = batch.labels.to(DEV)
        eng = _mk_engine()
        a = eng.forward_logits(pinned)
        b = eng.forward_logits((x, y))
        assert _rel(a, b) < 2e-2
        eng.train_dropout = False
        la = float(eng.train_step(pinned))
        wa = eng.p32.clone()
        eng2 = _mk_engine()
        eng2.train_dropout = False
        lb = float(eng2.train_step((x, y)))
        assert math.isfinite(la) and abs(la - lb) <= 2e-2 * max(1.0, abs(lb))
        assert _rel(wa, eng2.p32) < 2e-2


class _Counting:
    """A loader wrapper that counts the samples it hands out."""

    def __init__(self, ld):
        self.ld, self.n = ld, 0

    def __len__(self):
        return len(self.ld)

    def set_epoch(self, e):
        self.ld.set_epoch(e)

    def __iter__(self):
        for b in self.ld:
            self.n += int(b.labels.numel())
            yield b


def test_trainer_fit_one_epoch_on_a_mixed_folder(tmp_path, capsys):
    from distributed_vgg_f_b200.data.loader import DataManager
    from distributed_vgg_f_b200.trainer import Trainer
    from test_ragged_input_cpu import _write_mixed

    root = _write_mixed(str(tmp_path / "mixed"))
    train = DataManager(root, 4, train=True, pipeline="fused")
    val = DataManager(root, 4, train=False, pipeline="fused")
    assert train.cache.ragged and val.cache.ragged
    eng = _mk_engine(batch=4, hw=224)
    tl, vl = _Counting(train.get_loader()), _Counting(val.get_loader())
    Trainer(eng, None, tl, vl, torch.device(DEV), verbose_throughput=False).fit(1)
    out = capsys.readouterr().out
    m = re.search(r"train loss: ([\d.naif]+), train acc: [\d.]+%, test loss: ([\d.naif]+)", out)
    assert m and all(math.isfinite(float(v)) for v in m.groups()), out
    assert tl.n == train.data_size and vl.n == val.data_size
