"""Input sizes other than the reference's 256 / 224 (--train-resize-size, --train-crop-size, --val-resize-size,
--val-crop-size) without a GPU: flag checks, the fused transform against torchvision at the new sizes, the
loader's uniform / ragged decision, a two-rank gloo run through the CLI, checkpoints and tools.predict."""
import json
import os
import re
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "reference")


def _parse(extra):
    from distributed_vgg_f_b200.cli import parse_command_line

    return parse_command_line(["-iu", "tcp://127.0.0.1:1", "-rn", "0", "-ws", "1", "-rd", "/nonexistent"] + extra,
                              init=False)


@pytest.mark.parametrize("extra,flag", [
    (["--train-crop-size", "288"], "--train-crop-size 288 exceeds --train-resize-size 256"),
    (["--val-resize-size", "200"], "--val-crop-size 224 exceeds --val-resize-size 200"),
    (["--train-crop-size", "24", "--train-resize-size", "32"], "--train-crop-size must be >= 32"),
    (["--val-crop-size", "16"], "--val-crop-size must be >= 32"),
])
def test_flags_are_refused_naming_the_flag(extra, flag, capsys):
    with pytest.raises(SystemExit):
        _parse(extra)
    assert flag in capsys.readouterr().err


def test_flag_defaults_are_the_references(capsys):
    from distributed_vgg_f_b200.cli import input_sizes

    a = _parse([])
    assert input_sizes(a) == dict(train_resize_size=256, train_crop_size=224, val_resize_size=256, val_crop_size=224)
    assert input_sizes(a) == input_sizes(None)
    a = _parse(["--train-crop-size", "176", "--val-resize-size", "232", "--val-crop-size", "224"])
    assert (a.train_crop_size, a.val_resize_size, a.val_crop_size) == (176, 232, 224)
    assert _parse(["--val-resize-size", "320", "--val-crop-size", "288"]).val_crop_size == 288
    assert _parse(["--train-crop-size", "33", "--engine", "oracle"]).train_crop_size == 33     # the oracle takes any


@pytest.mark.parametrize("hw", [56, 520, 180, 33, 0])
def test_native_engine_refuses_sizes_it_does_not_run(hw):
    from distributed_vgg_f_b200.engine.native_engine import check_native_hw

    with pytest.raises(ValueError, match="multiples of 8 from 64 to 512"):
        check_native_hw(hw, "eval_hw")
    for ok in (64, 128, 176, 200, 224, 232, 288, 512):
        assert check_native_hw(ok) == ok


@pytest.mark.parametrize("resize,crop", [(144, 128), (200, 176), (232, 224), (288, 256)])
def test_fused_transform_matches_torchvision_at_new_sizes(resize, crop):
    """augment_reference (what the kernel evaluates) against torchvision's own ops on PIL images, same draws."""
    from distributed_vgg_f_b200.data import transforms as T
    from distributed_vgg_f_b200.data.synthetic import synthetic_uint8_batch

    imgs, _ = synthetic_uint8_batch(3, 128, seed=resize)
    rng = np.random.default_rng(crop)
    imgs = np.clip(imgs.astype(np.int16) + rng.integers(-20, 20, imgs.shape), 0, 255).astype(np.uint8)
    params = T.sample_train_params(3, 128, 128, torch.Generator().manual_seed(crop))
    params[0, 6], params[1, 6] = 0.0, 1.0
    ours = T.augment_reference(torch.from_numpy(imgs), params, (resize, resize), out_hw=crop)
    assert ours.shape == (3, 3, crop, crop)
    for i in range(3):
        theirs = T.torchvision_chain_fixed(imgs[i], params[i], resize=resize, crop=crop)
        d = (ours[i] - theirs).abs()
        assert float((d < 0.04).float().mean()) > 0.995, (i, float(d.max()))
        assert float(d.mean()) < 0.012


def test_reference_transforms_take_the_sizes():
    from torchvision import transforms as TV

    from distributed_vgg_f_b200.data import transforms as T

    tr = T.reference_transforms(True, 200, 176).transforms
    assert isinstance(tr[0], TV.RandomResizedCrop) and tr[0].size == (200, 200)
    assert isinstance(tr[3], TV.CenterCrop) and tr[3].size == (176, 176)
    va = T.reference_transforms(False, 232, 224).transforms
    assert va[0].size == 232 and va[1].size == (224, 224)


def test_loader_uniform_or_ragged_follows_the_resize_size(tmp_path):
    """One image size of at most the split's resize size is cached uniform; larger images go ragged."""
    from PIL import Image

    from distributed_vgg_f_b200.data.loader import DataManager

    for split in ("TrainData", "ValidationData"):
        for c in ("a", "b"):
            d = tmp_path / split / c
            d.mkdir(parents=True)
            for i in range(2):
                Image.new("RGB", (200, 200), (i * 50, 100, 30)).save(str(d / ("%d.png" % i)))
    root = str(tmp_path)
    kw = dict(pipeline="fused", seed=0)
    assert not DataManager(root, 2, train=True, **kw).cache.ragged                       # 200 <= 256
    small = DataManager(root, 2, train=True, resize_size=144, crop_size=128, **kw)
    assert small.cache.ragged                                                             # 200 > 144
    batch = next(iter(small.get_loader()))
    assert small.get_loader().crop == 128 and batch.geom[:, 3:].tolist() == [[144, 144]] * 2
    assert batch.to_float(out_hw=128)[0].shape == (2, 3, 128, 128)
    val = DataManager(root, 2, train=False, resize_size=232, crop_size=224, **kw)
    assert not val.cache.ragged
    vb = next(iter(val.get_loader()))
    assert vb.resized_hw == (232, 232) and val.get_loader().crop == 224
    ref = DataManager(root, 2, train=False, pipeline="reference", resize_size=232, crop_size=224)
    assert next(iter(ref.get_loader()))[0].shape == (2, 3, 224, 224)


def test_mix_boxes_use_the_crop_size():
    from distributed_vgg_f_b200.data import transforms as T

    for hw in (128, 176):
        for idx in range(20):
            d = T.draw_mix(0.0, 1.0, 0, 1, 0, idx, hw=hw)
            x1, y1, x2, y2 = d.box
            assert 0 <= x1 <= x2 <= hw and 0 <= y1 <= y2 <= hw


def test_oracle_at_128_matches_the_golden_forward():
    from distributed_vgg_f_b200 import vgg_funnel_model

    torch.manual_seed(0)
    model = vgg_funnel_model(3).eval()
    x = torch.randn(1, 3, 128, 128, generator=torch.Generator().manual_seed(2))
    with torch.no_grad():
        y = model(x)
    assert torch.allclose(y, torch.from_numpy(np.load(os.path.join(GOLDEN, "ref_forward_128.npy"))), rtol=1e-5,
                          atol=1e-6)
    with torch.no_grad():                       # 176: an odd 11 x 11 map before the last pool, 5 x 5 after it
        assert model(torch.randn(1, 3, 176, 176)).shape == (1, 3)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


SIZES = ["--train-crop-size", "176", "--val-resize-size", "232", "--val-crop-size", "224"]


def test_cli_two_ranks_gloo_fixres(synth_root, tmp_path):
    port = _free_port()
    ck, log = str(tmp_path / "ck.pt"), str(tmp_path / "log.jsonl")
    procs = []
    for r in range(2):
        cmd = [sys.executable, "-m", "distributed_vgg_f_b200", "-iu", "tcp://127.0.0.1:%d" % port, "-rn", str(r),
               "-ws", "2", "-rd", synth_root, "-ep", "1", "-nc", "-lr", "0.001", "-mb", "4", "--model", "vggf-tiny",
               "--engine", "oracle", "--save", ck, "--log-jsonl", log] + SIZES
        env = dict(os.environ, PYTHONPATH=ROOT, OMP_NUM_THREADS="2")
        procs.append(subprocess.Popen(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                                      text=True))
    outs = [p.communicate(timeout=600)[0] for p in procs]
    assert all(p.returncode == 0 for p in procs), outs
    pat = re.compile(r"test loss: ([\d.]+), test acc: ([\d.]+)%")
    tests = []
    for out in outs:
        assert "[Info] input sizes: train RandomResizedCrop 256 -> crop 176, eval Resize 232 -> crop 224" in out
        tests.append(pat.findall(out))
    assert tests[0] and tests[0] == tests[1]
    with open(log) as f:
        rec = json.loads(f.readline())
    assert rec["input_sizes"] == dict(train_resize_size=256, train_crop_size=176, val_resize_size=232,
                                      val_crop_size=224)
    payload = torch.load(ck, weights_only=False)
    assert (payload["args"]["train_crop_size"], payload["args"]["val_resize_size"],
            payload["args"]["val_crop_size"]) == (176, 232, 224)

    # tools.predict takes the checkpoint's evaluation sizes; --resize / --crop override them
    from distributed_vgg_f_b200.tools import predict as P

    assert P.eval_sizes(torch.load(ck, weights_only=False)["args"]) == (232, 224)
    seen = []
    real = P.reference_transforms

    def spy(train, resize, crop):
        seen.append((train, resize, crop))
        return real(train, resize, crop)

    P.reference_transforms = spy
    try:
        img = os.path.join(synth_root, "ValidationData")
        logits, files = P.predict(ck, [img], model="vggf-tiny", engine="oracle")
        assert logits.shape == (len(files), 3) and bool(torch.isfinite(logits).all())
        P.predict(ck, [img], model="vggf-tiny", engine="oracle", resize=160, crop=128)
        with pytest.raises(ValueError, match="exceeds"):
            P.predict(ck, [img], model="vggf-tiny", engine="oracle", resize=128, crop=160)
    finally:
        P.reference_transforms = real
    assert seen == [(False, 232, 224), (False, 160, 128)]


def test_default_run_writes_no_size_record(synth_root, tmp_path):
    """At the four defaults: no banner line, no JSONL key (the records stay as they were)."""
    out = subprocess.run([sys.executable, "-m", "distributed_vgg_f_b200", "-iu", "tcp://127.0.0.1:1", "-rn", "0",
                          "-ws", "1", "-rd", synth_root, "-ep", "1", "-nc", "-mb", "8", "--model", "vggf-tiny",
                          "--engine", "oracle", "--log-jsonl", str(tmp_path / "l.jsonl")],
                         cwd=ROOT, env=dict(os.environ, PYTHONPATH=ROOT, OMP_NUM_THREADS="2"), capture_output=True,
                         text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "input sizes" not in out.stdout
    with open(tmp_path / "l.jsonl") as f:
        assert "input_sizes" not in json.loads(f.readline())
