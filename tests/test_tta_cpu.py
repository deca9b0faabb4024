"""Test-time augmentation (--val-tta) without a GPU: the flag, the view origins against torchvision's five_crop /
ten_crop, the view chains of augment_reference and ragged_reference against torchvision and PIL, the DeviceMeter
reduction against a float64 formula, CLI runs on a synthetic folder against a hand-written torchvision loop for both
pipelines, --model-ema, and --shard-eval at two gloo ranks."""
import contextlib
import io
import json
import re
import socket

import numpy as np
import pytest
import torch

from distributed_vgg_f_b200.data import transforms as T

BASE = ["-iu", "tcp://127.0.0.1:29999", "-rn", "0", "-ws", "1", "-nc", "-mb", "4", "--model", "vggf-tiny",
        "--engine", "oracle"]
# validation images of the synthetic set are 128 x 128: a resize below that makes both splits ragged (Pillow-exact)
SIZES = ["--train-crop-size", "64", "--val-crop-size", "64", "--train-resize-size", "72", "--val-resize-size", "71"]


def _parse(extra):
    from distributed_vgg_f_b200 import cli
    return cli.parse_command_line(["-iu", "x", "-rn", "0", "-ws", "1", "-rd", "/r"] + extra, init=False)


# ------------------------------------------------------------------------------------------------ flags
def test_default_is_none_and_every_mode_parses():
    assert _parse([]).val_tta == "none"
    for mode in ("none", "flip", "five-crop", "ten-crop"):
        assert _parse(["--val-tta", mode]).val_tta == mode
    with pytest.raises(SystemExit), contextlib.redirect_stderr(io.StringIO()):
        _parse(["--val-tta", "twelve-crop"])


def test_view_tables():
    assert [len(T.tta_views(m)) for m in T.TTA_MODES] == [1, 2, 5, 10]
    with pytest.raises(ValueError):
        T.tta_views("multi-scale")
    with pytest.raises(ValueError):
        T.view_origin(T.TTA_CENTRE, 60, 80, 64, 64)          # the view does not fit


# ------------------------------------------------------------------------------- views against torchvision
@pytest.mark.parametrize("RH,RW,C", [(256, 256, 224), (255, 255, 224), (256, 341, 224), (71, 96, 64), (73, 64, 64),
                                     (100, 101, 98)])
def test_view_origins_are_torchvisions_five_crop_and_ten_crop(RH, RW, C):
    from torchvision.transforms import functional as TF

    img = torch.arange(RH * RW, dtype=torch.float64).view(1, RH, RW)

    def crop(view):
        y0, x0, flip = T.view_origin(view, RH, RW, C, C)
        src = TF.hflip(img) if flip else img
        return src[:, y0:y0 + C, x0:x0 + C]

    ten = TF.ten_crop(img, [C, C])
    for v, ref in zip(T.tta_views("ten-crop"), ten):
        assert torch.equal(crop(v), ref)
    for v, ref in zip(T.tta_views("five-crop"), TF.five_crop(img, [C, C])):
        assert torch.equal(crop(v), ref)
    centre = TF.center_crop(img, [C, C])
    flip = T.tta_views("flip")
    assert torch.equal(crop(flip[0]), centre) and torch.equal(crop(flip[1]), TF.hflip(centre))


@pytest.mark.parametrize("R,C", [(256, 224), (255, 224), (96, 64), (65, 64)])
def test_augment_reference_views_are_crops_of_the_resized_tensor(R, C):
    """The uniform path: each view of augment_reference is, bit for bit, torchvision's crop of the tensor the same
    chain makes of the whole R x R resized image."""
    from torchvision.transforms import functional as TF

    rng = np.random.default_rng(R)
    src = torch.from_numpy(rng.integers(0, 256, (2, 120, 120, 3), dtype=np.uint8))
    params = T.val_params(2, 120, 120)
    full = T.augment_reference(src, params, (R, R), out_hw=R)
    for mode, ref in (("ten-crop", TF.ten_crop(full, [C, C])), ("five-crop", TF.five_crop(full, [C, C])),
                      ("flip", (TF.center_crop(full, [C, C]), TF.hflip(TF.center_crop(full, [C, C]))))):
        for v, want in zip(T.tta_views(mode), ref):
            assert torch.equal(T.augment_reference(src, params, (R, R), out_hw=C, view=v), want), (mode, v)
    assert torch.equal(T.augment_reference(src, params, (R, R), out_hw=C, view=T.TTA_CENTRE),
                       T.augment_reference(src, params, (R, R), out_hw=C))


def _ragged(sizes, resize, seed=0):
    rng = np.random.default_rng(seed)
    imgs = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in sizes]
    data = torch.from_numpy(np.concatenate([a.reshape(-1) for a in imgs]))
    geom = T.ragged_geometry(sizes, False, resize)
    params = torch.cat([T.val_params(1, h, w) for h, w in sizes])
    return imgs, data, geom, params


@pytest.mark.parametrize("mode", ["flip", "five-crop", "ten-crop"])
def test_ragged_reference_views_are_pils_resize_and_ten_crop(mode):
    """Non-square images whose centre offsets end in .5; PIL's Resize, then TenCrop / FiveCrop / centre + mirror."""
    from PIL import Image

    sizes, resize, C = [(90, 133), (133, 90), (120, 120), (57, 200)], 71, 64
    imgs, data, geom, params = _ragged(sizes, resize)
    tf = T.reference_transforms(False, resize, C, mode)
    want = torch.stack([tf(Image.fromarray(a)) for a in imgs])                     # [n][V][3][C][C]
    for i, v in enumerate(T.tta_views(mode)):
        assert torch.equal(T.ragged_reference(data, geom, params, out_hw=C, view=v), want[:, i]), v


# ---------------------------------------------------------------------------------------- the reduction
def _formula(view_logits, target):
    z = np.asarray(view_logits, dtype=np.float64)
    p = np.exp(z - z.max(2, keepdims=True))
    p = (p / p.sum(2, keepdims=True)).mean(0)
    loss = -np.log(p[np.arange(len(target)), target]).sum()
    return loss, int((p.argmax(1) == target).sum()), p


@pytest.mark.parametrize("V,C", [(2, 3), (5, 3), (10, 1000)])
def test_device_meter_view_mean_matches_float64(V, C):
    from distributed_vgg_f_b200.ops import ref
    from distributed_vgg_f_b200.utils.metrics import DeviceMeter

    g = torch.Generator().manual_seed(V * C)
    z = torch.randn(V, 7, C, generator=g) * 3
    t = torch.randint(0, C, (7,), generator=g)
    z[:, 0, :] = 0.0                                      # a tie across every class: class 0 wins
    z[:, 1, 2 % C] = z[:, 1, 1 % C] = 9.0                 # a tie of two classes: the lower index wins
    t[0], t[1] = 1 % C, 2 % C
    m = DeviceMeter("cpu")
    m.add_tta(list(z), t)
    loss, correct, p = _formula(z.numpy(), t.numpy())
    assert abs(float(m.buf[0]) - loss) <= 1e-5 * max(1.0, loss)
    assert int(m.buf[1]) == correct and int(m.buf[2]) == 7
    assert np.argmax(p[0]) == 0 and np.argmax(p[1]) == min(1 % C, 2 % C)
    r = ref.tta_reduce64(z, t)
    assert abs(float(r["meter"][0]) - loss) <= 1e-9 * max(1.0, loss) and float(r["meter"][1]) == correct


# ------------------------------------------------------------------------------------------- CLI runs
def _main(argv):
    from distributed_vgg_f_b200 import cli

    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        assert cli.main(argv) == 0
    return buf.getvalue()


EVAL = re.compile(r"^\[Info\] Evaluation: test loss: ([\d.]+), test acc: ([\d.]+)%\.$", re.M)


@pytest.fixture(scope="module")
def trained(tmp_path_factory, synth_root):
    """One epoch of vggf-tiny with --model-ema and --val-tta ten-crop, saved and logged."""
    d = tmp_path_factory.mktemp("tta_runs")
    ck, log = str(d / "ck.pt"), str(d / "log.jsonl")
    text = _main(BASE + ["-rd", synth_root, "-ep", "1", "--seed", "5", "--model-ema", "--model-ema-steps", "1",
                         "--val-tta", "ten-crop", "--save", ck, "--log-jsonl", log] + SIZES)
    return text, ck, log


def test_training_run_reports_the_mode_and_its_ema_line(trained):
    text, _, log = trained
    assert "[Info] test-time augmentation: ten-crop (10 views per image, mean of their softmaxes)" in text
    assert re.search(r"^\[Info\] Epoch: 1/1, EMA test loss: [\d.]+, EMA test acc: [\d.]+%\.$", text, re.M)
    recs = [json.loads(s) for s in open(log).read().splitlines()]
    assert len(recs) == 1 and recs[0]["val_tta"] == "ten-crop" and "ema_test_acc" in recs[0]


def _hand_loop(ck, root, resize=71, crop=64):
    """Resize -> TenCrop -> model -> mean softmax, written out with torchvision and PIL alone."""
    from PIL import Image
    from torchvision import transforms as TV

    from distributed_vgg_f_b200.data.folder import scan_image_folder
    from distributed_vgg_f_b200.models.vggf import build_oracle, get_spec
    from distributed_vgg_f_b200.utils.checkpoint import strip_module_prefix

    net = build_oracle(get_spec("vggf-tiny", 3), seed=0).eval()
    net.load_state_dict(strip_module_prefix(torch.load(ck, weights_only=True)["model"]))
    norm = TV.Normalize([0.485, 0.456, 0.406], [0.229, 0.224, 0.225])
    _, samples = scan_image_folder(root + "/ValidationData")
    loss, correct = 0.0, 0
    with torch.no_grad():
        for path, label in samples:
            views = TV.TenCrop(crop)(TV.Resize(resize)(Image.open(path).convert("RGB")))
            x = torch.stack([norm(TV.functional.to_tensor(v)) for v in views])
            p = torch.softmax(net(x).double(), 1).mean(0)
            loss -= float(torch.log(p[label]))
            correct += int(int(p.argmax()) == label)
    return loss / len(samples), correct / len(samples)


@pytest.mark.parametrize("pipeline", ["fused", "reference"])
def test_eval_only_ten_crop_equals_a_torchvision_loop(trained, synth_root, pipeline):
    _, ck, _ = trained
    text = _main(BASE + ["-rd", synth_root, "--eval-only", "--resume", ck, "--val-tta", "ten-crop",
                         "--pipeline", pipeline] + SIZES)
    m = EVAL.search(text)
    assert m, text
    loss, acc = _hand_loop(ck, synth_root)
    assert abs(float(m.group(1)) - loss) <= 2e-6 + 1e-5 * loss
    assert abs(float(m.group(2)) - 100 * acc) < 0.006


def test_eval_only_none_is_unchanged(trained, synth_root):
    _, ck, _ = trained
    plain = _main(BASE + ["-rd", synth_root, "--eval-only", "--resume", ck] + SIZES)
    named = _main(BASE + ["-rd", synth_root, "--eval-only", "--resume", ck, "--val-tta", "none"] + SIZES)
    assert EVAL.search(plain).groups() == EVAL.search(named).groups()
    assert "test-time augmentation" not in named


# ------------------------------------------------------------------------------------- two gloo ranks
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _rank_main(rank, world, port, root, ck, out):
    import torch.distributed as dist

    from distributed_vgg_f_b200.data.loader import DataManager
    from distributed_vgg_f_b200.models.vggf import build_oracle, get_spec
    from distributed_vgg_f_b200.trainer import Trainer
    from distributed_vgg_f_b200.utils.checkpoint import strip_module_prefix

    dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%d" % port, rank=rank, world_size=world)
    net = build_oracle(get_spec("vggf-tiny", 3), seed=0)
    net.load_state_dict(strip_module_prefix(torch.load(ck, weights_only=True)["model"]))
    val = DataManager(root, 3, train=False, world_size=world, rank=rank, shard_eval=True, resize_size=71,
                      crop_size=64, tta="five-crop")
    tr = Trainer(net, None, [], val.get_loader(), torch.device("cpu"), verbose_throughput=False, shard_eval=True,
                 val_tta="five-crop")
    loss, acc = tr._evaluate()
    if rank == 0:
        torch.save(torch.tensor([loss.sum, loss.count, acc.correct], dtype=torch.float64), out)
    dist.destroy_process_group()


def test_shard_eval_at_two_gloo_ranks_equals_one_process(trained, synth_root, tmp_path):
    import torch.multiprocessing as mp

    _, ck, _ = trained
    res = {}
    for world in (2, 1):
        out = str(tmp_path / ("w%d.pt" % world))
        mp.spawn(_rank_main, args=(world, _free_port(), synth_root, ck, out), nprocs=world, join=True)
        res[world] = torch.load(out)
    assert res[2][1] == res[1][1] and res[2][2] == res[1][2]
    assert abs(float(res[2][0] - res[1][0])) <= 1e-5 * float(res[1][0])
