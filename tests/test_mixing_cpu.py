"""Label smoothing, MixUp and CutMix without a GPU: the flags, the per-batch draws against torchvision's
own code, the loaders with the flags off, and the torch-op trainer against F.cross_entropy on
torchvision-mixed targets."""
import os
import re
import socket
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---------------------------------------------------------------------------------------------- CLI
@pytest.mark.parametrize("flag,value,ok", [("--label-smoothing", "0.1", True), ("--label-smoothing", "0", True),
                                           ("--label-smoothing", "1.0", False), ("--label-smoothing", "-0.1", False),
                                           ("--mixup-alpha", "0.2", True), ("--mixup-alpha", "-1", False),
                                           ("--cutmix-alpha", "1.0", True), ("--cutmix-alpha", "-0.5", False)])
def test_cli_validates_the_flags(flag, value, ok, capsys):
    from distributed_vgg_f_b200 import cli

    argv = ["-iu", "tcp://127.0.0.1:1", "-rn", "0", "-ws", "1", "-rd", "/nonexistent", flag, value]
    if ok:
        args = cli.parse_command_line(argv, init=False)
        assert getattr(args, flag[2:].replace("-", "_")) == float(value)
    else:
        with pytest.raises(SystemExit):
            cli.parse_command_line(argv, init=False)


def test_cli_defaults_are_off():
    from distributed_vgg_f_b200 import cli

    args = cli.build_parser().parse_args(["-iu", "x", "-rn", "0", "-ws", "1", "-rd", "/r"])
    assert (args.label_smoothing, args.mixup_alpha, args.cutmix_alpha) == (0.0, 0.0, 0.0)


# -------------------------------------------------------------------------------------------- draws
def _torchvision_batch(mixup_alpha, cutmix_alpha, seed, x, y, C):
    """torchvision's classification reference: RandomChoice([MixUp, CutMix]) when both are on, run on
    the collated batch under the given global seed."""
    from torchvision.transforms import v2

    ts = []
    if mixup_alpha > 0:
        ts.append(v2.MixUp(alpha=mixup_alpha, num_classes=C))
    if cutmix_alpha > 0:
        ts.append(v2.CutMix(alpha=cutmix_alpha, num_classes=C))
    t = ts[0] if len(ts) == 1 else v2.RandomChoice(ts)
    with torch.random.fork_rng(devices=[]):
        torch.manual_seed(seed)
        return t(x.clone(), y.clone())


@pytest.mark.parametrize("mixup_alpha,cutmix_alpha", [(0.2, 0.0), (0.0, 1.0), (0.2, 1.0), (1.0, 0.5)])
def test_draws_equal_torchvision_for_the_same_seed(mixup_alpha, cutmix_alpha):
    from distributed_vgg_f_b200.data import transforms as T

    C, b, hw = 5, 6, 224
    g = torch.Generator().manual_seed(0)
    x = torch.randn(b, 3, hw, hw, generator=g)
    y = torch.randint(0, C, (b,), generator=g)
    kinds = set()
    for index in range(12):
        seed = T.mix_seed(3, 1, 0, index)
        mix = T.draw_mix(mixup_alpha, cutmix_alpha, 3, 1, 0, index, hw=hw)
        kinds.add(mix.kind)
        want_x, want_y = _torchvision_batch(mixup_alpha, cutmix_alpha, seed, x, y, C)
        assert torch.equal(T.apply_mix(x, y, mix), want_x)
        assert torch.equal(T.mixed_targets(y, C, mix), want_y)
        if mix.kind == "cutmix":
            x1, y1, x2, y2 = mix.box
            assert 0 <= x1 <= x2 <= hw and 0 <= y1 <= y2 <= hw
            assert mix.lam == 1.0 - (x2 - x1) * (y2 - y1) / (hw * hw)
    assert kinds == ({"mixup"} if not cutmix_alpha else {"cutmix"} if not mixup_alpha else {"mixup", "cutmix"})


def test_draws_are_reproducible_and_leave_the_global_rng_alone():
    from distributed_vgg_f_b200.data import transforms as T

    torch.manual_seed(11)
    before = torch.rand(3)
    torch.manual_seed(11)
    a = [T.draw_mix(0.2, 1.0, 0, e, r, i) for e in range(2) for r in range(2) for i in range(3)]
    after = torch.rand(3)
    assert torch.equal(before, after)
    assert a == [T.draw_mix(0.2, 1.0, 0, e, r, i) for e in range(2) for r in range(2) for i in range(3)]
    assert len(set(a)) == len(a)                     # every (epoch, rank, index) draws its own
    assert T.draw_mix(0.0, 0.0, 0, 0, 0, 0) is None


def test_pairing_rolls_over_the_actual_batch():
    """Sample i's partner is (i - 1) mod b for short batches too, and a batch of one pairs with itself."""
    from distributed_vgg_f_b200.data import transforms as T

    for b in (1, 3):
        x = torch.arange(b, dtype=torch.float32).view(b, 1, 1, 1).expand(b, 3, 4, 4).contiguous()
        y = torch.arange(b)
        out = T.apply_mix(x, y, T.MixDraw("mixup", 0.75, (0, 0, 0, 0)))
        partner = (torch.arange(b) - 1) % b
        assert torch.allclose(out[:, 0, 0, 0], 0.75 * torch.arange(b) + 0.25 * partner.float())
        cut = T.apply_mix(x, y, T.MixDraw("cutmix", 0.75, (0, 0, 2, 2)))
        assert torch.equal(cut[:, 0, 0, 0], partner.float()) and torch.equal(cut[:, 0, 3, 3], torch.arange(b).float())


# ------------------------------------------------------------------------------------------ loaders
def _epoch(loader):
    out = []
    for bt in loader:
        out.append(tuple(t.clone() if isinstance(t, torch.Tensor) else t for t in bt))
    return out


@pytest.mark.parametrize("ragged", [False, True])
def test_flags_off_leave_fused_batches_unchanged_and_on_only_add_the_draw(tmp_path, ragged):
    from distributed_vgg_f_b200.data.loader import DecodedCache, _FusedLoader
    from distributed_vgg_f_b200.data.synthetic import make_synthetic_imagefolder
    from distributed_vgg_f_b200.data.folder import scan_image_folder

    root = str(tmp_path / "d")
    make_synthetic_imagefolder(root, train_per_class=4, val_per_class=1, size=300 if ragged else 64, seed=1)
    _, samples = scan_image_folder(os.path.join(root, "TrainData"))
    cache = DecodedCache(samples, threads=2)
    assert cache.ragged == ragged
    base = _epoch(_FusedLoader(cache, 5, True, None, True, seed=2, pin=False, native=False))
    off = _epoch(_FusedLoader(cache, 5, True, None, True, seed=2, pin=False, native=False,
                              mixup_alpha=0.0, cutmix_alpha=0.0))
    on = _epoch(_FusedLoader(cache, 5, True, None, True, seed=2, pin=False, native=False,
                             mixup_alpha=0.2, cutmix_alpha=1.0))
    val = _epoch(_FusedLoader(cache, 5, False, None, False, seed=2, pin=False, native=False,
                              mixup_alpha=0.2, cutmix_alpha=1.0))
    assert len(base) == len(off) == len(on) == 3
    for a, b, c in zip(base, off, on):
        assert a[-1] is None and b[-1] is None and c[-1] is not None
        for i, t in enumerate(a):
            if isinstance(t, torch.Tensor):
                assert torch.equal(t, b[i]) and torch.equal(t, c[i])       # bytes, params, labels, geometry
    assert all(bt[-1] is None for bt in val)                              # validation is never mixed


def test_reference_loader_yields_pairs_when_off_and_mixed_triples_when_on(tmp_path):
    from distributed_vgg_f_b200.data import transforms as T
    from distributed_vgg_f_b200.data.folder import scan_image_folder
    from distributed_vgg_f_b200.data.loader import _ReferenceLoader
    from distributed_vgg_f_b200.data.synthetic import make_synthetic_imagefolder

    root = str(tmp_path / "d")
    make_synthetic_imagefolder(root, train_per_class=3, val_per_class=1, size=64, seed=1)
    _, samples = scan_image_folder(os.path.join(root, "TrainData"))
    off = _ReferenceLoader(samples, 4, True, None, False, seed=0)
    on = _ReferenceLoader(samples, 4, True, None, False, seed=0, mixup_alpha=0.4, cutmix_alpha=0.4)
    torch.manual_seed(5)
    plain = list(off)
    torch.manual_seed(5)
    mixed = list(on)
    assert all(len(bt) == 2 for bt in plain) and all(len(bt) == 3 for bt in mixed)
    for k, ((x, y), (xm, ym, mix)) in enumerate(zip(plain, mixed)):
        assert torch.equal(y, ym) and mix == T.draw_mix(0.4, 0.4, 0, 0, 0, k)
        assert torch.equal(xm, T.apply_mix(x, y, mix))


# ------------------------------------------------------------------------------------ oracle trainer
@pytest.mark.parametrize("kind", ["smooth", "mixup", "cutmix"])
@pytest.mark.parametrize("weighted", [False, True])
def test_oracle_trainer_loss_is_cross_entropy_on_torchvision_mixed_targets(kind, weighted):
    from torchvision.transforms import v2

    from distributed_vgg_f_b200.data import transforms as T
    from distributed_vgg_f_b200.data.loader import FusedBatch
    from distributed_vgg_f_b200.models.vggf import build_oracle, vggf_tiny_spec
    from distributed_vgg_f_b200.trainer import Trainer

    C, b = 3, 5
    model = build_oracle(vggf_tiny_spec(C), seed=0)
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    g = torch.Generator().manual_seed(4)
    src = torch.randint(0, 256, (b, 72, 72, 3), dtype=torch.uint8, generator=g)
    params = T.sample_train_params(b, 72, 72, g)
    labels = torch.tensor([0, 2, 2, 1, 0])
    eps = 0.1 if kind == "smooth" else 0.05
    mix = None
    if kind == "mixup":
        mix = T.MixDraw("mixup", 0.3, (0, 0, 0, 0))
    elif kind == "cutmix":
        mix = T.MixDraw("cutmix", 1.0 - 30 * 20 / 224 ** 2, (10, 5, 40, 25))
    batch = FusedBatch(src, params, labels, (72, 72), None, mix)
    cw = torch.tensor([1.0, 2.0, 0.5]) if weighted else None
    # expected: torchvision's transform on the unmixed float batch, F.cross_entropy on its targets
    x = T.augment_reference(src, params, (72, 72))           # 224 x 224, as FusedBatch.to_float
    tgt = labels
    if mix is not None:
        tv = v2.MixUp(alpha=1.0, num_classes=C) if kind == "mixup" else v2.CutMix(alpha=1.0, num_classes=C)
        p = dict(labels=labels, batch_size=b, lam=mix.lam, box=mix.box, lam_adjusted=mix.lam)
        x, tgt = tv.transform(x, p), tv.transform(labels, p)
    model.train()
    with torch.no_grad():
        out = model(x)
    want = F.cross_entropy(out, tgt, weight=cw, label_smoothing=eps)
    opt = torch.optim.SGD(model.parameters(), lr=0.0)
    tr = Trainer(model, opt, [batch], [], "cpu", class_weights=cw, verbose_throughput=False, label_smoothing=eps)
    avg, acc = tr._train()
    assert avg.count == b and abs(avg.average - float(want)) < 1e-5
    cls = tgt.argmax(1) if tgt.dim() == 2 else tgt
    assert acc.correct == int((out.argmax(1) == cls).sum())


# ------------------------------------------------------------------------------------- 2 gloo ranks
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def test_two_gloo_ranks_with_all_three_flags_keep_replicas_identical(synth_root):
    port = _free_port()
    procs = []
    for r in range(2):
        cmd = [sys.executable, "-m", "distributed_vgg_f_b200", "-iu", "tcp://127.0.0.1:%d" % port, "-rn", str(r),
               "-ws", "2", "-rd", synth_root, "-ep", "1", "-nc", "-lr", "0.001", "-mb", "4", "--model", "vggf-tiny",
               "--engine", "oracle", "--label-smoothing", "0.1", "--mixup-alpha", "0.2", "--cutmix-alpha", "1.0"]
        env = dict(os.environ, PYTHONPATH=ROOT, OMP_NUM_THREADS="2")
        procs.append(subprocess.Popen(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                                      text=True))
    outs = [p.communicate(timeout=600)[0] for p in procs]
    assert all(p.returncode == 0 for p in procs), outs
    pat = re.compile(r"\[Info\] Epoch: 1/1, train loss: ([\d.]+), train acc: ([\d.]+)%, "
                     r"test loss: ([\d.]+), test acc: ([\d.]+)%\.")
    lines = [pat.findall(o) for o in outs]
    assert all(len(l) == 1 for l in lines), outs
    # unsharded validation on synchronised replicas: the same test loss and accuracy on both ranks;
    # each rank trained on its own shard with its own draws
    assert lines[0][0][2:] == lines[1][0][2:]
    assert lines[0][0][0] != lines[1][0][0]
