"""--deterministic without a GPU: the flag's way to both engines, the split arithmetic the workspace is
sized from, the fp32-order emulation of splitk_reduce, and two identical torch-op runs."""
import io
import contextlib

import pytest
import torch

from distributed_vgg_f_b200 import cli, ops
from distributed_vgg_f_b200.ops import ref as R

needs_ext = pytest.mark.skipif(not ops.available(), reason="needs the built extension (host code only)")
BASE = ["-iu", "tcp://127.0.0.1:29999", "-rn", "0", "-ws", "1", "-rd", "/nonexistent"]


def test_flag_parses_and_defaults_to_off():
    p = cli.build_parser()
    assert p.parse_args(BASE).deterministic is False
    assert p.parse_args(BASE + ["--deterministic"]).deterministic is True


def test_flag_reaches_the_native_engine(monkeypatch, tmp_path):
    """manage_training passes deterministic= to NativeEngine (stopped at construction: no GPU here)."""
    from distributed_vgg_f_b200 import train
    from distributed_vgg_f_b200.engine import native_engine

    seen = {}

    class Stop(Exception):
        pass

    def fake(*a, **k):
        seen.update(k)
        raise Stop

    monkeypatch.setattr(native_engine, "NativeEngine", fake)
    monkeypatch.setattr(train, "_want_native", lambda args, device: True)
    for extra, want in (([], False), (["--deterministic"], True)):
        argv = BASE[:-1] + [str(tmp_path / "s"), "-nc", "-mb", "4", "--model", "vggf-tiny", "--synthetic", "2"] + extra
        with pytest.raises(Stop):
            train.manage_training(cli.parse_command_line(argv))
        assert seen["deterministic"] is want


@needs_ext
def test_nvls_is_refused_with_the_reason():
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine
    from distributed_vgg_f_b200.models.vggf import vggf_mini_spec

    with pytest.raises(ValueError, match="nvls leaves the summation order to the NVLink switch"):
        NativeEngine(vggf_mini_spec(3), device="cuda:0", batch=4, allreduce="nvls", deterministic=True, distributed=False)


# splits at 132 SMs and batch 64, 224^2, worked out by hand from the launchers' rules:
#   conv0: 132 CTAs x 2 consumers; Cin 64 (halo kernel): 132 SMs / (Cout / 64) work items;
#   FC: min(k-blocks, 256 / row tiles); 512 -> 512 at 14^2: 196 pixel tiles, 144 tiles per split ->
#   4 splits = 576 items = 4.4 waves of 49 k-blocks (5 x 49 = 245) beat 3 splits (4 x 66 = 264) and 2 (3 x 98)
VGGF_SPLITS = {("features.0", "wgrad"): (264, 4096), ("features.2", "wgrad"): (132, 64 * 9 * 64),
               ("features.5", "wgrad"): (66, 128 * 9 * 64), ("features.28", "wgrad"): (4, 512 * 9 * 512),
               ("classifier.0", "fprop"): (8, 64 * 4096), ("classifier.6.0", "fprop"): (64, 64 * 512),
               ("classifier.3", "dgrad"): (8, 64 * 4096), ("classifier.0", "bias"): (4, 4096)}


@needs_ext
def test_workspace_arithmetic_at_132_sms():
    from distributed_vgg_f_b200.engine.native_engine import deterministic_plan, deterministic_workspace_elems
    from distributed_vgg_f_b200.models.vggf import get_spec

    plan = deterministic_plan(get_spec("vggf", 3), 64, 224, 132)
    got = {(n, w): (s, e) for n, w, s, e in plan}
    for key, want in VGGF_SPLITS.items():
        assert got[key] == want, key
    assert ("classifier.0", "dgrad") not in got and ("classifier.6.3", "fprop") not in got   # first FC; fused head
    assert deterministic_workspace_elems(plan) == 4 * 512 * 9 * 512          # 37.7 MB
    # VGG-16 / 1000 classes: the GEMM head's forward and dgrad are split too; the convolutions are VGG-F's
    p16 = {(n, w): (s, e) for n, w, s, e in deterministic_plan(get_spec("vgg16", 1000), 64, 224, 132, fused_head=False)}
    assert p16[("classifier.6", "fprop")] == (32, 64 * 1000) and p16[("classifier.6", "dgrad")] == (8, 64 * 4096)
    assert p16[("features.28", "wgrad")] == got[("features.28", "wgrad")]
    mini = deterministic_plan(get_spec("vggf-mini", 3), 4, 64, 132)
    C = ops.require()
    for name, what, splits, elems in mini:
        assert splits >= 1 and elems % 4 == 0
    assert deterministic_workspace_elems(mini) == max(s * e for _, _, s, e in mini)
    assert C.gemm_splits(25088, 8) == 8 and C.gemm_splits(100, 8) == 2 and C.gemm_splits(64 * 5, 4) == 3


@needs_ext
def test_split_count_depends_on_the_sm_count_only_through_the_argument():
    C = ops.require()
    assert C.conv_wgrad_splits(64, 224, 224, 64, 64, 132) == 132
    assert C.conv_wgrad_splits(64, 224, 224, 64, 64, 114) == 114
    assert C.conv0_wgrad_splits(1, 8, 8, 132) == 2


@needs_ext
def test_tools_plan_deterministic():
    from distributed_vgg_f_b200.tools import plan

    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        assert plan.main(["--deterministic", "--sms", "132"]) == 0
    out = buf.getvalue()
    assert "132 SMs: workspace 37.7 MB" in out
    assert any(line.split()[:3] == ["features.2", "wgrad", "132"] for line in out.splitlines())


def test_tools_plan_says_so_without_the_extension(monkeypatch, capsys):
    from distributed_vgg_f_b200.tools import plan

    monkeypatch.setattr(ops, "_C", None)
    assert plan.main(["--deterministic"]) == 1
    assert "build it first" in capsys.readouterr().out


@pytest.mark.parametrize("splits,n", [(1, 17), (5, 64), (33, 100)])
def test_ordered_emulation_is_the_python_loop_and_close_to_float64(splits, n):
    import numpy as np

    g = torch.Generator().manual_seed(splits)
    s = torch.randn(splits, n, generator=g) * 10
    dst = torch.randn(n, generator=g)
    for d, alpha in ((None, 1.0), (dst, 0.37)):
        got = R.splitk_reduce_ordered(s, d, alpha)
        a32 = np.float32(alpha)
        for i in range(n):
            acc = np.float32(s[0, i].item())
            for k in range(1, splits):
                acc = np.float32(acc + np.float32(s[k, i].item()))
            acc = np.float32(a32 * acc)
            if d is not None:
                acc = np.float32(np.float32(d[i].item()) + acc)
            assert got[i].item() == float(acc)
        ref, _ = R.splitk_reduce64(s, d, alpha)
        ulp = torch.finfo(torch.float32).eps * (abs(alpha) * s.double().abs().sum(0) + (0 if d is None else d.double().abs()))
        assert bool(((got.double() - ref).abs() <= (splits + 2) * ulp).all())


def test_torch_op_engine_repeats_itself_under_the_flag(tmp_path):
    """Two runs of two epochs on --synthetic data (dropout on): identical checkpoints."""
    from distributed_vgg_f_b200.train import manage_training

    try:
        states = []
        for run in ("a", "b"):
            ck = str(tmp_path / (run + ".pt"))
            argv = BASE[:-1] + [str(tmp_path / "synth"), "-ep", "2", "-nc", "-mb", "4", "--model", "vggf-tiny",
                                "--synthetic", "4", "--engine", "oracle", "--deterministic", "--save", ck]
            manage_training(cli.parse_command_line(argv))
            assert torch.are_deterministic_algorithms_enabled()
            states.append(torch.load(ck, map_location="cpu", weights_only=True))
    finally:
        torch.use_deterministic_algorithms(False)
    a, b = states
    assert a["model"].keys() == b["model"].keys()
    for k in a["model"]:
        assert torch.equal(a["model"][k], b["model"][k]), k
    for k, st in a["optimizer"]["state"].items():
        for name, t in st.items():
            assert torch.equal(torch.as_tensor(t), torch.as_tensor(b["optimizer"]["state"][k][name])), (k, name)
