"""Every native kernel launch the engine makes, replayed against the float64 reference on guarded operands.

The kernel tests pick their shapes by hand; this one takes them from the engine.  ``ops._C`` is
swapped for a recording proxy during one train_step and one eval_step of several configurations.
Each distinct call signature of a recorded kernel (shapes, strides, dtypes, storage offset
mod 16 elements, scalars, which optional tensors are present) is then run once more in exact mode
on fresh guarded tensors laid out the same way, so the vector-store alignment paths match, and
checked twice (launch_replay.py): its values against the reference (exact where the arithmetic
allows it, else against kernel_check's bound), and its footprint against the write contract of the
kernel -- nothing outside what it may write changes, every element it must store is stored, and
accumulation targets are added to.  The optimizer runs on a side stream, so its replay, like every
other, uses fresh tensors with the recorded storage offset mod 16 elements.  When a dispatch rule or
a split heuristic of the engine changes, the replay follows it.
"""
import pytest
import torch

import kernel_check as KC
from launch_replay import CONTRACT, RECORDED, _record, replay_all

pytestmark = pytest.mark.gpu
DEV = "cuda"


def test_replay_every_wgmma_launch_of_the_engine(capsys):
    from distributed_vgg_f_b200.models.vggf import vgg16_spec, vggf_spec

    assert set(CONTRACT) == set(RECORDED)
    configs = [
        (vggf_spec(3), 64, (64, 37), {}, {}),                   # default step, and a ragged last batch of 37
        (vggf_spec(3), 64, (64, 37), {}, {"fused": True}),      # uint8 images through augment (NHWC, pad 4)
        (vggf_spec(3), 16, (16,), {}, {}),                      # 32-wide GEMM tiles on the FC layers
        (vgg16_spec(1000), 32, (32,), {}, {}),                  # unfused head: GEMM + fc_bias_act + CE
        (vggf_spec(3), 64, (64,), {"B200_FUSE_POOL": "0"}, {}),  # separate conv and pool kernels
        (vggf_spec(3), 8, (8,), {}, {"input_hw": 64, "reload": True}),  # 2x2 feature map: avgpool
        (vggf_spec(3), 8, (8,), {"B200_FUSE_POOL": "0"}, {"input_hw": 128, "optimizer": "sgd",
                                                           "weight_decay": 1e-4, "class_weights": [0.5, 1.0, 2.0]}),
        (vggf_spec(3), 37, (37,), {"B200_FUSED_HEAD": "0"}, {}),  # unfused 3-class head
    ]
    C, sigs = _record(configs)
    assert sigs
    missing = set(RECORDED) - {s[0] for s in sigs}
    assert not missing, "kernels the configurations never reached: %s" % sorted(missing)
    g = torch.Generator(device=DEV).manual_seed(0)
    kinds = replay_all(C, sigs, g, KC.sm_count())
    with capsys.disabled():
        print("\n[replay] %d launch signatures replayed: %s" % (len(sigs), ", ".join("%s=%d" % kv for kv in
                                                                                      sorted(kinds.items()))))
