"""The 256-wide channel tiles of the implicit-GEMM convolutions (umma_kernel at BN = 256), forced with
bn=256 and checked against the float64 references: fprop, fprop + fused pool, dgrad (plain, ReLU
mask, mask + column sum) and wgrad, at the 56^2, 28^2 and 14^2 layer shapes, at batch 64 and at a
ragged batch of 37.  A 256-wide tile adds the same k16 steps in the same order to each output
element as two 128-wide tiles, so fprop and dgrad must also equal their bn=128 results bit for bit."""
import math

import pytest
import torch

import kernel_check as KC
from distributed_vgg_f_b200.ops import ref as R

pytestmark = pytest.mark.gpu

DEV = "cuda"
MODES = ["exact", "gauss"]
# (N, H, W, Cin, Cout): a small case (the sanitizer runs it), then the layer shapes at batch 64 and 37
SHAPES = [(2, 28, 28, 256, 256)] + [(n, h, h, ci, co) for n in (64, 37) for h, ci, co in (
    (56, 256, 256), (28, 256, 512), (28, 512, 512), (14, 512, 512), (14, 512, 256))]
WIDE = pytest.mark.parametrize("N,H,W,Cin,Cout", SHAPES)


def _ops():
    from distributed_vgg_f_b200 import ops
    ops.require()
    return ops


def _case(N, H, W, Cin, Cout, seed, mode):
    g = KC.generator(seed * 1000003 + N * 7919 + H * 131 + Cin + 3 * Cout, DEV)
    x = KC.operand((N, H, W, Cin), mode, 9 * Cin, g, DEV)
    w = KC.operand((Cout, 3, 3, Cin), mode, 9 * max(Cin, Cout), g, DEV, scale=1.0 / math.sqrt(9 * Cin))
    b = KC.bias(Cout, mode, g, DEV)
    return x, w, b, g


@pytest.mark.parametrize("mode", MODES)
@WIDE
def test_wide_fprop(N, H, W, Cin, Cout, mode):
    ops = _ops()
    x, w, b, _ = _case(N, H, W, Cin, Cout, 11, mode)
    y = ops.conv3x3_fprop(x, w, b, relu=True, bn=256)
    ref, mag = R.conv3x3_fprop64(x, w, b, relu=True)
    KC.check(y, ref, mag, chain=KC.conv_chain(Cin), exact=mode == "exact", family="conv_fprop", what="bn=256")
    del ref, mag
    assert torch.equal(y, ops.conv3x3_fprop(x, w, b, relu=True, bn=128))


@pytest.mark.parametrize("mode", MODES)
@WIDE
def test_wide_fprop_pool(N, H, W, Cin, Cout, mode):
    ops = _ops()
    x, w, b, _ = _case(N, H, W, Cin, Cout, 12, mode)
    p, mask = ops.conv3x3_fprop_pool(x, w, b, bn=256)
    ref, mag = R.conv3x3_fprop64(x, w, b, relu=True)
    KC.check_pool(p, mask, ref, mag, chain=KC.conv_chain(Cin), exact=mode == "exact", what="bn=256")
    del ref, mag
    p128, mask128 = ops.conv3x3_fprop_pool(x, w, b, bn=128)
    assert torch.equal(p, p128) and torch.equal(mask, mask128)


@pytest.mark.parametrize("mode", MODES)
@WIDE
def test_wide_dgrad(N, H, W, Cin, Cout, mode):
    ops = _ops()
    exact = mode == "exact"
    _, w, _, g = _case(N, H, W, Cin, Cout, 13, mode)
    dz = KC.operand((N, H, W, Cout), mode, 9 * Cout, g, DEV)
    chain = KC.conv_chain(Cout)
    dx = ops.conv3x3_dgrad(dz, w, Cin, bn=256)
    ref, mag = R.conv3x3_dgrad64(dz, w)
    KC.check(dx, ref, mag, chain=chain, exact=exact, family="conv_dgrad", what="bn=256")
    assert torch.equal(dx, ops.conv3x3_dgrad(dz, w, Cin, bn=128))
    mask_src = KC.operand((N, H, W, Cin), "gauss", 1, g, DEV)
    dx2 = ops.conv3x3_dgrad(dz, w, Cin, mask_src=mask_src, bn=256)
    ref, mag = R.conv3x3_dgrad64(dz, w, mask_src=mask_src)
    KC.check(dx2, ref, mag, chain=chain, exact=exact, family="conv_dgrad", what="bn=256 masked")
    del ref, mag
    assert torch.equal(dx2, ops.conv3x3_dgrad(dz, w, Cin, mask_src=mask_src, bn=128))
    cs = torch.zeros(Cin, device=DEV)
    dx3 = ops.conv3x3_dgrad(dz, w, Cin, mask_src=mask_src, colsum=cs, bn=256)
    assert torch.equal(dx3, dx2)
    stored = dx2.to(torch.float64).reshape(-1, Cin)
    KC.check(cs, stored.sum(0), stored.abs().sum(0), chain=KC.conv_colsum_chain(N * H * W, Cin, KC.sm_count()),
             exact=False, family="conv_colsum", what="bn=256")


@pytest.mark.parametrize("mode", MODES)
@WIDE
def test_wide_wgrad(N, H, W, Cin, Cout, mode):
    ops = _ops()
    g = KC.generator(N * 7 + H + Cin * 3 + Cout + 17, DEV)
    P = N * H * W
    x = KC.operand((N, H, W, Cin), mode, P, g, DEV)
    dz = KC.operand((N, H, W, Cout), mode, P, g, DEV)
    dw = torch.zeros(Cout, 3, 3, Cin, device=DEV)
    ops.conv3x3_wgrad(dz, x, dw, bn=256)
    ref, mag = R.conv3x3_wgrad64(dz, x)
    KC.check(dw, ref, mag, chain=KC.wgrad_chain(N, H, W, Cin, Cout, KC.sm_count(), bn=256), exact=mode == "exact",
             family="conv_wgrad", what="bn=256")
