"""One representative of every class of size-dependent convolution and pooling launch the native engine can make
(conv_space.py: classes at this device's SM count) against the float64 references of ops.ref, in exact and
gauss operand modes.  Outputs sit in guarded buffers prefilled with NaN: every element must be written and
nothing outside the output may change.  Before each convolution launch, conv_plan of its arguments must still
give the representative's class."""
import math
import zlib

import pytest
import torch
import torch.nn.functional as F

import conv_space as S
import kernel_check as KC
from distributed_vgg_f_b200 import ops
from distributed_vgg_f_b200.ops import ref as R
from guarded import NAN, fmax, guarded

pytestmark = pytest.mark.gpu
DEV = "cuda"
MODES = ("exact", "gauss")


def _sms() -> int:
    return KC.sm_count()


def _space():
    """Enumerated only where these tests run: a collection without a device (or without the extension) gets
    no representatives instead of paying for the enumeration."""
    if not (torch.cuda.is_available() and ops.available()):
        return {}, ()
    return S.classes(_sms()), S.representatives(_sms())


CLASSES, REPS = _space()


def _reps(*kinds):
    return [pytest.param(r, id=r.name) for r in REPS if r.launch.kind in kinds]


@pytest.fixture(scope="session", autouse=True)
def coverage_table(pytestconfig):
    """The classes and their representatives, printed once per session."""
    with pytestconfig.pluginmanager.get_plugin("capturemanager").global_and_fixture_disabled():
        print("\n[conv space, %d SMs] %d classes, %d representatives\n%s" %
              (_sms(), len(CLASSES), len(REPS), S.table(CLASSES, REPS)))


def _nhwc(N, H, W, C, dtype=torch.bfloat16, poison=NAN, values=None):
    g = guarded((N, H, W, C), (H * W * C, W * C, C, 1), dtype, 0, poison, DEV, values)
    g.seal()
    return g


def _flat(n, dtype=torch.float32, values=None):
    g = guarded((n,), (1,), dtype, 0, NAN, DEV, values)
    g.seal()
    return g


def _gen(r, mode):
    return KC.generator(zlib.crc32((r.name + mode).encode()), DEV)


def _plan_is(r):
    C = ops.require()
    assert S.signature(C, r.launch, KC.sm_count()) == r.sig, r.name
    return C.conv_plan(r.launch.kind, r.launch.N, r.launch.H, r.launch.W, r.launch.Cin, r.launch.Cout, KC.sm_count())


def _weights(Cout, Cin, mode, g):
    return KC.operand((Cout, 3, 3, Cin), mode, 9 * max(Cin, Cout), g, DEV, scale=1.0 / math.sqrt(9 * Cin))


# ------------------------------------------------------------------------------------------ convolutions
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("r", _reps("fprop"))
def test_fprop(r, mode):
    N, H, W, Cin, Cout = r.launch[1:]
    g = _gen(r, mode)
    x = KC.operand((N, H, W, Cin), mode, 9 * Cin, g, DEV)
    w = _weights(Cout, Cin, mode, g)
    b = KC.bias(Cout, mode, g, DEV)
    y = _nhwc(N, H, W, Cout)
    _plan_is(r)
    ops.require().conv_fprop(x, w, b, y.t, True, 0)
    torch.cuda.synchronize()
    y.check(written=[y.t], what="conv_fprop y")
    ref, mag = R.conv3x3_fprop64(x, w, b, relu=True)
    KC.check(y.t, ref, mag, chain=KC.conv_chain(Cin), exact=mode == "exact", family="conv_fprop", what=r.name)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("r", _reps("fprop_pool"))
def test_fprop_pool_and_unpool(r, mode):
    N, H, W, Cin, Cout = r.launch[1:]
    exact = mode == "exact"
    g = _gen(r, mode)
    x = KC.operand((N, H, W, Cin), mode, 9 * Cin, g, DEV)
    w = _weights(Cout, Cin, mode, g)
    b = KC.bias(Cout, mode, g, DEV)
    OH, OW = H // 2, W // 2
    p = _nhwc(N, OH, OW, Cout)
    m = guarded((N, OH, OW, Cout // 32, 4), (OH * OW * Cout // 8, OW * Cout // 8, Cout // 8, 4, 1), torch.int32, 0,
                -1, DEV)
    m.seal()
    _plan_is(r)
    ops.require().conv_fprop_pool(x, w, b, p.t, m.t, 0)
    torch.cuda.synchronize()
    p.check(written=[p.t], what="conv_fprop_pool pooled")
    m.check(written=[m.t], what="conv_fprop_pool mask")
    ref, mag = R.conv3x3_fprop64(x, w, b, relu=True)
    KC.check_pool(p.t, m.t, ref, mag, chain=KC.conv_chain(Cin), exact=exact, what=r.name)
    del ref, mag
    # its backward: unpool2x2 with the fused column sum
    dp = KC.operand((N, OH, OW, Cout), mode, 1, g, DEV)
    dz = _nhwc(N, H, W, Cout)
    cs = _flat(Cout, values=torch.zeros(Cout, device=DEV))
    ops.unpool2x2(dp, m.t, out=dz.t, colsum=cs.t)
    torch.cuda.synchronize()
    dz.check(written=[dz.t], what="unpool2x2 dz")
    cs.check(written=[cs.t], what="unpool2x2 colsum")
    idx, pos = R.pool_mask_decode(m.t, Cout)
    want, want_cs, cs_mag = R.unpool2x2_64(dp, idx, pos)
    KC.check(dz.t, want, want, chain=0, exact=True, family="unpool2x2", what=r.name)
    KC.check(cs.t, want_cs, cs_mag, chain=KC.unpool_colsum_chain(N * OH * OW, Cout, KC.sm_count()), exact=False,
             family="unpool_colsum", what=r.name)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("r", _reps("dgrad"))
def test_dgrad(r, mode):
    """Plain, masked (the ReLU backward of the layer below) and masked with the fused column sum."""
    N, H, W, Cin, Cout = r.launch[1:]
    exact = mode == "exact"
    g = _gen(r, mode)
    dz = KC.operand((N, H, W, Cout), mode, 9 * Cout, g, DEV)
    w = _weights(Cout, Cin, mode, g)
    mask_src = KC.operand((N, H, W, Cin), "gauss", 1, g, DEV)
    plan = _plan_is(r)
    chain = KC.conv_chain(Cout)
    for masked, colsum in ((False, False), (True, False), (True, True)):
        what = "%s%s %s" % ("masked" if masked else "plain", " + colsum" if colsum else "", r.name)
        dx = _nhwc(N, H, W, Cin)
        cs = _flat(Cin, values=torch.zeros(Cin, device=DEV)) if colsum else None
        ops.require().conv_dgrad(dz, w, mask_src if masked else None, dx.t, cs.t if colsum else None, 0)
        torch.cuda.synchronize()
        dx.check(written=[dx.t], what="conv_dgrad dx " + what)
        ref, mag = R.conv3x3_dgrad64(dz, w, mask_src=mask_src if masked else None)
        KC.check(dx.t, ref, mag, chain=chain, exact=exact, family="conv_dgrad", what=what)
        if colsum:
            cs.check(written=[cs.t], what="conv_dgrad colsum")
            stored = dx.t.to(torch.float64).reshape(-1, Cin)
            tiles = plan["tiles"] * -(-Cin // 64)
            KC.check(cs.t, stored.sum(0), stored.abs().sum(0),
                     chain=KC.conv_colsum_chain(N * H * W, Cin, KC.sm_count(), tiles=tiles), exact=False,
                     family="conv_colsum", what=what)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("r", _reps("wgrad", "wgrad_partial"))
def test_wgrad(r, mode):
    """wgrad: the atomic split-K kernel, accumulating onto dw; wgrad_partial: conv3x3_wgrad_det (every split's
    partials in its own workspace slice, added in split order), overwriting dw."""
    kind, N, H, W, Cin, Cout = r.launch
    g = _gen(r, mode)
    P = N * H * W
    x = KC.operand((N, H, W, Cin), mode, P, g, DEV)
    dz = KC.operand((N, H, W, Cout), mode, P, g, DEV)
    plan = _plan_is(r)
    n = Cout * 9 * Cin
    ref, mag = R.conv3x3_wgrad64(dz, x)
    if kind == "wgrad":
        dw0 = KC.bias(n, mode, g, DEV)
        dw = _flat(n, values=dw0)
        ops.require().conv_wgrad(dz, x, dw.t.view(Cout, 3, 3, Cin), 1.0, 0, 0)
        ref, mag = ref + dw0.double().view_as(ref), mag + dw0.double().abs().view_as(mag)
    else:
        dw = _flat(n)
        ws = _flat(plan["ksplit"] * ops.require().workspace_slice(n))
        splits = ops.conv3x3_wgrad_det(dz, x, dw.t.view(Cout, 3, 3, Cin), ws.t)
        assert splits == plan["ksplit"]
        torch.cuda.synchronize()
        ws.check(written=[ws.t], what="conv3x3_wgrad_partial workspace")
    torch.cuda.synchronize()
    dw.check(written=[dw.t], what=kind + " dw")
    KC.check(dw.t.view(Cout, 3, 3, Cin), ref, mag, chain=KC.wgrad_chain(N, H, W, Cin, Cout, KC.sm_count(), kind) + 1,
             exact=mode == "exact", family="conv_wgrad", what=r.name)


# ------------------------------------------------------------------------------------------ first layer
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("r", _reps("conv0_fprop", "conv0_wgrad"))
def test_conv0(r, mode):
    """conv0_fprop; conv0_wgrad atomic (onto a non-zero dw) and reproducible (partials + ordered reduce)."""
    kind, N, H, W = r.launch[:4]
    exact = mode == "exact"
    g = _gen(r, mode)
    C = ops.require()
    x4 = torch.zeros(N, H, W, 4, dtype=torch.bfloat16, device=DEV)
    if kind == "conv0_fprop":
        x4[..., :3] = KC.operand((N, H, W, 3), mode, 27, g, DEV)
        w0 = torch.zeros(64, 64, dtype=torch.bfloat16, device=DEV)
        w0[:, :27] = KC.operand((64, 27), mode, 27, g, DEV, scale=0.2)
        bias = KC.bias(64, mode, g, DEV)
        y = _nhwc(N, H, W, 64)
        C.conv0_fprop(x4, w0, bias, y.t)
        torch.cuda.synchronize()
        y.check(written=[y.t], what="conv0_fprop y")
        ref, mag = R.conv0_fprop64(x4, w0, bias)
        KC.check(y.t, ref, mag, chain=KC.gemm_chain(64), exact=exact, family="conv0_fprop", what=r.name)
        return
    P = N * H * W
    x4[..., :3] = KC.operand((N, H, W, 3), mode, P, g, DEV)
    dz = KC.operand((N, H, W, 64), mode, P, g, DEV)
    ref, mag = R.conv0_wgrad64(dz, x4)
    chain = KC.conv0_wgrad_chain(P, KC.sm_count()) + 1
    dw0 = KC.bias(64 * 64, mode, g, DEV)
    dw = _flat(64 * 64, values=dw0)
    C.conv0_wgrad(dz, x4, dw.t.view(64, 64))
    torch.cuda.synchronize()
    dw.check(written=[dw.t], what="conv0_wgrad dw")
    KC.check(dw.t.view(64, 64), ref + dw0.double().view(64, 64), mag + dw0.double().abs().view(64, 64), chain=chain,
             exact=exact, family="conv0_wgrad", what=r.name)
    splits = C.conv0_wgrad_splits(N, H, W, KC.sm_count())
    dw = _flat(64 * 64)
    ws = _flat(splits * C.workspace_slice(64 * 64))
    assert ops.conv0_wgrad_det(dz, x4, dw.t.view(64, 64), ws.t) == splits
    torch.cuda.synchronize()
    dw.check(written=[dw.t], what="conv0_wgrad_det dw")
    ws.check(written=[ws.t], what="conv0_wgrad_partial workspace")
    KC.check(dw.t.view(64, 64), ref, mag, chain=chain, exact=exact, family="conv0_wgrad", what="det " + r.name)


# ------------------------------------------------------------------------------------------ pooling
@pytest.mark.parametrize("r", _reps("maxpool_fwd", "maxpool_relu_bwd", "unpool"))
def test_maxpool(r):
    """Post-ReLU integer maps (ties and zeros, exact in bf16 and in every sum): floor-mode forward against
    float64 max_pool2d; the ReLU backward (with and without its column sum) and unpool2x2 against the
    first-maximum routing of ops.ref."""
    kind, N, H, W, _, C = r.launch
    g = _gen(r, "exact")
    OH, OW = H // 2, W // 2
    vals = torch.relu(torch.randint(-2, 3, (N, H, W, C), device=DEV, generator=g)).to(torch.bfloat16)
    dpv = torch.randint(-3, 4, (N, OH, OW, C), device=DEV, generator=g).to(torch.bfloat16)
    if kind == "maxpool_fwd":
        y = _nhwc(N, H, W, C, poison=fmax(torch.bfloat16), values=vals)
        p = _nhwc(N, OH, OW, C)
        ops.maxpool2x2(y.t, out=p.t)
        torch.cuda.synchronize()
        y.check(what="maxpool_fwd y")
        p.check(written=[p.t], what="maxpool_fwd out")
        assert torch.equal(p.t.double(), F.max_pool2d(vals.double().permute(0, 3, 1, 2), 2, 2).permute(0, 2, 3, 1))
        return
    if kind == "unpool":
        idx = torch.randint(0, 4, (N, OH, OW, C), device=DEV, generator=g)
        pos = torch.randint(0, 2, (N, OH, OW, C), device=DEV, generator=g).bool()
        mask = R.pool_mask_encode(idx, pos)
        want, want_cs, cs_mag = R.unpool2x2_64(dpv, idx, pos)
    else:
        want, want_cs, cs_mag = R.maxpool2x2_relu_bwd64(vals, dpv)
    for colsum in (False, True):
        dz = _nhwc(N, H, W, C)
        cs = _flat(C, values=torch.zeros(C, device=DEV)) if colsum else None
        if kind == "unpool":
            ops.unpool2x2(dpv, mask, out=dz.t, colsum=cs.t if colsum else None)
        else:
            ops.maxpool2x2_relu_bwd(vals, dpv, out=dz.t, colsum=cs.t if colsum else None)
        torch.cuda.synchronize()
        dz.check(written=[dz.t], what=kind + " dz")
        KC.check(dz.t, want, want, chain=0, exact=True, family=kind, what=r.name)
        if colsum:
            cs.check(written=[cs.t], what=kind + " colsum")
            KC.check(cs.t, want_cs, cs_mag, chain=0, exact=True, family=kind + "_colsum", what=r.name)


def _avg_exact(H: int) -> bool:
    """Every window of H -> 7 has a power-of-two size, so 1/size and the mean are exact."""
    return all((b - a) & (b - a - 1) == 0 for a, b in R._ap_windows(H, 7))


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("r", _reps("avgpool_fwd", "avgpool_bwd"))
def test_adaptive_avgpool(r, mode):
    kind, N, H, W, _, C = r.launch
    if mode == "exact" and not _avg_exact(H):
        pytest.skip("window sizes that are not powers of two: their reciprocals are not exact")
    exact = mode == "exact"
    g = _gen(r, mode)
    if kind == "avgpool_fwd":
        x = KC.operand((N, H, W, C), mode, 16, g, DEV)
        y = _nhwc(N, 7, 7, C)
        ops.adaptive_avgpool(x, 7, 7, out=y.t)
        torch.cuda.synchronize()
        y.check(written=[y.t], what="avgpool_fwd y")
        ref, mag = R.adaptive_avgpool64(x, 7, 7)
        KC.check(y.t, ref, mag, chain=KC.avgpool_chain(R.ap_max_window(H, 7) ** 2), exact=exact, family="avgpool_fwd",
                 what=r.name)
        return
    dy = KC.operand((N, 7, 7, C), mode, 16, g, DEV)
    dx = _nhwc(N, H, W, C)
    ops.adaptive_avgpool_bwd(dy, H, W, out=dx.t)
    torch.cuda.synchronize()
    dx.check(written=[dx.t], what="avgpool_bwd dx")
    ref, mag = R.adaptive_avgpool_bwd64(dy, H, W)
    KC.check(dx.t, ref, mag, chain=KC.avgpool_chain(R.ap_max_cover(H, 7) ** 2), exact=exact, family="avgpool_bwd",
             what=r.name)
