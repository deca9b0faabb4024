"""Evidence, without a GPU, that the kernel tests have teeth.

1. The float64 references of ops.ref agree with torch's own float64 conv2d, autograd and max_pool2d.
2. An emulated kernel (fp32 accumulation of bf16 operands in 64-deep k-blocks, optional split-K,
   bf16 round-to-nearest-even) passes the per-element criterion of kernel_check in both input modes,
   and each typical kernel defect planted into its output fails it.
"""
import pytest
import torch
import torch.nn.functional as F

import kernel_check as KC
from distributed_vgg_f_b200.ops import ref as R

MODES = ["exact", "gauss"]
CPU = torch.device("cpu")
F64 = torch.float64


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _nchw(t):
    return t.to(F64).permute(0, 3, 1, 2)


def _nhwc(t):
    return t.permute(0, 2, 3, 1)


# ------------------------------------------------------------------- references vs torch float64
@pytest.mark.parametrize("a_mn,b_mn,epi", [(False, False, "f32_atomic_t"), (True, False, "f32_store_t"),
                                           (True, True, "f32_store"), (True, True, "bf16_store"),
                                           (False, False, "bf16_bias_relu"), (True, True, "f32_atomic")])
def test_gemm64_matches_matmul(a_mn, b_mn, epi):
    g = _gen(0)
    M, N, K = 13, 7, 21
    A = torch.randn(K + 3, M + 5, generator=g) if a_mn else torch.randn(M + 2, K + 6, generator=g)
    B = torch.randn(K + 1, N + 4, generator=g) if b_mn else torch.randn(N + 3, K + 2, generator=g)
    bias = torch.randn(N + 9, generator=g)
    ref, mag = R.gemm64(A, B, M=M, N=N, K=K, a_mn=a_mn, b_mn=b_mn, epi=epi, bias=bias, alpha=-0.5)
    a = (A[:K, :M].t() if a_mn else A[:M, :K]).to(F64)
    b = (B[:K, :N].t() if b_mn else B[:N, :K]).to(F64)
    want = torch.relu(a @ b.t() + bias[:N].to(F64)) if epi == "bf16_bias_relu" else -0.5 * (a @ b.t())
    want_mag = (a.abs() @ b.abs().t() + bias[:N].to(F64).abs()) if epi == "bf16_bias_relu" else 0.5 * (a.abs() @ b.abs().t())
    if epi.endswith("_t"):
        want, want_mag = want.t(), want_mag.t()
    torch.testing.assert_close(ref, want, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(mag, want_mag, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("N,H,W,Cin,Cout", [(2, 5, 7, 8, 6), (1, 1, 3, 4, 4), (3, 4, 4, 3, 5)])
def test_conv_references_match_torch(N, H, W, Cin, Cout):
    g = _gen(1)
    x = torch.randn(N, H, W, Cin, generator=g, dtype=F64)
    w = torch.randn(Cout, 3, 3, Cin, generator=g, dtype=F64)
    b = torch.randn(Cout, generator=g, dtype=F64)
    dz = torch.randn(N, H, W, Cout, generator=g, dtype=F64)
    mask_src = torch.randn(N, H, W, Cin, generator=g)
    xr = _nchw(x).requires_grad_(True)
    wr = _nchw(w).requires_grad_(True)
    z = F.conv2d(xr, wr, None, padding=1)
    z.backward(_nchw(dz))
    y, ymag = R.conv3x3_fprop64(x, w, b, relu=True)
    torch.testing.assert_close(y, _nhwc(torch.relu(z.detach() + b.view(1, -1, 1, 1))))
    torch.testing.assert_close(ymag, _nhwc(F.conv2d(_nchw(x).abs(), _nchw(w).abs(), b.abs(), padding=1)))
    dx, dxmag = R.conv3x3_dgrad64(dz, w)
    torch.testing.assert_close(dx, _nhwc(xr.grad))
    dxm, _ = R.conv3x3_dgrad64(dz, w, mask_src=mask_src)
    torch.testing.assert_close(dxm, _nhwc(xr.grad) * (mask_src > 0))
    torch.testing.assert_close(dxmag, _nhwc(F.conv_transpose2d(_nchw(dz).abs(), _nchw(w).abs(), padding=1)))
    dw, _ = R.conv3x3_wgrad64(dz, x, scale=0.5)
    torch.testing.assert_close(dw, 0.5 * wr.grad.permute(0, 2, 3, 1))


def test_conv0_references_match_torch():
    g = _gen(2)
    N, H, W = 2, 6, 5
    x4 = torch.randn(N, H, W, 4, generator=g, dtype=F64)
    w0 = torch.randn(64, 64, generator=g, dtype=F64)
    b = torch.randn(64, generator=g, dtype=F64)
    dz = torch.randn(N, H, W, 64, generator=g, dtype=F64)
    wr = w0[:, :27].reshape(64, 3, 3, 3).permute(0, 3, 1, 2).clone().requires_grad_(True)
    z = F.conv2d(_nchw(x4[..., :3]), wr, None, padding=1)
    z.backward(_nchw(dz))
    y, _ = R.conv0_fprop64(x4, w0, b)
    torch.testing.assert_close(y, _nhwc(torch.relu(z.detach() + b.view(1, -1, 1, 1))))
    dw0, _ = R.conv0_wgrad64(dz, x4)
    torch.testing.assert_close(dw0[:, :27], wr.grad.permute(0, 2, 3, 1).reshape(64, 27))
    assert torch.count_nonzero(dw0[:, 27:]) == 0


def test_pool_references_match_torch():
    g = _gen(3)
    y = torch.relu(torch.randint(-2, 4, (2, 6, 8, 64), generator=g).to(F64))     # integer data: many ties
    val, idx, pos = R.pool2x2_select(y)
    p, ind = F.max_pool2d(_nchw(y), 2, 2, return_indices=True)
    torch.testing.assert_close(val, _nhwc(p))
    # torch's flat index h*W + w  ->  window position (h % 2) * 2 + (w % 2): its first maximum rule
    W = y.shape[2]
    torch.testing.assert_close(idx, _nhwc((ind // W % 2) * 2 + ind % W % 2))
    assert torch.equal(pos, val > 0)
    # the mask words round-trip, and unpool is the backward of relu -> max_pool2d
    mask = R.pool_mask_encode(idx, pos)
    i2, p2 = R.pool_mask_decode(mask, 64)
    assert torch.equal(i2, idx) and torch.equal(p2, pos)
    dp = torch.randn(val.shape, generator=g, dtype=F64)
    dz, cs, csmag = R.unpool2x2_64(dp, idx, pos)
    want = _nhwc(R.pool_relu_bwd(_nchw(y), _nchw(dp)))
    torch.testing.assert_close(dz, want)
    torch.testing.assert_close(cs, want.sum((0, 1, 2)))
    torch.testing.assert_close(csmag, want.abs().sum((0, 1, 2)))


# ------------------------------------------------------------------------------ emulated kernels
def _emu_gemm(A, B, ksplit=1, drop_block=None, double_split=None):
    """fp32 accumulation of bf16 A [M][K] x B [N][K]^T in 64-deep k-blocks, split-K partials added
    in fp32; optionally without one k-block or with one split's partial added twice."""
    M, K = A.shape
    iters = -(-K // 64)
    per = -(-iters // ksplit)
    out = torch.zeros(M, B.shape[0])
    for s in range(0, iters, per):
        acc = torch.zeros(M, B.shape[0])
        for kb in range(s, min(s + per, iters)):
            if kb == drop_block:
                continue
            acc += A[:, kb * 64:(kb + 1) * 64].float() @ B[:, kb * 64:(kb + 1) * 64].float().t()
        out += acc
        if s // per == double_split:
            out += acc
    return out


def _emu_conv(x, w, b, skip_tap_border=False):
    """fp32 conv fprop as the kernel does it (tap by tap, 64-channel k-blocks), + bias, ReLU, bf16 RNE.
    skip_tap_border: tap (0, 1) is left out on the last image row only."""
    N, H, W, Cin = x.shape
    acc = torch.zeros(N * H * W, w.shape[0])
    xp = torch.zeros(N, H + 2, W + 2, Cin, dtype=x.dtype)
    xp[:, 1:H + 1, 1:W + 1] = x
    last_row = (torch.arange(H).view(1, H, 1).expand(N, H, W) == H - 1).reshape(-1, 1)
    for kh in range(3):
        for kw in range(3):
            xs = xp[:, kh:kh + H, kw:kw + W].reshape(-1, Cin).float()
            part = torch.zeros_like(acc)
            for c in range(0, Cin, 64):
                part += xs[:, c:c + 64] @ w[:, kh, kw, c:c + 64].float().t()
            if skip_tap_border and (kh, kw) == (0, 1):
                part = part * ~last_row
            acc += part
    return torch.relu(acc + b).view(N, H, W, -1)


def _trunc_bf16(t):
    """bf16 by truncation (round toward zero) instead of RNE."""
    return (t.float().view(torch.int32) & ~0xFFFF).view(torch.float32).to(torch.bfloat16)


def _rejects(fn):
    with pytest.raises(AssertionError):
        fn()


@pytest.mark.parametrize("mode", MODES)
def test_gemm_criterion_passes_emulation_and_catches_defects(mode):
    g = _gen(10)
    M, N, K = 200, 40, 1000                        # ragged M tile (128 + 72), ragged N tile (32 + 8), K tail
    A = KC.operand((M, K), mode, K, g, CPU)
    B = KC.operand((N, K), mode, K, g, CPU)
    ref, mag = R.gemm64(A, B, M=M, N=N, K=K)
    exact = mode == "exact"
    chain = KC.gemm_chain(K, 4)
    KC.check(_emu_gemm(A, B, ksplit=4), ref, mag, chain=chain, exact=exact)
    KC.check(_emu_gemm(A, B, ksplit=1).to(torch.bfloat16), ref, mag, chain=KC.gemm_chain(K), exact=exact)
    _rejects(lambda: KC.check(_emu_gemm(A, B, ksplit=4, drop_block=7), ref, mag, chain=chain, exact=exact))
    _rejects(lambda: KC.check(_emu_gemm(A, B, ksplit=4, double_split=3), ref, mag, chain=chain, exact=exact))
    out = _emu_gemm(A, B, ksplit=4)
    for tail in ((slice(128, None), slice(None)), (slice(None), slice(32, None))):
        bad = out.clone()
        bad[tail] = 0                              # the last ragged M tile / N tile never written
        _rejects(lambda: KC.check(bad, ref, mag, chain=chain, exact=exact))


@pytest.mark.parametrize("mode", MODES)
def test_conv_criterion_passes_emulation_and_catches_defects(mode):
    g = _gen(11)
    N, H, W, Cin, Cout = 2, 6, 10, 128, 96
    exact = mode == "exact"
    x = KC.operand((N, H, W, Cin), mode, 9 * Cin, g, CPU)
    w = KC.operand((Cout, 3, 3, Cin), mode, 9 * Cin, g, CPU, scale=0.1)
    b = KC.bias(Cout, mode, g, CPU)
    ref, mag = R.conv3x3_fprop64(x, w, b)
    chain = KC.conv_chain(Cin)
    good = _emu_conv(x, w, b)
    KC.check(good.to(torch.bfloat16), ref, mag, chain=chain, exact=exact)
    _rejects(lambda: KC.check(_emu_conv(x, w, b, skip_tap_border=True).to(torch.bfloat16), ref, mag,
                              chain=chain, exact=exact))
    shifted = good.clone()
    shifted[..., 64:95] = good[..., 65:96]         # the last 32-channel chunk one channel off
    _rejects(lambda: KC.check(shifted.to(torch.bfloat16), ref, mag, chain=chain, exact=exact))
    _rejects(lambda: KC.check(_trunc_bf16(good), ref, mag, chain=chain, exact=exact))


@pytest.mark.parametrize("mode", MODES)
def test_wgrad_criterion_catches_a_missing_pixel_block(mode):
    g = _gen(12)
    N, H, W, C = 4, 8, 16, 64
    exact = mode == "exact"
    P = N * H * W
    dz = KC.operand((N, H, W, C), mode, P, g, CPU)
    x = KC.operand((N, H, W, C), mode, P, g, CPU)
    ref, mag = R.conv3x3_wgrad64(dz, x)
    # emulation: the pixel reduction in 64-pixel k-blocks per tap, fp32
    A = dz.reshape(P, C)
    taps = list(R._taps(x))
    chain = KC.wgrad_chain(N, H, W, C, C, sms=132)

    def emu(drop=None):
        out = torch.zeros(C, 3, 3, C)
        for kh, kw, xs in taps:
            out[:, kh, kw] = _emu_gemm(A.t().contiguous(), xs.t().to(torch.bfloat16).contiguous(),
                                       drop_block=drop)
        return out

    KC.check(emu(), ref, mag, chain=chain, exact=exact)
    _rejects(lambda: KC.check(emu(drop=3), ref, mag, chain=chain, exact=exact))


@pytest.mark.parametrize("mode", MODES)
def test_pool_criterion_passes_emulation_and_catches_defects(mode):
    g = _gen(13)
    N, H, W, Cin, Cout = 2, 8, 12, 64, 64
    exact = mode == "exact"
    x = KC.operand((N, H, W, Cin), mode, 9 * Cin, g, CPU)
    w = KC.operand((Cout, 3, 3, Cin), mode, 9 * Cin, g, CPU, scale=0.1)
    b = KC.bias(Cout, mode, g, CPU)
    ref, mag = R.conv3x3_fprop64(x, w, b)
    chain = KC.conv_chain(Cin)
    y = _emu_conv(x, w, b).to(torch.bfloat16)                 # what the epilogue rounds before pooling
    val, idx, pos = R.pool2x2_select(y.float())
    KC.check_pool(val.to(torch.bfloat16), R.pool_mask_encode(idx, pos), ref, mag, chain=chain, exact=exact)
    # truncating instead of rounding before the max
    tv, _, _ = R.pool2x2_select(_trunc_bf16(_emu_conv(x, w, b)).float())
    _rejects(lambda: KC.check_pool(tv.to(torch.bfloat16), R.pool_mask_encode(idx, pos), ref, mag, chain=chain,
                                   exact=exact))
    # "max > 0" bit dropped in one chunk
    _rejects(lambda: KC.check_pool(val.to(torch.bfloat16), R.pool_mask_encode(idx, pos & (torch.arange(Cout) < 32)),
                                   ref, mag, chain=chain, exact=exact))
    # argmax ties resolved last-first: integer data ties often; Gaussian windows that tie are not judged
    win = R.pool_windows(y.float())
    last = 3 - win.flip(-1).argmax(-1)
    ties = bool(((last != idx) & pos).any())
    if exact:
        assert ties
        _rejects(lambda: KC.check_pool(val.to(torch.bfloat16), R.pool_mask_encode(last, pos), ref, mag,
                                       chain=chain, exact=exact))
    # a wrong argmax where the window is clear-cut fails in both modes
    wrong = torch.where(pos, (idx + 1) % 4, idx)
    _rejects(lambda: KC.check_pool(val.to(torch.bfloat16), R.pool_mask_encode(wrong, pos), ref, mag, chain=chain,
                                   exact=exact))


def test_exact_mode_sums_are_fp32_integers():
    """The premise of exact mode: at the deepest reductions the kernels run, every partial sum of
    integer operands stays an integer below 2^24, so fp32 adds them exactly in any order."""
    assert 16 * KC.EXACT_DEPTH < 2 ** 24                    # conv fprop / dgrad (9 x 512), FC dgrad
    assert 64 * 224 * 224 < 2 ** 24                         # pixel-depth wgrad at batch 64, {-1, 0, 1}
    assert 25088 < 2 ** 24                                  # FC1 forward, {-1, 0, 1}
    g = _gen(14)
    a = KC.operand((4, 25088), "exact", 25088, g, CPU)
    assert set(a.float().unique().tolist()) <= {-1.0, 0.0, 1.0}
    a = KC.operand((4, 4608), "exact", 4608, g, CPU)
    assert float(a.float().abs().max()) <= 4
