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
from distributed_vgg_f_b200 import ops
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
    chain = KC.split_chain(1, 8)     # wgrad_halo64 at 132 SMs: 8 pixel tiles, one per split (next test)

    def emu(drop=None):
        out = torch.zeros(C, 3, 3, C)
        for kh, kw, xs in taps:
            out[:, kh, kw] = _emu_gemm(A.t().contiguous(), xs.t().to(torch.bfloat16).contiguous(),
                                       drop_block=drop)
        return out

    KC.check(emu(), ref, mag, chain=chain, exact=exact)
    _rejects(lambda: KC.check(emu(drop=3), ref, mag, chain=chain, exact=exact))


@pytest.mark.skipif(not ops.available(), reason="needs the built extension (host code only)")
def test_wgrad_chain_is_the_planned_split():
    """The split the criterion above assumes is the one the launcher plans for that shape."""
    p = ops.require().conv_plan("wgrad", 4, 8, 16, 64, 64, 132)
    assert (p["path"], p["tiles_per_split"], p["ksplit"]) == ("wgrad_halo64", 1, 8)
    assert KC.wgrad_chain(4, 8, 16, 64, 64, 132) == KC.split_chain(1, 8)


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


# ========================================================= memory-bound kernels: references vs torch
def test_philox_known_answers():
    """Random123's known-answer vectors of Philox4x32-10."""
    kat = [((0, 0), (0, 0, 0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
           ((0xffffffff, 0xffffffff), (0xffffffff,) * 4, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
           ((0xa4093822, 0x299f31d0), (0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344),
            (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]
    for key, ctr, want in kat:
        got = tuple(int(w) for w in R.philox4x32_10(key, ctr))
        assert got == want, [hex(v) for v in got]


def test_dropout_mask_layout():
    """Element 4q + j of the flattened [B][N] uses word j of quad q, counter (q, offset); fp32 p."""
    seed, offset, B, N, p = (1 << 33) + 12345, (1 << 32) + 1, 3, 10, 0.6
    keep, ks = R.dropout_mask64(seed, offset, B, N, p)
    for i in (0, 5, 7, 29):
        q, j = divmod(i, 4)
        w = R.philox4x32_10((seed & 0xFFFFFFFF, seed >> 32), (q, 0, offset & 0xFFFFFFFF, offset >> 32))[j]
        u = (int(w) >> 8) / 2 ** 24
        assert bool(keep.view(-1)[i]) == (not u < float(torch.tensor(p, dtype=torch.float32)))
    assert ks == float(torch.tensor(1.0) / (torch.tensor(1.0) - torch.tensor(0.6)))
    assert ks != 2.5                                      # fp32 1 / (1 - 0.6f) is 2.5000002
    big, _ = R.dropout_mask64(seed, offset, 64, N, p)
    assert torch.equal(big[:B], keep)                     # a row's mask does not depend on the batch size
    frac = 1 - float(R.dropout_mask64(7, 1, 64, 4096, 0.5)[0].float().mean())
    assert 0.49 < frac < 0.51


def test_maxpool_references_match_torch():
    g = _gen(20)
    y = torch.relu(torch.randint(-2, 3, (2, 6, 8, 16), generator=g).to(F64))      # ties and all-zero windows
    val, idx = R.maxpool2x2_64(y)
    p, ind = F.max_pool2d(_nchw(y), 2, 2, return_indices=True)
    torch.testing.assert_close(val, _nhwc(p))
    W = y.shape[2]
    assert torch.equal(idx, _nhwc((ind // W % 2) * 2 + ind % W % 2))
    dp = torch.randn(val.shape, generator=g, dtype=F64)
    dz, cs, csmag = R.maxpool2x2_relu_bwd64(y, dp)
    yr = _nchw(y).clone().requires_grad_(True)
    F.max_pool2d(yr, 2, 2).backward(_nchw(dp))
    want = _nhwc(yr.grad * (yr > 0))
    torch.testing.assert_close(dz, want)
    torch.testing.assert_close(cs, want.sum((0, 1, 2)))
    torch.testing.assert_close(csmag, want.abs().sum((0, 1, 2)))


@pytest.mark.parametrize("H", [2, 4, 5, 7, 10, 14])
def test_avgpool_references_match_torch(H):
    g = _gen(21)
    x = torch.randn(2, H, H + 1, 8, generator=g, dtype=F64)
    ref, mag = R.adaptive_avgpool64(x, 7, 7)
    xr = _nchw(x).clone().requires_grad_(True)
    y = F.adaptive_avg_pool2d(xr, (7, 7))
    torch.testing.assert_close(ref, _nhwc(y.detach()))
    torch.testing.assert_close(mag, _nhwc(F.adaptive_avg_pool2d(_nchw(x).abs(), (7, 7))))
    dy = torch.randn(ref.shape, generator=g, dtype=F64)
    y.backward(_nchw(dy))
    dx, _ = R.adaptive_avgpool_bwd64(dy, H, H + 1)
    torch.testing.assert_close(dx, _nhwc(xr.grad))


@pytest.mark.parametrize("weighted", [False, True])
def test_cross_entropy_reference_matches_torch(weighted):
    g = _gen(22)
    B, C = 9, 5
    z = torch.randn(B, C, generator=g, dtype=F64) * 3
    z[0, 1] = z[0, 3] = z[0].max() + 1                      # a tie for the argmax: the lower index wins
    t = torch.randint(0, C, (B,), generator=g)
    t[0] = 1
    w = torch.rand(C, generator=g, dtype=F64) + 0.1 if weighted else None
    out = R.cross_entropy64(z, t, ldd=8, class_weights=w, grad_scale=0.125 if not weighted else None)
    zr = z.clone().requires_grad_(True)
    loss = F.cross_entropy(zr, t, weight=w)
    loss.backward()
    torch.testing.assert_close(out["loss"], loss.detach())
    scale = 1.0 if weighted else 0.125 * B                  # torch's gradient is that of the mean: 1/B
    torch.testing.assert_close(out["dlogits"][:, :C], zr.grad * scale)
    assert torch.count_nonzero(out["dlogits"][:, C:]) == 0
    assert float(out["meter"][1]) == float((torch.argmax(z, 1) == t).sum()) and float(out["meter"][2]) == B
    assert float(out["meter"][1]) >= 1                       # row 0's tie counted as correct


def test_optimizer_references_match_torch():
    g = _gen(23)
    n = 64
    p0 = torch.randn(n, generator=g, dtype=F64)
    hp = dict(lr=1e-2, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.05)
    pr = p0.clone().requires_grad_(True)
    opt = torch.optim.Adam([pr], lr=hp["lr"], betas=(hp["beta1"], hp["beta2"]), eps=hp["eps"],
                           weight_decay=hp["weight_decay"])
    p, m, v = p0.clone(), torch.zeros(n, dtype=F64), torch.zeros(n, dtype=F64)
    for step in range(1, 5):
        gr = torch.randn(n, generator=g, dtype=F64)
        out = R.adam_step64(p, m, v, gr * 8, step=step, grad_scale=0.125, **hp)
        p, m, v = out["p"][0], out["m"][0], out["v"][0]
        pr.grad = gr.clone()
        opt.step()
        torch.testing.assert_close(p, pr.detach(), rtol=1e-12, atol=1e-12)
        torch.testing.assert_close(m, opt.state[pr]["exp_avg"], rtol=1e-12, atol=1e-12)
        torch.testing.assert_close(v, opt.state[pr]["exp_avg_sq"], rtol=1e-12, atol=1e-12)
    for momentum in (0.9, 0.0):
        pr = p0.clone().requires_grad_(True)
        opt = torch.optim.SGD([pr], lr=0.1, momentum=momentum, weight_decay=0.01)
        p, buf = p0.clone(), torch.zeros(n, dtype=F64)
        for step in range(3):
            gr = torch.randn(n, generator=g, dtype=F64)
            out = R.sgd_step64(p, buf, gr, lr=0.1, momentum=momentum, weight_decay=0.01, first=step == 0)
            p, buf = out["p"][0], out["buf"][0]
            pr.grad = gr.clone()
            opt.step()
            torch.testing.assert_close(p, pr.detach(), rtol=1e-12, atol=1e-12)


def test_nchw_to_nhwc_reference():
    x = torch.randn(2, 3, 4, 5, generator=_gen(24))
    y, _ = R.nchw_to_nhwc64(x, 8)
    torch.testing.assert_close(y[..., :3], x.to(F64).permute(0, 2, 3, 1))
    assert torch.count_nonzero(y[..., 3:]) == 0


# ============================================= memory-bound kernels: emulations and planted defects
def _emu_pool_bwd(y, dp, last=False):
    """maxpool2x2_relu_bwd: first (or, planted, last) maximum of each window gets dp where max > 0."""
    win = R.pool_windows(y.float())
    val = win.amax(-1)
    idx = 3 - win.flip(-1).argmax(-1) if last else R._first_max(win)[1]
    dz, _, _ = R.unpool2x2_64(dp, idx, val > 0)
    return dz.to(torch.bfloat16)


def test_pool_bwd_criterion_catches_last_maximum_ties():
    g = _gen(30)
    y = torch.relu(torch.randint(-2, 3, (2, 8, 8, 16), generator=g)).to(torch.bfloat16)
    dp = KC.operand((2, 4, 4, 16), "exact", 1, g, CPU)
    ref, _, _ = R.maxpool2x2_relu_bwd64(y, dp)
    KC.check(_emu_pool_bwd(y, dp), ref, ref.abs(), chain=0, exact=True)
    _rejects(lambda: KC.check(_emu_pool_bwd(y, dp, last=True), ref, ref.abs(), chain=0, exact=True))


def _emu_avgpool(x, OH, floor_end=False):
    N, H, W, C = x.shape
    out = torch.zeros(N, OH, OH, C)
    for oh in range(OH):
        h0, h1 = oh * H // OH, ((oh + 1) * H if floor_end else (oh + 1) * H + OH - 1) // OH
        for ow in range(OH):
            w0, w1 = ow * W // OH, ((ow + 1) * W if floor_end else (ow + 1) * W + OH - 1) // OH
            acc = torch.zeros(N, C)
            for h in range(h0, h1):
                for w in range(w0, w1):
                    acc += x[:, h, w].float()
            out[:, oh, ow] = acc * (1.0 / float(max((h1 - h0) * (w1 - w0), 1)))
    return out.to(torch.bfloat16)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("H", [5, 10])
def test_avgpool_criterion_catches_ap_end_without_ceiling(mode, H):
    g = _gen(31)
    x = KC.operand((2, H, H, 8), mode, 9, g, CPU)
    ref, mag = R.adaptive_avgpool64(x, 7, 7)
    chain = KC.avgpool_chain(R.ap_max_window(H, 7) ** 2)
    exact = mode == "exact" and H == 5                 # window sizes 1, 2, 4: powers of two
    KC.check(_emu_avgpool(x, 7), ref, mag, chain=chain, exact=exact)
    _rejects(lambda: KC.check(_emu_avgpool(x, 7, floor_end=True), ref, mag, chain=chain, exact=exact))


def _emu_bias_grad(dz, C, scale, sms, drop_block=None):
    """bias_grad's block split (elementwise.cu): blocks of rows_per_block rows summed in fp32,
    added atomically; optionally one block left out."""
    rows = dz.shape[0]
    c8 = C // 8
    CG = min(c8, 256)
    RL = max(256 // CG, 1)
    nblk = max(min(-(-rows // (RL * 16)), sms * 8 // -(-c8 // CG)), 1)
    rpb = -(-rows // nblk)
    db = torch.zeros(C)
    for b, r0 in enumerate(range(0, rows, rpb)):
        if b != drop_block:
            db += dz[r0:r0 + rpb, :C].float().sum(0) * scale
    return db


@pytest.mark.parametrize("mode", MODES)
def test_bias_grad_criterion_catches_a_dropped_row_block(mode):
    g = _gen(32)
    rows, C, sms = 20000, 64, 132
    dz = KC.operand((rows, C), mode, rows, g, CPU)
    ref, mag = R.bias_grad64(dz, C, 0.5)
    chain = KC.bias_grad_chain(rows, C, sms)
    exact = mode == "exact"
    KC.check(_emu_bias_grad(dz, C, 0.5, sms), ref, mag, chain=chain, exact=exact)
    _rejects(lambda: KC.check(_emu_bias_grad(dz, C, 0.5, sms, drop_block=3), ref, mag, chain=chain, exact=exact))


def _emu_fc_bias_act(acc, bias, p, seed, offset, counter="quad", scale=None):
    """fc_bias_act in fp32 with a Philox mask; planted: the counter from the element index."""
    B, N = acc.shape
    v = torch.relu(acc + bias)
    if counter == "quad":
        keep, ks = R.dropout_mask64(seed, offset, B, N, p)
    else:
        i = torch.arange(B * N, dtype=torch.int64)
        r = R.philox4x32_10((seed & 0xFFFFFFFF, seed >> 32), (i, i >> 32, offset, 0))[0]
        keep = ~((r >> 8).to(F64) * 2 ** -24 < float(torch.tensor(p, dtype=torch.float32))).view(B, N)
        ks = R.dropout_mask64(seed, offset, 1, 1, p)[1]
    ks = torch.tensor(ks if scale is None else scale, dtype=torch.float32)
    return torch.where(keep, v * ks, torch.zeros_like(v))


@pytest.mark.parametrize("mode", MODES)
def test_dropout_criterion_catches_mask_and_scale_defects(mode):
    g = _gen(33)
    B, N, p, seed = 37, 100, 0.6, 1000003 * 5 + 2
    acc = KC.operand((B, N), mode, 1, g, CPU).float()
    bias = KC.bias(N, mode, g, CPU)
    ref, mag = R.fc_bias_act64(acc, bias, relu=True, drop_p=p, seed=seed, offset=7)
    good = _emu_fc_bias_act(acc, bias, p, seed, 7)
    KC.check(good, ref, mag, chain=0, exact=True)
    KC.check(good.to(torch.bfloat16), ref, mag, chain=0, exact=True)
    _rejects(lambda: KC.check(_emu_fc_bias_act(acc, bias, p, seed, 7, counter="element"), ref, mag, chain=0,
                              exact=True))
    _rejects(lambda: KC.check(_emu_fc_bias_act(acc, bias, p, seed, 6), ref, mag, chain=0, exact=True))
    _rejects(lambda: KC.check(_emu_fc_bias_act(acc, bias, p, seed, 7, scale=2.5), ref, mag, chain=0, exact=True))


def _emu_ce(z, t, ldd, w=None, pad=0.0, high_ties=False):
    """cross_entropy_kernel in fp32 torch ops: (loss, dlogits [B][ldd] bf16, correct count)."""
    B, C = z.shape
    mx = z.amax(1, keepdim=True)
    lse = mx + (z - mx).exp().sum(1, keepdim=True).log()
    wt = w[t] if w is not None else torch.ones(B)
    norm = 1.0 / wt.sum() if w is not None else torch.tensor(1.0 / B)
    dl = torch.full((B, ldd), pad)
    dl[:, :C] = ((z - lse).exp() - F.one_hot(t, C).float()) * wt[:, None] * norm
    nll = wt * (lse.view(-1) - z.gather(1, t.view(-1, 1)).view(-1))
    loss = nll.sum() / (wt.sum() if w is not None else B)
    am = (C - 1 - z.flip(1).argmax(1)) if high_ties else R._first_max(z)[1]
    return loss, dl.to(torch.bfloat16), float((am == t).sum())


@pytest.mark.parametrize("weighted", [False, True])
def test_cross_entropy_criterion_catches_padding_and_tie_defects(weighted):
    g = _gen(34)
    B, C, ldd = 64, 10, 16
    z = torch.randn(B, C, generator=g) * 30                 # __expf at large |x|
    t = torch.randint(0, C, (B,), generator=g)
    z[:8, 7] = z[:8, 2] = z[:8].amax(1) + 1                 # ties for the argmax in 8 rows, target 2
    t[:8] = 2
    w = torch.rand(C, generator=g) + 0.1 if weighted else None
    ref = R.cross_entropy64(z, t, ldd=ldd, class_weights=w)
    bnd = KC.ce_bound(z, t, class_weights=w, se_chain=-(-C // 32) + 5, warps=32)
    err = torch.zeros(B, ldd, dtype=F64)
    err[:, :C] = bnd["dlogits"]
    loss, dl, correct = _emu_ce(z, t, ldd, w)
    KC.check(loss.view(1), ref["loss"].view(1), torch.zeros(1, dtype=F64), chain=0, exact=False,
             err=bnd["loss"].view(1))
    KC.check(dl, ref["dlogits"], torch.zeros_like(ref["dlogits"]), chain=0, exact=False, err=err)
    assert correct == float(ref["meter"][1])
    _, bad, _ = _emu_ce(z, t, ldd, w, pad=7.0)
    _rejects(lambda: KC.check(bad, ref["dlogits"], torch.zeros_like(err), chain=0, exact=False, err=err))
    assert _emu_ce(z, t, ldd, w, high_ties=True)[2] != float(ref["meter"][1])


def _emu_adam(p, m, v, g, *, lr, b1, b2, eps, wd, step, gs, bc_off=0, eps_in_sqrt=False, drop_wd=False):
    """adam_kernel in fp32 torch ops; the planted defects are options."""
    f = torch.float32
    s = step + bc_off
    bc1i = torch.tensor(1.0 / (1.0 - b1 ** s), dtype=f)
    bc2i = torch.tensor(1.0 / (1.0 - b2 ** s) ** 0.5, dtype=f)
    b1_, b2_ = torch.tensor(b1, dtype=f), torch.tensor(b2, dtype=f)
    gk = g * gs + (0.0 if drop_wd else torch.tensor(wd, dtype=f) * p)
    m1 = b1_ * m + (1 - b1_) * gk
    v1 = b2_ * v + (1 - b2_) * gk * gk
    d = (v1 + eps).sqrt() * bc2i if eps_in_sqrt else v1.sqrt() * bc2i + eps
    p1 = p - torch.tensor(lr, dtype=f) * bc1i * m1 / d
    return p1, m1, v1


def test_adam_criterion_catches_optimizer_defects():
    g = _gen(35)
    n = 4096
    f32 = R._f32
    hp = dict(lr=f32(1e-3), b1=f32(0.9), b2=f32(0.999), eps=f32(1e-8), wd=f32(0.01), gs=0.125)
    p = torch.randn(n, generator=g)
    m = torch.randn(n, generator=g) * 1e-3
    v = torch.rand(n, generator=g) * 1e-6
    gr = torch.randn(n, generator=g) * 10 ** (torch.rand(n, generator=g) * -6)   # magnitudes 1 .. 1e-6
    step = 10
    ref = R.adam_step64(p, m, v, gr, lr=hp["lr"], beta1=hp["b1"], beta2=hp["b2"], eps=hp["eps"],
                        weight_decay=hp["wd"], step=step, grad_scale=hp["gs"])

    def ok(out):
        for got, key in zip(out, ("p", "m", "v")):
            r, e = ref[key]
            KC.check(got, r, torch.zeros_like(r), chain=0, exact=False, err=e)

    kw = dict(lr=hp["lr"], b1=hp["b1"], b2=hp["b2"], eps=hp["eps"], wd=hp["wd"], step=step, gs=hp["gs"])
    good = _emu_adam(p, m, v, gr, **kw)
    ok(good)
    _rejects(lambda: ok(_emu_adam(p, m, v, gr, bc_off=1, **kw)))
    _rejects(lambda: ok(_emu_adam(p, m, v, gr, eps_in_sqrt=True, **kw)))
    _rejects(lambda: ok(_emu_adam(p, m, v, gr, drop_wd=True, **kw)))
    # the shadow is RNE(p) of the kernel's own p, bit for bit
    KC.check(good[0].to(torch.bfloat16), good[0].to(F64), good[0].to(F64), chain=0, exact=True)
    _rejects(lambda: KC.check(_trunc_bf16(good[0]), good[0].to(F64), good[0].to(F64), chain=0, exact=True))


def test_sgd_criterion_passes_emulation():
    g = _gen(36)
    n = 4096
    p, buf, gr = (torch.randn(n, generator=g) for _ in range(3))
    for first in (True, False):
        ref = R.sgd_step64(p, buf, gr, lr=R._f32(0.01), momentum=R._f32(0.9), weight_decay=R._f32(1e-4),
                           first=first, grad_scale=0.125)
        f = torch.float32
        gk = gr * 0.125 + torch.tensor(R._f32(1e-4), dtype=f) * p
        b1 = gk if first else torch.tensor(R._f32(0.9), dtype=f) * buf + gk
        p1 = p - torch.tensor(R._f32(0.01), dtype=f) * b1
        KC.check(p1, ref["p"][0], torch.zeros(n, dtype=F64), chain=0, exact=False, err=ref["p"][1])
        KC.check(b1, ref["buf"][0], torch.zeros(n, dtype=F64), chain=0, exact=False, err=ref["buf"][1])
        _rejects(lambda: KC.check(p + torch.tensor(R._f32(0.01)) * gr * 0.125, ref["p"][0], torch.zeros(n, dtype=F64),
                                  chain=0, exact=False, err=ref["p"][1]))       # weight decay and momentum dropped
