"""Numerics of every sm_90a kernel against a plain PyTorch fp32 reference of the same op.

bf16 operands: inputs are rounded to bf16 first, the reference is evaluated in fp32 on those
rounded values, so the only differences are accumulation order and the final bf16 rounding.
"""
import math

import pytest
import torch
import torch.nn.functional as F

import kernel_check as KC
from distributed_vgg_f_b200.ops import ref as R

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _ops():
    from distributed_vgg_f_b200 import ops
    ops.require()
    return ops


def rel_err(got: torch.Tensor, ref: torch.Tensor) -> float:
    got, ref = got.float(), ref.float()
    return float((got - ref).abs().max() / (ref.abs().max() + 1e-12))


def bf(t):
    return t.to(torch.bfloat16)


MODES = ["exact", "gauss"]


def _rup8(v):
    return (v + 7) // 8 * 8


# ------------------------------------------------------------------------------------------ GEMM
GEMM_KK_SHAPES = [
    (128, 64, 64), (256, 64, 512), (4096, 64, 4096), (200, 48, 200), (4096, 96, 25088 // 8),
    # N <= 32: 32-wide tiles (FC forward at batch <= 32, ragged last batches)
    (4096, 1, 25088), (4096, 5, 4096), (512, 16, 4096), (4096, 32, 25088), (10, 37, 512),
    # N > 128: batches above 128 run two or more N tiles of the swap-AB forward
    (4096, 256, 4096), (1000, 130, 512), (512, 200, 25088 // 8)]
GEMM_KK = pytest.mark.parametrize("M,N,K", GEMM_KK_SHAPES)
KSPLITS = [1, 4, 8]
KSPLIT = pytest.mark.parametrize("ksplit", KSPLITS)


@GEMM_KK
@KSPLIT
def test_gemm_kk_transposed_out(M, N, K, ksplit):
    """FC forward form (swap-AB): out[b, n] += sum_k W[n, k] X[b, k]."""
    _gemm_kk(M, N, K, ksplit, "gauss")


@GEMM_KK
@KSPLIT
def test_gemm_kk_transposed_out_exact(M, N, K, ksplit):
    _gemm_kk(M, N, K, ksplit, "exact")


def _gemm_kk(M, N, K, ksplit, mode):
    ops = _ops()
    g = KC.generator(M * 7 + N * 3 + K + ksplit, DEV)
    Kp = _rup8(K)
    A = KC.operand((M, Kp), mode, K, g, DEV)[:, :K]
    B = KC.operand((N, Kp), mode, K, g, DEV)[:, :K]
    out = torch.zeros(N, M, device=DEV)
    ops.gemm(A, B, out, M=M, N=N, K=K, epi="f32_atomic_t", ksplit=ksplit, ldo=M)
    ref, mag = R.gemm64(A, B, M=M, N=N, K=K, epi="f32_atomic_t")
    KC.check(out, ref, mag, chain=KC.gemm_chain(K, ksplit), exact=mode == "exact", family="gemm")


GEMM_MNK_SHAPES = [(128, 64, 64), (25088 // 4, 64, 4096), (300, 40, 130), (4096, 32, 4096), (512, 3, 10),
                   (4096, 256, 4096), (300, 129, 130)]                  # N > 128: two N tiles
GEMM_MNK = pytest.mark.parametrize("M,N,K", GEMM_MNK_SHAPES)


@GEMM_MNK
def test_gemm_mnk_store_t(M, N, K):
    """FC dgrad form: A stored [K][M] (W[n_out][k_in] read as A[m=k_in, k=n_out]); B = dz [N][K] with
    ldb = round_up(K, 8)."""
    _gemm_mnk(M, N, K, 1, "f32_store_t", "gauss")


@GEMM_MNK
def test_gemm_mnk_store_t_exact(M, N, K):
    _gemm_mnk(M, N, K, 1, "f32_store_t", "exact")


GEMM_MNK_ATOMIC = [(4096, 64, 4096, 8), (4096, 37, 4096, 8), (4096, 16, 512, 8), (25088, 5, 4096, 8),
                   (4096, 64, 4096, 1), (512, 10, 10, 1), (25088, 256, 4096, 8), (4096, 144, 512, 1),
                   (4096, 192, 4096, 4)]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("M,N,K,ksplit", GEMM_MNK_ATOMIC)
def test_gemm_mnk_atomic_t(M, N, K, ksplit, mode):
    """FC dgrad as the engine runs it: M = fin, N = batch, K = fout, split-K into the atomic epilogue."""
    _gemm_mnk(M, N, K, ksplit, "f32_atomic_t", mode)


def _gemm_mnk(M, N, K, ksplit, epi, mode):
    ops = _ops()
    g = KC.generator(M + N * 5 + K * 3 + ksplit, DEV)
    A_km = KC.operand((K, _rup8(M)), mode, K, g, DEV)[:, :M]       # [K][M]
    B = KC.operand((N, _rup8(K)), mode, K, g, DEV)[:, :K]          # [N][K]
    out = torch.zeros(N, M, device=DEV)
    ops.gemm(A_km, B, out, M=M, N=N, K=K, a_mn=True, epi=epi, ksplit=ksplit, ldo=M)
    ref, mag = R.gemm64(A_km, B, M=M, N=N, K=K, a_mn=True, epi=epi)
    KC.check(out, ref, mag, chain=KC.gemm_chain(K, ksplit), exact=mode == "exact", family="gemm")


# FC wgrad: M = fout, N = fin, K = batch; A = dz [K][round_up(fout, 8)] (lda > M when fout % 8 != 0)
WGRAD_FC = [(128, 64, 64), (4096, 1024, 64), (512, 256, 96), (3 * 8, 512, 64), (256, 72, 64),
            (10, 4096, 5), (10, 4096, 37), (1000, 4096, 16), (4096, 512, 37), (10, 512, 64), (4096, 4096, 5)]


@pytest.mark.parametrize("M,N,K", WGRAD_FC)
def test_gemm_mnmn_store(M, N, K):
    """FC wgrad form: dW[n_out, k_in] = sum_b dY[b, n_out] X[b, k_in]; both operands [K][*]."""
    _gemm_mnmn(M, N, K, "gauss")


@pytest.mark.parametrize("M,N,K", WGRAD_FC)
def test_gemm_mnmn_store_exact(M, N, K):
    _gemm_mnmn(M, N, K, "exact")


def _gemm_mnmn(M, N, K, mode):
    ops = _ops()
    g = KC.generator(M + N + K, DEV)
    A_km = KC.operand((K, _rup8(M)), mode, K, g, DEV)
    B_kn = KC.operand((K, N), mode, K, g, DEV)
    out = torch.empty(M, N, device=DEV)
    ops.gemm(A_km, B_kn, out, M=M, N=N, K=K, a_mn=True, b_mn=True, epi="f32_store", alpha=0.5)
    ref, mag = R.gemm64(A_km, B_kn, M=M, N=N, K=K, a_mn=True, b_mn=True, alpha=0.5)
    KC.check(out, ref, mag, chain=KC.gemm_chain(K), exact=mode == "exact", family="gemm")


GEMM_MNMN_BF16_SHAPES = [
    (128, 64, 64, 0), (4096, 1024, 64, 0), (512, 256, 96, 8), (256, 72, 64, 0), (24, 512, 64, 4),
    (10, 4096, 5, 0), (10, 4096, 37, 8), (1000, 4096, 16, 0), (4096, 512, 37, 4)]
GEMM_MNMN_BF16 = pytest.mark.parametrize("M,N,K,off", GEMM_MNMN_BF16_SHAPES)


@GEMM_MNMN_BF16
def test_gemm_mnmn_bf16_store(M, N, K, off):
    """FC wgrad written straight to the bf16 wire: out = bf16(alpha * dY^T X).  ``off`` shifts the
    output start by a few elements (32-byte vs 16-byte vs scalar store paths), N=72 is ragged."""
    _gemm_mnmn_bf16(M, N, K, off, "gauss")


@GEMM_MNMN_BF16
def test_gemm_mnmn_bf16_store_exact(M, N, K, off):
    _gemm_mnmn_bf16(M, N, K, off, "exact")


def _gemm_mnmn_bf16(M, N, K, off, mode):
    ops = _ops()
    g = KC.generator(M * 3 + N + K + off, DEV)
    A_km = KC.operand((K, _rup8(M)), mode, K, g, DEV)
    B_kn = KC.operand((K, N), mode, K, g, DEV)
    buf = torch.full((M * N + 64,), 7.0, dtype=torch.bfloat16, device=DEV)
    out = buf[off:off + M * N].view(M, N)
    ops.gemm(A_km, B_kn, out, M=M, N=N, K=K, a_mn=True, b_mn=True, epi="bf16_store", alpha=0.125)
    ref, mag = R.gemm64(A_km, B_kn, M=M, N=N, K=K, a_mn=True, b_mn=True, alpha=0.125)
    KC.check(out, ref, mag, chain=KC.gemm_chain(K), exact=mode == "exact", family="gemm")
    assert bool((buf[:off] == 7.0).all()) and bool((buf[off + M * N:] == 7.0).all())


def test_gemm_bf16_bias_relu():
    """Layer-0 im2col GEMM: bf16(relu(A W^T + b))."""
    _gemm_bias_relu(1000, 64, 64, "gauss")


BIAS_RELU_SHAPES = [(1000, 64, 64), (300, 48, 64), (129, 96, 128)]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("M,N,K", BIAS_RELU_SHAPES)
def test_gemm_bf16_bias_relu_ragged_n(M, N, K, mode):
    """A ragged N (48, 96) must write nothing past column N of a row nor past the end of the output,
    and read no bias past N (the bias is a slice of a NaN-filled buffer)."""
    _gemm_bias_relu(M, N, K, mode)


def _gemm_bias_relu(M, N, K, mode):
    ops = _ops()
    g = KC.generator(M + N + K, DEV)
    A = KC.operand((M, K), mode, K, g, DEV)
    W = KC.operand((N, K), mode, K, g, DEV, scale=0.2)
    bias_buf = torch.full((N + 64,), float("nan"), device=DEV)
    bias_buf[16:16 + N] = KC.bias(N, mode, g, DEV)
    bias = bias_buf[16:16 + N]
    buf = torch.full((M * N + 256,), 7.0, dtype=torch.bfloat16, device=DEV)
    out = buf[:M * N].view(M, N)
    ops.gemm(A, W, out, M=M, N=N, K=K, epi="bf16_bias_relu", bias=bias)
    ref, mag = R.gemm64(A, W, M=M, N=N, K=K, epi="bf16_bias_relu", bias=bias)
    KC.check(out, ref, mag, chain=KC.gemm_chain(K), exact=mode == "exact", family="gemm")
    assert bool((buf[M * N:] == 7.0).all())


# ------------------------------------------------------------------------------------------ conv
def _conv_case(N, H, W, Cin, Cout, seed=0, mode="gauss"):
    g = KC.generator(seed * 1000003 + N * 7919 + H * 131 + Cin + Cout, DEV)
    x = KC.operand((N, H, W, Cin), mode, 9 * Cin, g, DEV)
    w = KC.operand((Cout, 3, 3, Cin), mode, 9 * Cin, g, DEV, scale=1.0 / math.sqrt(9 * Cin))
    b = KC.bias(Cout, mode, g, DEV)
    return x, w, b, g


CONV_SHAPES = [(2, 16, 16, 64, 64), (1, 28, 28, 128, 256), (4, 14, 14, 512, 512), (2, 56, 56, 64, 128),
               (3, 12, 20, 64, 64), (1, 224, 224, 64, 64),
               # halo-tile kernel (H % 16 == 0, W % 8 == 0, W >= 32): resident / streaming weights
               (2, 32, 32, 64, 64), (1, 32, 32, 64, 128), (1, 48, 64, 128, 128), (1, 32, 32, 256, 256),
               (3, 16, 40, 128, 64)]
# one layer per VGG resolution, at batch 64 and at a ragged last batch of 37
VGG_SHAPES = [(n, h, h, c, c) for n in (64, 37) for h, c in ((224, 64), (112, 128), (56, 256), (28, 512), (14, 512))]
CONV_ALL = pytest.mark.parametrize("N,H,W,Cin,Cout", CONV_SHAPES + VGG_SHAPES)


@CONV_ALL
def test_conv_fprop(N, H, W, Cin, Cout):
    _conv_fprop(N, H, W, Cin, Cout, "gauss")


@CONV_ALL
def test_conv_fprop_exact(N, H, W, Cin, Cout):
    _conv_fprop(N, H, W, Cin, Cout, "exact")


def _conv_fprop(N, H, W, Cin, Cout, mode):
    ops = _ops()
    x, w, b, _ = _conv_case(N, H, W, Cin, Cout, mode=mode)
    y = ops.conv3x3_fprop(x, w, b, relu=True)
    ref, mag = R.conv3x3_fprop64(x, w, b, relu=True)
    KC.check(y, ref, mag, chain=KC.conv_chain(Cin), exact=mode == "exact", family="conv_fprop")


def test_conv_fprop_rejects_a_bias_wider_than_its_scratch():
    """The fprop epilogue stages the bias in 512 floats of shared memory: Cout > 512 with a bias is
    refused on the host (without a bias the layer is fine)."""
    ops = _ops()
    x = torch.zeros(1, 8, 8, 64, dtype=torch.bfloat16, device=DEV)
    w = torch.zeros(576, 3, 3, 64, dtype=torch.bfloat16, device=DEV)
    with pytest.raises(RuntimeError, match="Cout <= 512"):
        ops.conv3x3_fprop(x, w, torch.zeros(576, device=DEV))
    with pytest.raises(RuntimeError, match="Cout <= 512"):
        ops.conv3x3_fprop_pool(x, w, torch.zeros(576, device=DEV))
    torch.cuda.synchronize()


@CONV_ALL
def test_conv_dgrad(N, H, W, Cin, Cout):
    _conv_dgrad(N, H, W, Cin, Cout, "gauss")


@CONV_ALL
def test_conv_dgrad_exact(N, H, W, Cin, Cout):
    _conv_dgrad(N, H, W, Cin, Cout, "exact")


def _conv_dgrad(N, H, W, Cin, Cout, mode):
    ops = _ops()
    x, w, _, g = _conv_case(N, H, W, Cin, Cout, seed=1, mode=mode)
    exact = mode == "exact"
    dz = KC.operand((N, H, W, Cout), mode, 9 * Cout, g, DEV)
    dx = ops.conv3x3_dgrad(dz, w, Cin)
    ref, mag = R.conv3x3_dgrad64(dz, w)
    chain = KC.conv_chain(Cout)
    KC.check(dx, ref, mag, chain=chain, exact=exact, family="conv_dgrad")
    # fused ReLU mask
    mask_src = KC.operand((N, H, W, Cin), "gauss", 1, g, DEV)
    dx2 = ops.conv3x3_dgrad(dz, w, Cin, mask_src=mask_src)
    ref, mag = R.conv3x3_dgrad64(dz, w, mask_src=mask_src)
    KC.check(dx2, ref, mag, chain=chain, exact=exact, family="conv_dgrad", what="masked")
    # fused column sum (= bias gradient of the previous layer): sums exactly what was stored
    if Cin <= 512:
        cs = torch.zeros(Cin, device=DEV)
        dx3 = ops.conv3x3_dgrad(dz, w, Cin, mask_src=mask_src, colsum=cs)
        assert torch.equal(dx3, dx2)
        stored = dx2.to(torch.float64).reshape(-1, Cin)
        KC.check(cs, stored.sum(0), stored.abs().sum(0), chain=KC.conv_colsum_chain(N * H * W, Cin, KC.sm_count()),
                 exact=False, family="conv_colsum")


@CONV_ALL
def test_conv_wgrad(N, H, W, Cin, Cout):
    _conv_wgrad(N, H, W, Cin, Cout, "gauss")


@CONV_ALL
def test_conv_wgrad_exact(N, H, W, Cin, Cout):
    _conv_wgrad(N, H, W, Cin, Cout, "exact")


def _conv_wgrad(N, H, W, Cin, Cout, mode):
    ops = _ops()
    g = KC.generator(N * 7 + H + Cin * 3 + Cout, DEV)
    P = N * H * W
    x = KC.operand((N, H, W, Cin), mode, P, g, DEV)
    dz = KC.operand((N, H, W, Cout), mode, P, g, DEV)
    dw = torch.zeros(Cout, 3, 3, Cin, device=DEV)
    ops.conv3x3_wgrad(dz, x, dw)
    ref, mag = R.conv3x3_wgrad64(dz, x)
    KC.check(dw, ref, mag, chain=KC.wgrad_chain(N, H, W, Cin, Cout, KC.sm_count()), exact=mode == "exact",
             family="conv_wgrad")


CONV0_SHAPES = [(2, 16, 16), (1, 30, 22), (3, 64, 64), (64, 224, 224), (37, 224, 224)]
CONV0 = pytest.mark.parametrize("N,H,W", CONV0_SHAPES)


@CONV0
def test_conv0_fused(N, H, W):
    """First conv straight from NHWC4 pixels (im2col tile built in shared memory): fprop + wgrad.
    64 x 224 x 224 gives every CTA many tiles, so the stage ring and the builder groups wrap."""
    _conv0(N, H, W, "gauss")


@CONV0
def test_conv0_fused_exact(N, H, W):
    _conv0(N, H, W, "exact")


def _conv0(N, H, W, mode):
    ops = _ops()
    C = ops.require()
    exact = mode == "exact"
    g = KC.generator(N * 31 + H + W, DEV)
    x4 = torch.zeros(N, H, W, 4, dtype=torch.bfloat16, device=DEV)
    x4[..., :3] = KC.operand((N, H, W, 3), mode, 27, g, DEV)
    w0 = torch.zeros(64, 64, dtype=torch.bfloat16, device=DEV)
    w0[:, :27] = KC.operand((64, 27), mode, 27, g, DEV, scale=0.2)
    bias = KC.bias(64, mode, g, DEV)
    y = torch.empty(N, H, W, 64, dtype=torch.bfloat16, device=DEV)
    C.conv0_fprop(x4, w0, bias, y)
    ref, mag = R.conv0_fprop64(x4, w0, bias)
    KC.check(y, ref, mag, chain=KC.gemm_chain(64), exact=exact, family="conv0_fprop")
    P = N * H * W
    x4w = torch.zeros_like(x4)
    x4w[..., :3] = KC.operand((N, H, W, 3), mode, P, g, DEV)
    dz = KC.operand((N, H, W, 64), mode, P, g, DEV)
    dw0 = torch.zeros(64, 64, device=DEV)
    C.conv0_wgrad(dz, x4w, dw0)
    ref, mag = R.conv0_wgrad64(dz, x4w)
    KC.check(dw0, ref, mag, chain=KC.conv0_wgrad_chain(P, KC.sm_count()), exact=exact, family="conv0_wgrad")


# ------------------------------------------------------------------------------------- pointwise
POOL_SHAPES = [(2, 32, 32, 64, 64), (1, 48, 64, 128, 128), (2, 56, 56, 64, 128), (3, 28, 28, 128, 256),
               (4, 14, 14, 512, 512), (1, 224, 224, 64, 64),
               # the pooled VGG layers at batch 64 and at a ragged batch of 37
               (64, 224, 224, 64, 64), (37, 112, 112, 128, 128), (64, 56, 56, 256, 256), (37, 28, 28, 512, 512),
               (64, 14, 14, 512, 512), (37, 14, 14, 512, 512)]


@pytest.mark.parametrize("N,H,W,Cin,Cout", POOL_SHAPES)
def test_conv_fprop_pool_fused(N, H, W, Cin, Cout):
    """conv + bias + ReLU + 2x2 max-pool in the conv epilogue (the default for pooled layers) against
    the float64 reference, and bit-identical to the separate kernels (same rounding point, same
    first-maximum rule); then its unpool backward."""
    _conv_pool(N, H, W, Cin, Cout, "gauss")


@pytest.mark.parametrize("N,H,W,Cin,Cout", POOL_SHAPES)
def test_conv_fprop_pool_fused_exact(N, H, W, Cin, Cout):
    _conv_pool(N, H, W, Cin, Cout, "exact")


def _conv_pool(N, H, W, Cin, Cout, mode):
    ops = _ops()
    exact = mode == "exact"
    x, w, b, g = _conv_case(N, H, W, Cin, Cout, seed=5, mode=mode)
    p, mask = ops.conv3x3_fprop_pool(x, w, b)
    ref, mag = R.conv3x3_fprop64(x, w, b, relu=True)
    KC.check_pool(p, mask, ref, mag, chain=KC.conv_chain(Cin), exact=exact)
    del ref, mag
    y = ops.conv3x3_fprop(x, w, b, relu=True)
    assert torch.equal(p, ops.maxpool2x2(y))
    idx, pos = R.pool_mask_decode(mask, Cout)
    _, ridx, rpos = R.pool2x2_select(y.float())
    assert torch.equal(pos, rpos) and torch.equal(torch.where(pos, idx, 0), torch.where(rpos, ridx, 0))
    dp = KC.operand((N, H // 2, W // 2, Cout), mode, 1, g, DEV)
    cs_ref = torch.zeros(Cout, device=DEV)
    dz_ref = ops.maxpool2x2_relu_bwd(y, dp, colsum=cs_ref)
    del y
    cs = torch.zeros(Cout, device=DEV)
    dz = ops.unpool2x2(dp, mask, colsum=cs)
    assert torch.equal(dz, dz_ref)
    want, want_cs, cs_mag = R.unpool2x2_64(dp, idx, pos)
    KC.check(dz, want, want, chain=0, exact=True, family="unpool2x2")
    chain = KC.unpool_colsum_chain(N * (H // 2) * (W // 2), Cout, KC.sm_count())
    KC.check(cs, want_cs, cs_mag, chain=chain, exact=False, family="unpool_colsum")
    KC.check(cs_ref, want_cs, cs_mag, chain=chain, exact=False, family="unpool_colsum", what="maxpool2x2_relu_bwd")


def test_maxpool_fwd_bwd():
    ops = _ops()
    torch.manual_seed(0)
    x = bf(torch.relu(torch.randn(3, 8, 12, 64, device=DEV)))
    y = ops.maxpool2x2(x)
    xr = x.float().permute(0, 3, 1, 2).clone().requires_grad_(True)
    yr = F.max_pool2d(xr, 2, 2)
    assert torch.equal(y.float(), yr.permute(0, 2, 3, 1))
    dp = bf(torch.randn_like(y.float()))
    dz = ops.maxpool2x2_relu_bwd(x, dp)
    yr.backward(dp.float().permute(0, 3, 1, 2))
    ref = (xr.grad * (xr > 0)).permute(0, 2, 3, 1)
    assert rel_err(dz, ref) < 1e-6
    # fused bias gradient (column sum of dz)
    cs = torch.zeros(64, device=DEV)
    dz2 = ops.maxpool2x2_relu_bwd(x, dp, colsum=cs)
    assert torch.equal(dz2, dz)
    assert rel_err(cs, dz.float().sum((0, 1, 2))) < 1e-4


@pytest.mark.parametrize("H", [4, 7, 14])
def test_adaptive_avgpool(H):
    ops = _ops()
    torch.manual_seed(0)
    x = bf(torch.randn(2, H, H, 64, device=DEV))
    y = ops.adaptive_avgpool(x, 7, 7)
    xr = x.float().permute(0, 3, 1, 2).clone().requires_grad_(True)
    yr = F.adaptive_avg_pool2d(xr, (7, 7))
    assert rel_err(y, yr.permute(0, 2, 3, 1)) < 1e-2
    dy = bf(torch.randn_like(y.float()))
    dx = ops.adaptive_avgpool_bwd(dy, H, H)
    yr.backward(dy.float().permute(0, 3, 1, 2))
    assert rel_err(dx, xr.grad.permute(0, 2, 3, 1)) < 1e-2


@pytest.mark.parametrize("rows,C", [(64, 4096), (5000, 64), (3000, 512), (64, 3)])
def test_bias_grad(rows, C):
    ops = _ops()
    torch.manual_seed(0)
    ld = (C + 7) // 8 * 8
    dz = bf(torch.randn(rows, ld, device=DEV))
    db = torch.zeros(C, device=DEV)
    ops.bias_grad(dz, db, rows, C, ld=ld, scale=0.5)
    ref = 0.5 * dz.float()[:, :C].sum(0)
    assert rel_err(db, ref) < 1e-3


def test_fc_epilogues_and_dropout():
    ops = _ops()
    torch.manual_seed(0)
    B, N = 64, 4096
    acc0 = torch.randn(B, N, device=DEV)
    bias = torch.randn(N, device=DEV)
    acc = acc0.clone()
    y = torch.empty(B, N, dtype=torch.bfloat16, device=DEV)
    ops.fc_bias_act(acc, bias, y, B=B, N=N, relu=True, drop_p=0.0)
    assert torch.count_nonzero(acc) == 0
    assert rel_err(y, torch.relu(acc0 + bias)) < 1e-2
    acc = acc0.clone()
    ops.fc_bias_act(acc, bias, y, B=B, N=N, relu=True, drop_p=0.5, seed=7, offset=3)
    base = torch.relu(acc0 + bias)
    kept = (y.float() != 0) | (base == 0)
    frac = float(((y.float() == 0) & (base > 0)).sum() / (base > 0).sum())
    assert 0.47 < frac < 0.53                      # Bernoulli(0.5) drop rate
    sel = (y.float() != 0)
    assert rel_err(y.float()[sel], 2.0 * base[sel]) < 1e-2
    y2 = torch.empty_like(y)
    acc = acc0.clone()
    ops.fc_bias_act(acc, bias, y2, B=B, N=N, relu=True, drop_p=0.5, seed=7, offset=3)
    assert torch.equal(y, y2)                      # same (seed, offset) -> same mask
    # backward epilogue
    g = torch.randn(B, N, device=DEV)
    dz = torch.empty(B, N, dtype=torch.bfloat16, device=DEV)
    ops.fc_grad_act(g.clone(), y, dz, B=B, N=N, relu=True, drop_p=0.5)
    assert rel_err(dz, g * (y.float() > 0) * 2.0) < 1e-2
    del kept


@pytest.mark.parametrize("B,C", [(64, 3), (96, 1000), (7, 10)])
def test_cross_entropy(B, C):
    ops = _ops()
    torch.manual_seed(0)
    logits = torch.randn(B, C, device=DEV) * 3
    target = torch.randint(0, C, (B,), device=DEV)
    ldd = (C + 7) // 8 * 8
    dl = torch.empty(B, ldd, dtype=torch.bfloat16, device=DEV)
    meter = torch.zeros(4, device=DEV)
    loss = torch.zeros(1, device=DEV)
    ops.cross_entropy(logits, target, dl, ldd, meter, loss)
    lr = logits.clone().requires_grad_(True)
    ref = F.cross_entropy(lr, target)
    ref.backward()
    assert abs(float(loss) - float(ref)) < 1e-4
    assert rel_err(dl[:, :C], lr.grad) < 1e-2
    assert torch.count_nonzero(dl[:, C:]) == 0
    assert abs(float(meter[0]) - float(ref) * B) < 1e-2
    assert int(meter[1]) == int((logits.argmax(1) == target).sum())
    assert int(meter[2]) == B


@pytest.mark.parametrize("B,C", [(64, 3), (33, 10)])
def test_cross_entropy_class_weights(B, C):
    """The reference's optional weighted loss (distributedVggf.py:164-166): torch semantics,
    loss = sum_i w[y_i] nll_i / sum_i w[y_i], and the gradient that goes with it."""
    ops = _ops()
    torch.manual_seed(1)
    logits = torch.randn(B, C, device=DEV) * 2
    target = torch.randint(0, C, (B,), device=DEV)
    w = torch.rand(C, device=DEV) + 0.1
    ldd = (C + 7) // 8 * 8
    dl = torch.empty(B, ldd, dtype=torch.bfloat16, device=DEV)
    meter = torch.zeros(4, device=DEV)
    loss = torch.zeros(1, device=DEV)
    ops.cross_entropy(logits, target, dl, ldd, meter, loss, class_weights=w)
    lr = logits.clone().requires_grad_(True)
    ref = F.cross_entropy(lr, target, weight=w)
    ref.backward()
    assert abs(float(loss) - float(ref)) < 1e-4
    assert rel_err(dl[:, :C], lr.grad) < 1e-2
    assert abs(float(meter[0]) - float(ref) * B) < 1e-2 and int(meter[2]) == B


def test_adam_matches_torch():
    ops = _ops()
    torch.manual_seed(0)
    n = 4096 * 5
    p0 = torch.randn(n, device=DEV)
    p = p0.clone()
    m = torch.zeros(n, device=DEV)
    v = torch.zeros(n, device=DEV)
    shadow = torch.empty(n, dtype=torch.bfloat16, device=DEV)
    ref_p = p0.clone().requires_grad_(True)
    opt = torch.optim.Adam([ref_p], lr=1e-3)
    for step in range(1, 4):
        g = torch.randn(n, device=DEV)
        gbuf = g.clone()
        ops.adam_step(p, m, v, g32=gbuf, shadow=shadow, lr=1e-3, step=step, zero=gbuf)
        assert torch.count_nonzero(gbuf) == 0
        ref_p.grad = g.clone()
        opt.step()
    assert rel_err(p, ref_p.detach()) < 1e-5
    assert rel_err(shadow, ref_p.detach()) < 1e-2
    # bf16 gradient source
    g16 = bf(torch.randn(n, device=DEV))
    p2, m2, v2 = p0.clone(), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    ops.adam_step(p2, m2, v2, g16=g16, lr=1e-3, step=1)
    r2 = p0.clone().requires_grad_(True)
    o2 = torch.optim.Adam([r2], lr=1e-3)
    r2.grad = g16.float()
    o2.step()
    assert rel_err(p2, r2.detach()) < 1e-5


def test_sgd_matches_torch():
    ops = _ops()
    torch.manual_seed(0)
    n = 4096
    p0 = torch.randn(n, device=DEV)
    p, mom = p0.clone(), torch.zeros(n, device=DEV)
    r = p0.clone().requires_grad_(True)
    opt = torch.optim.SGD([r], lr=0.01, momentum=0.9)
    for step in range(3):
        g = torch.randn(n, device=DEV)
        ops.sgd_step(p, mom, g32=g, lr=0.01, momentum=0.9, first=(step == 0))
        r.grad = g.clone()
        opt.step()
    assert rel_err(p, r.detach()) < 1e-5


def test_augment_matches_reference():
    ops = _ops()
    from distributed_vgg_f_b200.data import transforms as T
    from distributed_vgg_f_b200.data.synthetic import synthetic_uint8_batch

    imgs, _ = synthetic_uint8_batch(4, 128, seed=3)
    src = torch.from_numpy(imgs).to(DEV)
    g = torch.Generator().manual_seed(5)
    params = T.sample_train_params(4, 128, 128, g)
    ref = T.augment_reference(src, params, (256, 256))            # [4,3,224,224] fp32
    out = torch.empty(4, 224, 224, 8, dtype=torch.bfloat16, device=DEV)
    ops.augment(src, params.to(DEV), out, (256, 256), mode="nhwc", pad=8)
    got = out[..., :3].float().permute(0, 3, 1, 2)
    # bf16 rounding of values up to ~2.6 plus rare one-pixel floor() disagreements at exact ties
    diff = (got - ref).abs()
    assert float(diff.median()) < 5e-3
    assert float((diff > 0.05).float().mean()) < 2e-3
    # im2col mode equals unfolding the NHWC result
    col = torch.empty(4 * 224 * 224, 64, dtype=torch.bfloat16, device=DEV)
    ops.augment(src, params.to(DEV), col, (256, 256), mode="im2col", pad=64)
    unf = F.unfold(got, 3, padding=1).view(4, 3, 9, 224 * 224).permute(0, 3, 2, 1).reshape(-1, 27)
    assert torch.equal(col[:, :27].float(), unf)
    assert torch.count_nonzero(col[:, 27:]) == 0


def test_augment_kernel_matches_torchvision_chain():
    """The sm_90a input kernel against torchvision's OWN transform ops on PIL images with the same draws
    (distributedVggf.py:88-95) -- not against this repo's torch oracle."""
    ops = _ops()
    import numpy as np

    from distributed_vgg_f_b200.data import transforms as T
    from distributed_vgg_f_b200.data.synthetic import synthetic_uint8_batch

    imgs, _ = synthetic_uint8_batch(4, 128, seed=13)
    rng = np.random.default_rng(1)
    imgs = np.clip(imgs.astype(np.int16) + rng.integers(-20, 20, imgs.shape), 0, 255).astype(np.uint8)
    params = T.sample_train_params(4, 128, 128, torch.Generator().manual_seed(9))
    params[0, 6], params[1, 6] = 0.0, 1.0
    out = torch.empty(4, 224, 224, 4, dtype=torch.bfloat16, device=DEV)
    ops.augment(torch.from_numpy(imgs).to(DEV), params.to(DEV), out, (256, 256), mode="nhwc", pad=4)
    got = out[..., :3].float().permute(0, 3, 1, 2).cpu()
    for i in range(4):
        theirs = T.torchvision_chain_fixed(imgs[i], params[i])
        d = (got[i] - theirs).abs()
        # PIL's uint8 rounding of the resized image (0.009 after Normalize) + bf16 output rounding (2^-8 relative)
        assert float((d < 0.04).float().mean()) > 0.995, (i, float((d < 0.04).float().mean()), float(d.max()))
        assert float(d.mean()) < 0.012, (i, float(d.mean()))


# ------------------------------------------------------------------ fused head (K-FUN2+CE)
@pytest.mark.parametrize("B,C,K,weighted", [(64, 3, 512, False), (37, 5, 96, False), (64, 3, 512, True), (1, 8, 1024, False)])
def test_head_ce_fused_matches_torch(B, C, K, weighted):
    """Last Linear + cross-entropy + metrics + the layer's backward in one launch (loss_optim.cu::head_ce_kernel)
    against plain torch fp32 with the same rounding points (bf16 operands, dlogits rounded to bf16)."""
    from distributed_vgg_f_b200 import ops

    Cx = ops.require()
    g = torch.Generator(device="cuda").manual_seed(B * 131 + C)
    h = torch.relu(torch.randn(B, K, device="cuda", generator=g)).to(torch.bfloat16)       # post-ReLU: has zeros
    W = (torch.randn(C, K, device="cuda", generator=g) * 0.05).to(torch.bfloat16)
    bias = torch.randn(C, device="cuda", generator=g) * 0.1
    y = torch.randint(0, C, (B,), device="cuda", generator=g)
    cw = (torch.rand(C, device="cuda", generator=g) + 0.5) if weighted else None
    logits = torch.empty(B, C, device="cuda")
    dl = torch.full((B, 8), 7.0, device="cuda", dtype=torch.bfloat16)
    dW = torch.empty(C, K, device="cuda")
    db = torch.ones(C, device="cuda")                   # accumulated into
    dh = torch.empty(B, K, device="cuda", dtype=torch.bfloat16)
    meter = torch.zeros(4, device="cuda")
    loss = torch.zeros(1, device="cuda")
    Cx.head_ce(h, W, bias, y, logits, dl, 8, dW, db, dh, 2.0, True, meter, loss, cw)

    z = h.float() @ W.float().t() + bias
    ref_loss = torch.nn.functional.cross_entropy(z, y, weight=cw)
    wt = cw[y] if weighted else torch.ones(B, device="cuda")
    norm = wt.sum() if weighted else torch.tensor(float(B), device="cuda")
    g_ref = ((torch.softmax(z, 1) - torch.nn.functional.one_hot(y, C).float()) * wt[:, None] / norm)
    g_bf = g_ref.to(torch.bfloat16).float()
    torch.testing.assert_close(logits, z, rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(loss[0], ref_loss, rtol=1e-4, atol=1e-5)
    assert float(meter[1]) == float((z.argmax(1) == y).sum()) and float(meter[2]) == B
    torch.testing.assert_close(meter[0], ref_loss * B, rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(dl[:, :C].float(), g_bf, rtol=0, atol=1e-6 + 8e-3 * float(g_ref.abs().max()))
    assert float(dl[:, C:].float().abs().max()) == 0.0 if C < 8 else True
    used = dl[:, :C].float()                            # what the kernel itself rounded
    torch.testing.assert_close(dW, used.t() @ h.float(), rtol=1e-4, atol=1e-6)
    torch.testing.assert_close(db, 1.0 + used.sum(0), rtol=1e-4, atol=1e-6)
    dh_ref = ((used @ W.float()) * (h.float() > 0) * 2.0).to(torch.bfloat16)
    torch.testing.assert_close(dh.float(), dh_ref.float(), rtol=1e-2, atol=1e-6)
    # evaluation form: forward + metrics only
    logits2 = torch.empty_like(logits)
    Cx.head_ce(h, W, bias, y, logits2, None, 0, None, None, None, 1.0, False, None, loss, None)
    torch.testing.assert_close(logits2, z, rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(loss[0], torch.nn.functional.cross_entropy(z, y), rtol=1e-4, atol=1e-5)
