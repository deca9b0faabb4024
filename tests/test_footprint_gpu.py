"""The hand-picked edge shapes of the kernel tests, replayed on guarded operands.

The engine replay (test_engine_replay_gpu.py) covers the shapes the training step launches; the
deliberately ragged cases live in test_kernels_gpu.py and test_wide_tiles_gpu.py: GEMMs with M or
N far from a tile multiple, ``lda > M``, bf16 stores at element offsets 4 and 8, convolutions on
12 x 20 and 16 x 40 maps, pooled layers at a batch of 37, conv0 on a 30 x 22 image and the
256-wide channel tiles.  Each becomes a launch signature and runs through the same ``_replay``, in
exact mode: values against the float64 reference, footprint against the kernel's write contract.
"""
import pytest
import torch

import kernel_check as KC
import test_kernels_gpu as TK
import test_wide_tiles_gpu as TW
from launch_replay import _replay

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF, F32, I32 = torch.bfloat16, torch.float32, torch.int32


def _T(shape, dtype, stride=None, off=0):
    """The signature of a tensor of ``shape`` (row-major unless ``stride``) at storage offset ``off``."""
    if stride is None:
        stride, s = [], 1
        for n in reversed(shape):
            stride.insert(0, s)
            s *= n
    return ("T", tuple(shape), tuple(stride), dtype, off % 16)


def _rup8(v):
    return (v + 7) // 8 * 8


def _gemm(A, a_mn, B, b_mn, M, N, K, out, ldo, epi, bias=None, alpha=1.0, ksplit=1, bn=0):
    return ("gemm", A, a_mn, B, b_mn, M, N, K, out, ldo, epi, bias, alpha, ksplit, bn)


def _gemm_sigs():
    sigs = []
    for M, N, K in TK.GEMM_KK_SHAPES:                      # FC forward: [:, :K] of [*, Kp], transposed out
        for ks in TK.KSPLITS:
            sigs.append(_gemm(_T((M, K), BF, (_rup8(K), 1)), False, _T((N, K), BF, (_rup8(K), 1)), False, M, N, K,
                              _T((N, M), F32), M, "f32_atomic_t", ksplit=ks))
    for M, N, K in TK.GEMM_MNK_SHAPES:                     # FC dgrad, lda = rup8(M) > M
        sigs.append(_gemm(_T((K, M), BF, (_rup8(M), 1)), True, _T((N, K), BF, (_rup8(K), 1)), False, M, N, K,
                          _T((N, M), F32), M, "f32_store_t"))
    for M, N, K, ks in TK.GEMM_MNK_ATOMIC:
        sigs.append(_gemm(_T((K, M), BF, (_rup8(M), 1)), True, _T((N, K), BF, (_rup8(K), 1)), False, M, N, K,
                          _T((N, M), F32), M, "f32_atomic_t", ksplit=ks))
    for M, N, K in TK.WGRAD_FC:                            # FC wgrad, both operands [K][*]
        sigs.append(_gemm(_T((K, _rup8(M)), BF), True, _T((K, N), BF), True, M, N, K, _T((M, N), F32), N,
                          "f32_store", alpha=0.5))
    for M, N, K, off in TK.GEMM_MNMN_BF16_SHAPES:          # bf16 wire stores at element offsets 0, 4, 8
        sigs.append(_gemm(_T((K, _rup8(M)), BF), True, _T((K, N), BF), True, M, N, K, _T((M, N), BF, off=off), N,
                          "bf16_store", alpha=0.125))
    for M, N, K in TK.BIAS_RELU_SHAPES:                    # ragged N of 48 and 96
        sigs.append(_gemm(_T((M, K), BF), False, _T((N, K), BF), False, M, N, K, _T((M, N), BF), N,
                          "bf16_bias_relu", bias=_T((N,), F32)))
    return sigs


def _conv_sigs(N, H, W, Cin, Cout, bn=0, pool=False):
    x, w, y = _T((N, H, W, Cin), BF), _T((Cout, 3, 3, Cin), BF), _T((N, H, W, Cout), BF)
    sigs = [("conv_fprop", x, w, _T((Cout,), F32), y, True, bn),
            ("conv_dgrad", y, w, x, x, _T((Cin,), F32) if Cin <= 512 else None, bn),
            ("conv_wgrad", y, x, _T((Cout, 3, 3, Cin), F32), 1.0, 0, bn)]
    if pool:
        p = _T((N, H // 2, W // 2, Cout), BF)
        mask = _T((N, H // 2, W // 2, Cout // 32, 4), I32)
        sigs += [("conv_fprop_pool", x, w, _T((Cout,), F32), p, mask, bn),
                 ("unpool2x2", p, mask, y, _T((Cout,), F32))]
    return sigs


def _sigs():
    sigs = _gemm_sigs()
    for shape in TK.CONV_SHAPES:
        sigs += _conv_sigs(*shape)
    for shape in TK.POOL_SHAPES:
        if shape[0] != 64:                                  # batch 64 is what the engine replay launches
            sigs += [s for s in _conv_sigs(*shape, pool=True) if s[0] in ("conv_fprop_pool", "unpool2x2")]
    for N, H, W in TK.CONV0_SHAPES:
        if N * H * W < 2 ** 20:
            x4 = _T((N, H, W, 4), BF)
            sigs += [("conv0_fprop", x4, _T((64, 64), BF), _T((64,), F32), _T((N, H, W, 64), BF)),
                     ("conv0_wgrad", _T((N, H, W, 64), BF), x4, _T((64, 64), F32))]
    for shape in TW.SHAPES:
        sigs += _conv_sigs(*shape, bn=256, pool=True)
    return sigs


SIGS = _sigs()


def _id(sig):
    dims = [s[1] for s in sig[1:] if isinstance(s, tuple) and s and s[0] == "T"]
    extra = "-".join(str(v) for v in sig[1:] if isinstance(v, (int, float, str)) and not isinstance(v, bool))
    return "%s-%s-%s" % (sig[0], "x".join(str(d) for d in dims[0]), extra)


@pytest.mark.parametrize("sig", SIGS, ids=[_id(s) for s in SIGS])
def test_edge_shape_footprint(sig):
    from distributed_vgg_f_b200 import ops

    C = ops.require()
    if sig[0] == "gemm":                                    # epilogue name -> the extension's code
        sig = sig[:10] + (getattr(C, "EPI_" + sig[10].upper()),) + sig[11:]
    _replay(C, sig, torch.Generator(device=DEV).manual_seed(len(str(sig))), KC.sm_count())
    torch.cuda.empty_cache()
