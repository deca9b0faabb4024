"""Every wgmma launch the engine makes, replayed against the float64 reference.

The kernel tests pick their shapes by hand; this one takes them from the engine.  ``ops._C`` is
swapped for a recording proxy during one train_step and one eval_step of several configurations.
Each distinct GEMM / convolution / unpool call signature (shapes, strides, dtypes, storage offset
mod 16 elements, scalars, which optional tensors are present) is then run once more in exact mode
on fresh tensors laid out the same way, so the vector-store alignment paths match, and compared
with the reference.  When a dispatch rule or a split heuristic of the engine changes, the replay
follows it.
"""
import os

import pytest
import torch

import kernel_check as KC
from distributed_vgg_f_b200.ops import ref as R

pytestmark = pytest.mark.gpu
DEV = "cuda"

RECORDED = ("gemm", "conv_fprop", "conv_fprop_pool", "conv_dgrad", "conv_wgrad", "conv0_fprop", "conv0_wgrad",
            "unpool2x2")


def _sig(a):
    if isinstance(a, torch.Tensor):
        return ("T", tuple(a.shape), tuple(a.stride()), a.dtype, a.storage_offset() % 16)
    return a


class _Recorder:
    """Stands in for the extension module: logs the signatures of the recorded calls, forwards all."""

    def __init__(self, real):
        self._real = real
        self.sigs = {}

    def __getattr__(self, name):
        attr = getattr(self._real, name)
        if name not in RECORDED:
            return attr

        def call(*args):
            self.sigs.setdefault((name,) + tuple(_sig(a) for a in args), None)
            return attr(*args)
        return call


def _record(configs):
    from distributed_vgg_f_b200 import ops
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine

    real = ops.require()
    rec = _Recorder(real)
    for spec, batch, steps, env in configs:
        saved = {k: os.environ.get(k) for k in env}
        os.environ.update(env)
        try:
            eng = NativeEngine(spec, device=torch.device(DEV), batch=batch, seed=0, distributed=False)
            ops._C = rec
            try:
                for b in steps:
                    g = torch.Generator(device=DEV).manual_seed(b)
                    x = torch.randn(b, 3, eng.HW, eng.HW, device=DEV, generator=g)
                    y = torch.randint(0, spec.num_classes, (b,), device=DEV, generator=g)
                    eng.train_step((x, y))
                    eng.eval_step((x, y))
                eng.sync()
            finally:
                ops._C = real
        finally:
            for k, v in saved.items():
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = v
        del eng
        torch.cuda.empty_cache()
    return real, list(rec.sigs)


def _fresh(s, fill):
    """A tensor with the recorded shape, strides, dtype and storage offset mod 16, its whole storage
    filled by ``fill(numel, dtype)``."""
    _, shape, stride, dtype, off = s
    extent = 1 + sum((n - 1) * st for n, st in zip(shape, stride)) if all(n > 0 for n in shape) else 0
    base = fill(off + extent, dtype)
    return base.as_strided(shape, stride, off)


def _ints(depth, g):
    return lambda n, dt: KC.operand((n,), "exact", depth, g, DEV).to(dt)


def _zeros(n, dt):
    return torch.zeros(n, dtype=dt, device=DEV)


def _replay(C, sig, g, sms):
    name, args = sig[0], sig[1:]
    if name == "gemm":
        sA, a_mn, sB, b_mn, M, N, K, sOut, ldo, code, sBias, alpha, ksplit, bn = args
        epi = {C.EPI_F32_STORE: "f32_store", C.EPI_F32_ATOMIC: "f32_atomic", C.EPI_F32_ATOMIC_T: "f32_atomic_t",
               C.EPI_BF16_BIAS_RELU: "bf16_bias_relu", C.EPI_F32_STORE_T: "f32_store_t",
               C.EPI_BF16_STORE: "bf16_store"}[code]
        A, B, out = _fresh(sA, _ints(K, g)), _fresh(sB, _ints(K, g)), _fresh(sOut, _zeros)
        bias = None if sBias is None else _fresh(sBias, lambda n, dt: KC.bias(n, "exact", g, DEV))
        C.gemm(A, a_mn, B, b_mn, M, N, K, out, ldo, code, bias, alpha, ksplit, bn)
        ref, mag = R.gemm64(A, B, M=M, N=N, K=K, a_mn=a_mn, b_mn=b_mn, epi=epi, bias=bias, alpha=alpha)
        got = out.as_strided(tuple(ref.shape), (ldo, 1), out.storage_offset())
        KC.check(got, ref, mag, chain=KC.gemm_chain(K, ksplit), exact=True, family="gemm", what=str(sig))
    elif name in ("conv_fprop", "conv_fprop_pool"):
        sX, sW, sBias = args[:3]
        N, H, W, Cin = sX[1]
        x = _fresh(sX, _ints(9 * Cin, g))
        w = _fresh(sW, _ints(9 * Cin, g))
        Cout = w.numel() // (9 * Cin)
        bias = None if sBias is None else _fresh(sBias, lambda n, dt: KC.bias(n, "exact", g, DEV))
        ref, mag = R.conv3x3_fprop64(x, w.reshape(Cout, 3, 3, Cin), bias, relu=True if name == "conv_fprop_pool"
                                     else args[4])
        if name == "conv_fprop":
            y = _fresh(args[3], _zeros)
            C.conv_fprop(x, w, bias, y, args[4], args[5])
            KC.check(y.reshape(N, H, W, Cout), ref, mag, chain=KC.conv_chain(Cin), exact=True, family="conv_fprop",
                     what=str(sig))
        else:
            p, mask = _fresh(args[3], _zeros), _fresh(args[4], _zeros)
            C.conv_fprop_pool(x, w, bias, p, mask, args[5])
            KC.check_pool(p, mask, ref, mag, chain=KC.conv_chain(Cin), exact=True, what=str(sig))
    elif name == "conv_dgrad":
        sDz, sW, sMask, sDx, sCs, bn = args
        N, H, W, Cout = sDz[1]
        Cin = sDx[1][-1]
        dz, w = _fresh(sDz, _ints(9 * Cout, g)), _fresh(sW, _ints(9 * Cout, g))
        mask = None if sMask is None else _fresh(sMask, _ints(1, g))
        dx = _fresh(sDx, _zeros)
        cs = None if sCs is None else _fresh(sCs, _zeros)
        C.conv_dgrad(dz, w, mask, dx, cs, bn)
        ref, mag = R.conv3x3_dgrad64(dz, w.reshape(Cout, 3, 3, Cin), mask_src=mask)
        KC.check(dx, ref, mag, chain=KC.conv_chain(Cout), exact=True, family="conv_dgrad", what=str(sig))
        if cs is not None:
            st = dx.to(torch.float64).reshape(-1, Cin)
            KC.check(cs, st.sum(0), st.abs().sum(0), chain=KC.conv_colsum_chain(N * H * W, Cin, sms), exact=False,
                     what=str(sig))
    elif name == "conv_wgrad":
        sDz, sX, sDw, scale, ksplit, bn = args
        N, H, W, Cout = sDz[1]
        Cin = sX[1][-1]
        P = N * H * W
        dz, x, dw = _fresh(sDz, _ints(P, g)), _fresh(sX, _ints(P, g)), _fresh(sDw, _zeros)
        C.conv_wgrad(dz, x, dw, scale, ksplit, bn)
        ref, mag = R.conv3x3_wgrad64(dz, x, scale)
        KC.check(dw.reshape(ref.shape), ref, mag, chain=KC.wgrad_chain(N, H, W, Cin, Cout, sms), exact=True,
                 family="conv_wgrad", what=str(sig))
    elif name == "conv0_fprop":
        sX, sW, sBias, sY = args
        x4, w0 = _fresh(sX, _ints(27, g)), _fresh(sW, _ints(27, g))
        bias = _fresh(sBias, lambda n, dt: KC.bias(n, "exact", g, DEV))
        y = _fresh(sY, _zeros)
        C.conv0_fprop(x4, w0, bias, y)
        ref, mag = R.conv0_fprop64(x4, w0.reshape(64, 64), bias)
        KC.check(y.reshape(ref.shape), ref, mag, chain=KC.gemm_chain(64), exact=True, family="conv0_fprop",
                 what=str(sig))
    elif name == "conv0_wgrad":
        sDz, sX, sDw = args
        N, H, W, _ = sX[1]
        P = N * H * W
        dz, x4, dw0 = _fresh(sDz, _ints(P, g)), _fresh(sX, _ints(P, g)), _fresh(sDw, _zeros)
        C.conv0_wgrad(dz, x4, dw0)
        ref, mag = R.conv0_wgrad64(dz, x4)
        KC.check(dw0.reshape(64, 64), ref, mag, chain=KC.conv0_wgrad_chain(P, sms), exact=True,
                 family="conv0_wgrad", what=str(sig))
    elif name == "unpool2x2":
        sDp, sMask, sDz, sCs = args
        N, OH, OW, Cc = sDp[1]
        dp = _fresh(sDp, _ints(1, g))
        idx = torch.randint(0, 4, (N, OH, OW, Cc), device=DEV, generator=g)
        pos = torch.rand(N, OH, OW, Cc, device=DEV, generator=g) < 0.7
        mask = _fresh(sMask, _zeros)
        mask.copy_(R.pool_mask_encode(idx, pos).view(mask.shape))
        dz = _fresh(sDz, _zeros)
        cs = None if sCs is None else _fresh(sCs, _zeros)
        C.unpool2x2(dp, mask, dz, cs)
        want, want_cs, cs_mag = R.unpool2x2_64(dp, idx, pos)
        KC.check(dz, want, want, chain=0, exact=True, family="unpool2x2", what=str(sig))
        if cs is not None:
            KC.check(cs, want_cs, cs_mag, chain=KC.unpool_colsum_chain(N * OH * OW, Cc, sms), exact=False,
                     what=str(sig))
    else:
        raise AssertionError("no replay for %s" % name)


def test_replay_every_wgmma_launch_of_the_engine(capsys):
    from distributed_vgg_f_b200.models.vggf import vgg16_spec, vggf_spec

    configs = [
        (vggf_spec(3), 64, (64, 37), {}),                       # default step, and a ragged last batch of 37
        (vggf_spec(3), 16, (16,), {}),                          # 32-wide GEMM tiles on the FC layers
        (vgg16_spec(1000), 32, (32,), {}),                      # unfused head: GEMM + fc_bias_act + CE
        (vggf_spec(3), 64, (64,), {"B200_FUSE_POOL": "0"}),     # separate conv and pool kernels
    ]
    C, sigs = _record(configs)
    assert sigs
    g = torch.Generator(device=DEV).manual_seed(0)
    sms = KC.sm_count()
    for sig in sigs:
        _replay(C, sig, g, sms)
        torch.cuda.empty_cache()
    kinds = {}
    for s in sigs:
        kinds[s[0]] = kinds.get(s[0], 0) + 1
    with capsys.disabled():
        print("\n[replay] %d launch signatures replayed: %s" % (len(sigs), ", ".join("%s=%d" % kv for kv in
                                                                                      sorted(kinds.items()))))
