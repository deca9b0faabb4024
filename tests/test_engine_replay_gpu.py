"""Every native kernel launch the engine makes, replayed against the float64 reference.

The kernel tests pick their shapes by hand; this one takes them from the engine.  ``ops._C`` is
swapped for a recording proxy during one train_step and one eval_step of several configurations.
Each distinct call signature of a recorded kernel (shapes, strides, dtypes, storage offset
mod 16 elements, scalars, which optional tensors are present) is then run once more in exact mode
on fresh tensors laid out the same way, so the vector-store alignment paths match, and compared
with the reference (exact where the arithmetic allows it, else against kernel_check's bound).  The
optimizer runs on a side stream, so its replay, like every other, uses fresh tensors with the recorded
storage offset mod 16 elements.  When a dispatch rule or a split heuristic of the engine changes, the replay
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
            "unpool2x2", "maxpool_fwd", "maxpool_relu_bwd", "avgpool_fwd", "avgpool_bwd", "bias_grad", "fc_bias_act",
            "fc_grad_act", "cross_entropy", "head_ce", "adam", "sgd", "cast_to_bf16", "nchw_to_nhwc")


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
    for spec, batch, steps, env, kw in configs:
        saved = {k: os.environ.get(k) for k in env}
        os.environ.update(env)
        kw = dict(kw)
        cw = kw.pop("class_weights", None)
        reload = kw.pop("reload", False)
        try:
            eng = NativeEngine(spec, device=torch.device(DEV), batch=batch, seed=0, distributed=False, **kw)
            if cw is not None:
                eng.class_weights = torch.tensor(cw, device=DEV)
            ops._C = rec
            try:
                if reload:                       # loading a checkpoint: the fp32 -> bf16 shadow cast
                    eng.import_state(eng.export_state(), sync=False)
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


def _relu_ints(g):
    return lambda n, dt: torch.relu(torch.randint(-2, 3, (n,), device=DEV, generator=g)).to(dt)


def _gauss(g, scale=1.0):
    return lambda n, dt: (torch.randn(n, device=DEV, generator=g) * scale).to(dt)


def _opt(sig, g, fill):
    return None if sig is None else _fresh(sig, fill)


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
    elif name == "maxpool_fwd":
        x, y = _fresh(args[0], _relu_ints(g)), _fresh(args[1], _zeros)
        C.maxpool_fwd(x, y)
        val, _ = R.maxpool2x2_64(x)
        KC.check(y, val, val, chain=0, exact=True, family="maxpool_fwd", what=str(sig))
    elif name == "maxpool_relu_bwd":
        sY, sDp, sDz, sCs = args
        y, dp, dz, cs = _fresh(sY, _relu_ints(g)), _fresh(sDp, _ints(1, g)), _fresh(sDz, _zeros), _opt(sCs, g, _zeros)
        C.maxpool_relu_bwd(y, dp, dz, cs)
        want, want_cs, cs_mag = R.maxpool2x2_relu_bwd64(y, dp)
        KC.check(dz, want, want, chain=0, exact=True, family="maxpool_relu_bwd", what=str(sig))
        if cs is not None:
            KC.check(cs, want_cs, cs_mag, chain=0, exact=True, family="maxpool_colsum", what=str(sig))
    elif name in ("avgpool_fwd", "avgpool_bwd"):
        src, dst = _fresh(args[0], _ints(16, g)), _fresh(args[1], _zeros)
        getattr(C, name)(src, dst)
        if name == "avgpool_fwd":
            (H, OH), ref = (src.shape[1], dst.shape[1]), R.adaptive_avgpool64(src, dst.shape[1], dst.shape[2])
            terms = R.ap_max_window(H, OH) ** 2
        else:
            (H, OH), ref = (dst.shape[1], src.shape[1]), R.adaptive_avgpool_bwd64(src, dst.shape[1], dst.shape[2])
            terms = R.ap_max_cover(H, OH) ** 2
        sizes = {b - a for a, b in R._ap_windows(H, OH)}
        KC.check(dst, *ref, chain=KC.avgpool_chain(terms), exact=all(v & (v - 1) == 0 for v in sizes), family=name,
                 what=str(sig))
    elif name == "bias_grad":
        sDz, sDb, rows, Cc, ld, scale = args
        dz, db = _fresh(sDz, _ints(rows, g)), _fresh(sDb, _zeros)
        C.bias_grad(dz, db, rows, Cc, ld, scale)
        ref, mag = R.bias_grad64(dz.reshape(-1)[:rows * ld].view(rows, ld), Cc, scale)
        exact = float(scale) == 2.0 ** round(__import__("math").log2(scale))
        KC.check(db[:Cc], ref, mag, chain=KC.bias_grad_chain(rows, Cc, sms, ld), exact=exact, family="bias_grad",
                 what=str(sig))
    elif name == "fc_bias_act":
        sAcc, sBias, sY, sYf, B, N, relu, p, seed, offset, clear = args
        acc = _fresh(sAcc, _ints(1, g))
        bias = _opt(sBias, g, lambda n, dt: KC.bias(n, "exact", g, DEV))
        y, yf = _opt(sY, g, _zeros), _opt(sYf, g, _zeros)
        a0 = acc.reshape(-1)[:B * N].view(B, N).clone()
        C.fc_bias_act(acc, bias, y, yf, B, N, relu, p, seed, offset, clear)
        ref, mag = R.fc_bias_act64(a0, None if bias is None else bias[:N], relu=relu, drop_p=p, seed=seed,
                                   offset=offset)
        for out in (y, yf):
            if out is not None:
                KC.check(out.reshape(-1)[:B * N].view(B, N), ref, mag, chain=0, exact=True, family="fc_bias_act",
                         what=str(sig))
    elif name == "fc_grad_act":
        sAcc, sAct, sDz, B, N, relu, p, clear = args
        acc, act, dz = _fresh(sAcc, _ints(1, g)), _opt(sAct, g, _relu_ints(g)), _fresh(sDz, _zeros)
        a0 = acc.reshape(-1)[:B * N].view(B, N).clone()
        C.fc_grad_act(acc, act, dz, B, N, relu, p, clear)
        ref, mag = R.fc_grad_act64(a0, None if act is None else act.reshape(-1)[:B * N].view(B, N), relu=relu,
                                   drop_p=p)
        KC.check(dz.reshape(-1)[:B * N].view(B, N), ref, mag, chain=0, exact=True, family="fc_grad_act", what=str(sig))
    elif name in ("cross_entropy", "head_ce"):
        if name == "cross_entropy":
            sZ, sT, sDl, ldd, sMeter, sLoss, grad_scale, sCw = args
            z = _fresh(sZ, _gauss(g, 3.0))
            B, Cc = z.shape
        else:
            (sH, sW, sBias, sT, sZ, sDl, ldd, sDW, sDb, sDh, drop_scale, relu, sMeter, sLoss, sCw) = args
            h, W = _fresh(sH, _relu_ints(g)), _fresh(sW, _gauss(g, 0.1))
            bias = _fresh(sBias, _gauss(g, 0.1))
            B, Cc = sZ[1]
        t = _fresh(sT, lambda n, dt: torch.randint(0, Cc, (n,), device=DEV, generator=g))
        cw = _opt(sCw, g, lambda n, dt: torch.rand(n, device=DEV, generator=g) + 0.1)
        dl, meter, loss = _opt(sDl, g, _zeros), _opt(sMeter, g, _zeros), _opt(sLoss, g, _zeros)
        if name == "cross_entropy":
            C.cross_entropy(z, t, dl, ldd, meter, loss, grad_scale, cw)
            se_chain, warps = -(-Cc // 32) + 5, 32
        else:
            z = _fresh(sZ, _zeros)
            dW, db, dh = _opt(sDW, g, _zeros), _opt(sDb, g, _zeros), _opt(sDh, g, _zeros)
            C.head_ce(h, W, bias, t, z, dl, ldd, dW, db, dh, drop_scale, relu, meter, loss, cw)
            grad_scale = None
        ref = R.cross_entropy64(z, t, ldd=ldd, class_weights=cw, grad_scale=grad_scale)
        bnd = KC.ce_bound(z, t, class_weights=cw, grad_scale=None if cw is not None else
                          (1.0 / B if grad_scale is None else grad_scale), se_chain=se_chain if name == "cross_entropy"
                          else Cc, warps=warps if name == "cross_entropy" else 16)
        if loss is not None:
            KC.check(loss, ref["loss"].view(1), torch.zeros(1, dtype=torch.float64, device=DEV), chain=0, exact=False,
                     err=bnd["loss"].view(1), family=name + "_loss", what=str(sig))
        if dl is not None:
            err = torch.zeros(B, ldd, dtype=torch.float64, device=DEV)
            err[:, :Cc] = bnd["dlogits"]
            KC.check(dl.reshape(-1)[:B * ldd].view(B, ldd), ref["dlogits"], torch.zeros_like(err), chain=0,
                     exact=False, err=err, family=name + "_dlogits", what=str(sig))
        if meter is not None:
            assert float(meter[1]) == float(ref["meter"][1]) and float(meter[2]) == B, str(sig)
        if name == "head_ce":
            chain = KC.head_chain(h.shape[1], B)
            part = R.head_ce64(h, W, bias, dl_used=dl.reshape(-1)[:B * ldd].view(B, ldd)[:, :Cc] if dl is not None
                               else torch.zeros(B, Cc, device=DEV), drop_scale=drop_scale, relu=relu)
            KC.check(z, *part["logits"], chain=chain["logits"], exact=False, family="head_logits", what=str(sig))
            if dW is not None:
                KC.check(dW.reshape(Cc, -1), *part["dW"], chain=chain["dW"], exact=False, family="head_dW",
                         what=str(sig))
                KC.check(db.reshape(-1), *part["db"], chain=chain["db"], exact=False, family="head_db", what=str(sig))
            if dh is not None:
                KC.check(dh.reshape(B, -1), *part["dh"], chain=chain["dh"], exact=False, family="head_dh",
                         what=str(sig))
    elif name in ("adam", "sgd"):
        if name == "adam":
            sP, sM, sV, sG32, sG16, sSh, lr, b1, b2, eps, wd, step, gscale, sZero = args
        else:
            sP, sM, sG32, sG16, sSh, lr, mo, wd, first, gscale, sZero = args
        p, m = _fresh(sP, _gauss(g)), _fresh(sM, _gauss(g, 1e-3))
        v = _fresh(sV, lambda n, dt: torch.rand(n, device=DEV, generator=g) * 1e-6) if name == "adam" else None
        g32, g16 = _opt(sG32, g, _gauss(g, 1e-2)), _opt(sG16, g, _gauss(g, 1e-2))
        shadow = _opt(sSh, g, _zeros)
        zero = g32 if (sZero is not None and sZero == sG32) else _opt(sZero, g, _gauss(g))
        grad = (g32 if g32 is not None else g16).clone()
        p0, m0 = p.clone(), m.clone()
        if name == "adam":
            v0 = v.clone()
            C.adam(p, m, v, g32, g16, shadow, lr, b1, b2, eps, wd, step, gscale, zero)
            ref = R.adam_step64(p0, m0, v0, grad, lr=R._f32(lr), beta1=R._f32(b1), beta2=R._f32(b2), eps=R._f32(eps),
                                weight_decay=R._f32(wd), step=step, grad_scale=R._f32(gscale))
            outs = ((p, "p"), (m, "m"), (v, "v"))
        else:
            C.sgd(p, m, g32, g16, shadow, lr, mo, wd, first, gscale, zero)
            ref = R.sgd_step64(p0, m0, grad, lr=R._f32(lr), momentum=R._f32(mo), weight_decay=R._f32(wd), first=first,
                               grad_scale=R._f32(gscale))
            outs = ((p, "p"), (m, "buf"))
        for got, key in outs:
            r, e = ref[key]
            KC.check(got, r, torch.zeros_like(r), chain=0, exact=False, err=e, family="%s_%s" % (name, key),
                     what=str(sig))
        if shadow is not None:
            KC.check(shadow, p.double(), p.double(), chain=0, exact=True, family=name + "_shadow", what=str(sig))
        if zero is not None:
            assert torch.count_nonzero(zero) == 0, str(sig)
    elif name == "cast_to_bf16":
        x, y = _fresh(args[0], _gauss(g)), _fresh(args[1], _zeros)
        C.cast_to_bf16(x, y)
        KC.check(y, x.double(), x.double(), chain=0, exact=True, family="cast_to_bf16", what=str(sig))
    elif name == "nchw_to_nhwc":
        x, y = _fresh(args[0], _gauss(g)), _fresh(args[1], lambda n, dt: torch.full((n,), 7.0, device=DEV).to(dt))
        C.nchw_to_nhwc(x, y)
        ref, mag = R.nchw_to_nhwc64(x, y.shape[3])
        KC.check(y, ref, mag, chain=0, exact=True, family="nchw_to_nhwc", what=str(sig))
    else:
        raise AssertionError("no replay for %s" % name)


def test_replay_every_wgmma_launch_of_the_engine(capsys):
    from distributed_vgg_f_b200.models.vggf import vgg16_spec, vggf_spec

    configs = [
        (vggf_spec(3), 64, (64, 37), {}, {}),                   # default step, and a ragged last batch of 37
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
