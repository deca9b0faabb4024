"""Record the native kernel launches of the engine and replay each call signature on guarded operands.

``_record`` swaps ``ops._C`` for a recording proxy during training and evaluation steps of several
engine configurations and keeps each distinct call signature of a ``RECORDED`` kernel (shapes,
strides, dtypes, storage offset mod 16 elements, scalars, which optional tensors are present).
``_replay`` runs one signature once more in exact mode, on fresh guarded operands laid out the same
way (guarded.py), and checks both:

* the values, against the float64 references of ops.ref (exact where the arithmetic allows it, else
  against kernel_check's bound);
* the footprint, against ``CONTRACT``: what the kernel may do to each of its tensor arguments.

The contract is derived from the kernels, not from what the tests pass:

* ``READ``   read-only: the operand, its guards and gaps are bitwise unchanged;
* ``STORE``  every element is written: pre-filled with NaN (-1 for int32 words), so an element the
             kernel skips fails the value check;
* ``ACCUM``  added to (red.add / atomicAdd / ``+=``): pre-filled with integers in [-8, 8] and checked
             against prefill + reference, so a store instead of an add fails;
* ``UPDATE`` read, then written in place (optimizer state, a cleared accumulator).

Only the region a kernel writes is exempt from the footprint check, e.g. the first B x N elements
of an FC accumulator, ``meter[:3]``, the ``rows x cols`` at stride ``ldo`` of a GEMM output.
"""
import os

import torch

import guarded as G
import kernel_check as KC
from distributed_vgg_f_b200.ops import ref as R

DEV = "cuda"

READ, STORE, ACCUM, UPDATE = "read-only", "stored", "accumulated", "updated"


def _gemm_out(sc):
    return ACCUM if sc["atomic"] else STORE


def _cleared(sc):
    return UPDATE if sc["clear"] else READ


# One row per recorded kernel: tensor argument -> what the kernel does to it.  A callable takes the
# call's scalars.
CONTRACT = {
    "gemm": {"A": READ, "B": READ, "out": _gemm_out, "bias": READ},         # atomic epilogues red.add
    "conv_fprop": {"x": READ, "w": READ, "bias": READ, "y": STORE},
    "conv_fprop_pool": {"x": READ, "w": READ, "bias": READ, "pooled": STORE, "mask": STORE},  # all 4 words
    "conv_dgrad": {"dz": READ, "w": READ, "mask_src": READ, "dx": STORE, "colsum": ACCUM},
    "conv_wgrad": {"dz": READ, "x": READ, "dw": ACCUM},
    "conv0_fprop": {"x4": READ, "w0": READ, "bias": READ, "y": STORE},
    "conv0_wgrad": {"dz": READ, "x4": READ, "dw0": ACCUM},
    "unpool2x2": {"dp": READ, "mask": READ, "dz": STORE, "colsum": ACCUM},
    "maxpool_fwd": {"x": READ, "y": STORE},
    "maxpool_relu_bwd": {"y": READ, "dp": READ, "dz": STORE, "colsum": ACCUM},
    "avgpool_fwd": {"x": READ, "y": STORE},
    "avgpool_bwd": {"dy": READ, "dx": STORE},
    "bias_grad": {"dz": READ, "db": ACCUM},
    "fc_bias_act": {"acc": _cleared, "bias": READ, "y": STORE, "y_f32": STORE},
    "fc_grad_act": {"acc": _cleared, "act": READ, "dz": STORE},
    # dlogits: the padding columns [C, ldd) are stored as zeros by design
    "cross_entropy": {"logits": READ, "target": READ, "dlogits": STORE, "meter": ACCUM, "loss": STORE,
                      "class_weights": READ},
    "head_ce": {"h": READ, "W": READ, "bias": READ, "target": READ, "logits": STORE, "dlogits": STORE,
                "dW": STORE, "db": ACCUM, "dh": STORE, "meter": ACCUM, "loss": STORE, "class_weights": READ},
    # the shadow is stored, the gradient range named by `zero` cleared (it may be g32 itself)
    "adam": {"p": UPDATE, "m": UPDATE, "v": UPDATE, "g32": READ, "g16": READ, "shadow": STORE, "zero": UPDATE},
    "sgd": {"p": UPDATE, "mom": UPDATE, "g32": READ, "g16": READ, "shadow": STORE, "zero": UPDATE},
    "cast_to_bf16": {"x": READ, "y": STORE},
    "nchw_to_nhwc": {"x": READ, "y": STORE},                    # the padding channels are stored as zeros
    "augment": {"src": READ, "params": READ, "out": STORE},     # NHWC: the padding channels as zeros
}
RECORDED = ("gemm", "conv_fprop", "conv_fprop_pool", "conv_dgrad", "conv_wgrad", "conv0_fprop", "conv0_wgrad",
            "unpool2x2", "maxpool_fwd", "maxpool_relu_bwd", "avgpool_fwd", "avgpool_bwd", "bias_grad", "fc_bias_act",
            "fc_grad_act", "cross_entropy", "head_ce", "adam", "sgd", "cast_to_bf16", "nchw_to_nhwc", "augment")
# in-range crop box (top, left, height, width, cos, sin, flip, -): the poison of augment parameters
CROP_POISON = torch.tensor([0.0, 0.0, 1.0, 1.0, 1.0, 0.0, 0.0, 0.0])


def _sig(a):
    if isinstance(a, torch.Tensor):
        return ("T", tuple(a.shape), tuple(a.stride()), a.dtype, a.storage_offset() % 16)
    if isinstance(a, list):
        return tuple(a)
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


def _batch(spec, eng, b, fused):
    if not fused:
        g = torch.Generator(device=DEV).manual_seed(b)
        x = torch.randn(b, 3, eng.HW, eng.HW, device=DEV, generator=g)
        return x, torch.randint(0, spec.num_classes, (b,), device=DEV, generator=g)
    from distributed_vgg_f_b200.data import transforms as T
    from distributed_vgg_f_b200.data.loader import FusedBatch
    from distributed_vgg_f_b200.data.synthetic import synthetic_uint8_batch

    imgs, labels = synthetic_uint8_batch(b, 128, spec.num_classes, seed=b)
    return FusedBatch(torch.from_numpy(imgs), T.sample_train_params(b, 128, 128, torch.Generator().manual_seed(b)),
                      torch.from_numpy(labels), (256, 256), None)


def _record(configs):
    """configs: (spec, batch, step batch sizes, environment, engine keywords); the keywords may add
    class_weights, reload (a checkpoint round trip first) and fused (uint8 images + augment)."""
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
        fused = kw.pop("fused", False)
        try:
            eng = NativeEngine(spec, device=torch.device(DEV), batch=batch, seed=0, distributed=False, **kw)
            if cw is not None:
                eng.class_weights = torch.tensor(cw, device=DEV)
            ops._C = rec
            try:
                if reload:                       # loading a checkpoint: the fp32 -> bf16 shadow cast
                    eng.import_state(eng.export_state(), sync=False)
                for b in steps:
                    eng.train_step(_batch(spec, eng, b, fused))
                    eng.eval_step(_batch(spec, eng, b, fused))
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


# ------------------------------------------------------------------------------------- fills
def _ints(depth, g):
    return lambda n, dt: KC.operand((n,), "exact", depth, g, DEV).to(dt)


def _relu_ints(g):
    return lambda n, dt: torch.relu(torch.randint(-2, 3, (n,), device=DEV, generator=g)).to(dt)


def _gauss(g, scale=1.0):
    return lambda n, dt: (torch.randn(n, device=DEV, generator=g) * scale).to(dt)


def _bias(g):
    return lambda n, dt: KC.bias(n, "exact", g, DEV)


class _Call:
    """The guarded operands of one replayed call, allocated by their role in CONTRACT."""

    def __init__(self, name, g, **scalars):
        self.name, self.g, self.sc = name, g, scalars
        self.ops, self.pre = {}, {}

    def __call__(self, key, s, fill=None, poison=G.NAN, role=None):
        if s is None:
            return None
        _, shape, stride, dtype, off = s
        role = role or CONTRACT[self.name][key]
        role = role(self.sc) if callable(role) else role
        n = 1
        for d in shape:
            n *= d
        if role == STORE:
            values = None
            if dtype == torch.int32:
                poison = -1
        elif role == ACCUM:
            values = torch.randint(-8, 9, (n,), device=DEV, generator=self.g).to(dtype)
        else:
            values = fill(n, dtype)
        op = G.guarded(shape, stride, dtype, off, poison, DEV, values)
        self.ops[key] = (role, op)
        if role == ACCUM:
            self.pre[key] = op.t.clone()
        return op.t

    def seal(self):
        for _, op in self.ops.values():
            op.seal()

    def footprint(self, what, **regions):
        """Nothing outside what the contract lets the kernel write changed.  ``regions`` narrows
        the written region of an argument to a view of it."""
        for key, (role, op) in self.ops.items():
            written = () if role == READ else (regions.get(key, op.t),)
            op.check(written, what="%s %s (%s) %s" % (self.name, key, role, what))


def _plus(pre, ref, mag):
    """Reference and magnitude of an accumulation target pre-filled with ``pre``."""
    p = pre.to(torch.float64).reshape(ref.shape)
    return ref + p, mag + p.abs()


def _flat(t, n):
    return t.reshape(-1)[:n]


def _replay(C, sig, g, sms):
    name, args = sig[0], sig[1:]
    what = str(sig)
    if name == "gemm":
        sA, a_mn, sB, b_mn, M, N, K, sOut, ldo, code, sBias, alpha, ksplit, bn = args
        epi = {C.EPI_F32_STORE: "f32_store", C.EPI_F32_ATOMIC: "f32_atomic", C.EPI_F32_ATOMIC_T: "f32_atomic_t",
               C.EPI_BF16_BIAS_RELU: "bf16_bias_relu", C.EPI_F32_STORE_T: "f32_store_t",
               C.EPI_BF16_STORE: "bf16_store"}[code]
        c = _Call(name, g, atomic="atomic" in epi)
        A, B, out = c("A", sA, _ints(K, g)), c("B", sB, _ints(K, g)), c("out", sOut)
        bias = c("bias", sBias, _bias(g))
        c.seal()
        C.gemm(A, a_mn, B, b_mn, M, N, K, out, ldo, code, bias, alpha, ksplit, bn)
        ref, mag = R.gemm64(A, B, M=M, N=N, K=K, a_mn=a_mn, b_mn=b_mn, epi=epi, bias=bias, alpha=alpha)
        got = out.as_strided(tuple(ref.shape), (ldo, 1), out.storage_offset())
        if "out" in c.pre:
            ref, mag = _plus(c.pre["out"].as_strided(tuple(ref.shape), (ldo, 1), 0), ref, mag)
        KC.check(got, ref, mag, chain=KC.gemm_chain(K, ksplit) + 1, exact=True, family="gemm", what=what)
        c.footprint(what, out=got)
    elif name in ("conv_fprop", "conv_fprop_pool"):
        sX, sW, sBias = args[:3]
        N, H, W, Cin = sX[1]
        c = _Call(name, g)
        x, w = c("x", sX, _ints(9 * Cin, g)), c("w", sW, _ints(9 * Cin, g))
        Cout = w.numel() // (9 * Cin)
        bias = c("bias", sBias, _bias(g))
        if name == "conv_fprop":
            y = c("y", args[3])
            c.seal()
            C.conv_fprop(x, w, bias, y, args[4], args[5])
        else:
            p, mask = c("pooled", args[3]), c("mask", args[4])
            c.seal()
            C.conv_fprop_pool(x, w, bias, p, mask, args[5])
        ref, mag = R.conv3x3_fprop64(x, w.reshape(Cout, 3, 3, Cin), bias, relu=True if name == "conv_fprop_pool"
                                     else args[4])
        if name == "conv_fprop":
            KC.check(y.reshape(N, H, W, Cout), ref, mag, chain=KC.conv_chain(Cin), exact=True, family="conv_fprop",
                     what=what)
        else:
            KC.check_pool(p, mask, ref, mag, chain=KC.conv_chain(Cin), exact=True, what=what)
            assert not bool(mask.reshape(-1, 4)[:, 3].any()), what + ": mask word 3 not written as 0"
        c.footprint(what)
    elif name == "conv_dgrad":
        sDz, sW, sMask, sDx, sCs, bn = args
        N, H, W, Cout = sDz[1]
        Cin = sDx[1][-1]
        c = _Call(name, g)
        dz, w = c("dz", sDz, _ints(9 * Cout, g)), c("w", sW, _ints(9 * Cout, g))
        mask = c("mask_src", sMask, _ints(1, g))
        dx, cs = c("dx", sDx), c("colsum", sCs)
        c.seal()
        C.conv_dgrad(dz, w, mask, dx, cs, bn)
        ref, mag = R.conv3x3_dgrad64(dz, w.reshape(Cout, 3, 3, Cin), mask_src=mask)
        KC.check(dx, ref, mag, chain=KC.conv_chain(Cout), exact=True, family="conv_dgrad", what=what)
        if cs is not None:
            st = dx.to(torch.float64).reshape(-1, Cin)
            KC.check(cs[:Cin], *_plus(c.pre["colsum"][:Cin], st.sum(0), st.abs().sum(0)),
                     chain=KC.conv_colsum_chain(N * H * W, Cin, sms) + 1, exact=False, what=what)
        c.footprint(what, colsum=None if cs is None else cs[:Cin])
    elif name == "conv_wgrad":
        sDz, sX, sDw, scale, ksplit, bn = args
        N, H, W, Cout = sDz[1]
        Cin = sX[1][-1]
        P = N * H * W
        c = _Call(name, g)
        dz, x, dw = c("dz", sDz, _ints(P, g)), c("x", sX, _ints(P, g)), c("dw", sDw)
        c.seal()
        C.conv_wgrad(dz, x, dw, scale, ksplit, bn)
        ref, mag = R.conv3x3_wgrad64(dz, x, scale)
        KC.check(dw.reshape(ref.shape), *_plus(c.pre["dw"], ref, mag), chain=KC.wgrad_chain(N, H, W, Cin, Cout, sms) + 1,
                 exact=True, family="conv_wgrad", what=what)
        c.footprint(what)
    elif name == "conv0_fprop":
        sX, sW, sBias, sY = args
        c = _Call(name, g)
        x4, w0 = c("x4", sX, _ints(27, g)), c("w0", sW, _ints(27, g))
        bias, y = c("bias", sBias, _bias(g)), c("y", sY)
        c.seal()
        C.conv0_fprop(x4, w0, bias, y)
        ref, mag = R.conv0_fprop64(x4, w0.reshape(64, 64), bias)
        KC.check(y.reshape(ref.shape), ref, mag, chain=KC.gemm_chain(64), exact=True, family="conv0_fprop", what=what)
        c.footprint(what)
    elif name == "conv0_wgrad":
        sDz, sX, sDw = args
        N, H, W, _ = sX[1]
        P = N * H * W
        c = _Call(name, g)
        dz, x4, dw0 = c("dz", sDz, _ints(P, g)), c("x4", sX, _ints(P, g)), c("dw0", sDw)
        c.seal()
        C.conv0_wgrad(dz, x4, dw0)
        ref, mag = R.conv0_wgrad64(dz, x4)
        KC.check(dw0.reshape(64, 64), *_plus(c.pre["dw0"], ref, mag), chain=KC.conv0_wgrad_chain(P, sms) + 1,
                 exact=True, family="conv0_wgrad", what=what)
        c.footprint(what)
    elif name == "unpool2x2":
        sDp, sMask, sDz, sCs = args
        N, OH, OW, Cc = sDp[1]
        idx = torch.randint(0, 4, (N, OH, OW, Cc), device=DEV, generator=g)
        pos = torch.rand(N, OH, OW, Cc, device=DEV, generator=g) < 0.7
        words = R.pool_mask_encode(idx, pos).to(torch.int32)
        c = _Call(name, g)
        dp = c("dp", sDp, _ints(1, g))
        mask = c("mask", sMask, lambda n, dt: words.reshape(-1), poison=-1)
        dz, cs = c("dz", sDz), c("colsum", sCs)
        c.seal()
        C.unpool2x2(dp, mask, dz, cs)
        want, want_cs, cs_mag = R.unpool2x2_64(dp, idx, pos)
        KC.check(dz, want, want, chain=0, exact=True, family="unpool2x2", what=what)
        if cs is not None:
            KC.check(cs[:Cc], *_plus(c.pre["colsum"][:Cc], want_cs, cs_mag),
                     chain=KC.unpool_colsum_chain(N * OH * OW, Cc, sms) + 1, exact=False, what=what)
        c.footprint(what, colsum=None if cs is None else cs[:Cc])
    elif name == "maxpool_fwd":
        c = _Call(name, g)
        x, y = c("x", args[0], _relu_ints(g), poison=G.fmax(torch.bfloat16)), c("y", args[1])
        c.seal()
        C.maxpool_fwd(x, y)
        val, _ = R.maxpool2x2_64(x)
        KC.check(y, val, val, chain=0, exact=True, family="maxpool_fwd", what=what)
        c.footprint(what)
    elif name == "maxpool_relu_bwd":
        sY, sDp, sDz, sCs = args
        c = _Call(name, g)
        y = c("y", sY, _relu_ints(g), poison=G.fmax(torch.bfloat16))
        dp, dz, cs = c("dp", sDp, _ints(1, g)), c("dz", sDz), c("colsum", sCs)
        c.seal()
        C.maxpool_relu_bwd(y, dp, dz, cs)
        want, want_cs, cs_mag = R.maxpool2x2_relu_bwd64(y, dp)
        KC.check(dz, want, want, chain=0, exact=True, family="maxpool_relu_bwd", what=what)
        Cc = y.shape[3]
        if cs is not None:
            KC.check(cs[:Cc], *_plus(c.pre["colsum"][:Cc], want_cs, cs_mag), chain=0, exact=True,
                     family="maxpool_colsum", what=what)
        c.footprint(what, colsum=None if cs is None else cs[:Cc])
    elif name in ("avgpool_fwd", "avgpool_bwd"):
        c = _Call(name, g)
        src_key, dst_key = ("x", "y") if name == "avgpool_fwd" else ("dy", "dx")
        src, dst = c(src_key, args[0], _ints(16, g)), c(dst_key, args[1])
        c.seal()
        getattr(C, name)(src, dst)
        if name == "avgpool_fwd":
            (H, OH), ref = (src.shape[1], dst.shape[1]), R.adaptive_avgpool64(src, dst.shape[1], dst.shape[2])
            terms = R.ap_max_window(H, OH) ** 2
        else:
            (H, OH), ref = (dst.shape[1], src.shape[1]), R.adaptive_avgpool_bwd64(src, dst.shape[1], dst.shape[2])
            terms = R.ap_max_cover(H, OH) ** 2
        sizes = {b - a for a, b in R._ap_windows(H, OH)}
        KC.check(dst, *ref, chain=KC.avgpool_chain(terms), exact=all(v & (v - 1) == 0 for v in sizes), family=name,
                 what=what)
        c.footprint(what)
    elif name == "bias_grad":
        sDz, sDb, rows, Cc, ld, scale = args
        c = _Call(name, g)
        dz, db = c("dz", sDz, _ints(rows, g)), c("db", sDb)
        c.seal()
        C.bias_grad(dz, db, rows, Cc, ld, scale)
        ref, mag = R.bias_grad64(dz.reshape(-1)[:rows * ld].view(rows, ld), Cc, scale)
        exact = float(scale) == 2.0 ** round(__import__("math").log2(scale))
        KC.check(db[:Cc], *_plus(c.pre["db"][:Cc], ref, mag), chain=KC.bias_grad_chain(rows, Cc, sms, ld) + 1,
                 exact=exact, family="bias_grad", what=what)
        c.footprint(what, db=db[:Cc])
    elif name == "fc_bias_act":
        sAcc, sBias, sY, sYf, B, N, relu, p, seed, offset, clear = args
        c = _Call(name, g, clear=clear)
        acc = c("acc", sAcc, _ints(1, g))
        bias = c("bias", sBias, _bias(g))
        y, yf = c("y", sY), c("y_f32", sYf)
        a0 = _flat(acc, B * N).view(B, N).clone()
        c.seal()
        C.fc_bias_act(acc, bias, y, yf, B, N, relu, p, seed, offset, clear)
        ref, mag = R.fc_bias_act64(a0, None if bias is None else bias[:N], relu=relu, drop_p=p, seed=seed,
                                   offset=offset)
        for out in (y, yf):
            if out is not None:
                KC.check(_flat(out, B * N).view(B, N), ref, mag, chain=0, exact=True, family="fc_bias_act", what=what)
        if clear:
            assert torch.count_nonzero(_flat(acc, B * N)) == 0, what + ": acc not cleared"
        c.footprint(what, acc=_flat(acc, B * N), y=None if y is None else _flat(y, B * N),
                    y_f32=None if yf is None else _flat(yf, B * N))
    elif name == "fc_grad_act":
        sAcc, sAct, sDz, B, N, relu, p, clear = args
        c = _Call(name, g, clear=clear)
        acc, act, dz = c("acc", sAcc, _ints(1, g)), c("act", sAct, _relu_ints(g)), c("dz", sDz)
        a0 = _flat(acc, B * N).view(B, N).clone()
        c.seal()
        C.fc_grad_act(acc, act, dz, B, N, relu, p, clear)
        ref, mag = R.fc_grad_act64(a0, None if act is None else _flat(act, B * N).view(B, N), relu=relu, drop_p=p)
        KC.check(_flat(dz, B * N).view(B, N), ref, mag, chain=0, exact=True, family="fc_grad_act", what=what)
        if clear:
            assert torch.count_nonzero(_flat(acc, B * N)) == 0, what + ": acc not cleared"
        c.footprint(what, acc=_flat(acc, B * N), dz=_flat(dz, B * N))
    elif name in ("cross_entropy", "head_ce"):
        c = _Call(name, g)
        if name == "cross_entropy":
            sZ, sT, sDl, ldd, sMeter, sLoss, grad_scale, sCw = args
            z = c("logits", sZ, _gauss(g, 3.0), poison=G.fmax(torch.float32))
            B, Cc = z.shape
        else:
            (sH, sW, sBias, sT, sZ, sDl, ldd, sDW, sDb, sDh, drop_scale, relu, sMeter, sLoss, sCw) = args
            h, W = c("h", sH, _relu_ints(g)), c("W", sW, _gauss(g, 0.1))
            bias = c("bias", sBias, _gauss(g, 0.1))
            B, Cc = sZ[1]
        t = c("target", sT, lambda n, dt: torch.randint(0, Cc, (n,), device=DEV, generator=g), poison=Cc - 1)
        cw = c("class_weights", sCw, lambda n, dt: torch.rand(n, device=DEV, generator=g) + 0.1)
        dl, meter, loss = c("dlogits", sDl), c("meter", sMeter), c("loss", sLoss)
        regions = {"meter": None if meter is None else meter[:3], "loss": None if loss is None else loss[:1],
                   "dlogits": None if dl is None else _flat(dl, B * ldd)}
        if name == "cross_entropy":
            c.seal()
            C.cross_entropy(z, t, dl, ldd, meter, loss, grad_scale, cw)
            se_chain, warps = -(-Cc // 32) + 5, 32
        else:
            z = c("logits", sZ)
            dW, db, dh = c("dW", sDW), c("db", sDb), c("dh", sDh)
            K = h.shape[1]
            regions.update(logits=_flat(z, B * Cc), dW=None if dW is None else _flat(dW, Cc * K),
                           db=None if db is None else db[:Cc], dh=None if dh is None else _flat(dh, B * K))
            c.seal()
            C.head_ce(h, W, bias, t, z, dl, ldd, dW, db, dh, drop_scale, relu, meter, loss, cw)
            grad_scale = None
        ref = R.cross_entropy64(z, t, ldd=ldd, class_weights=cw, grad_scale=grad_scale)
        bnd = KC.ce_bound(z, t, class_weights=cw, grad_scale=None if cw is not None else
                          (1.0 / B if grad_scale is None else grad_scale), se_chain=se_chain if name == "cross_entropy"
                          else Cc, warps=warps if name == "cross_entropy" else 16)
        if loss is not None:
            KC.check(loss[:1], ref["loss"].view(1), torch.zeros(1, dtype=torch.float64, device=DEV), chain=0,
                     exact=False, err=bnd["loss"].view(1), family=name + "_loss", what=what)
        if dl is not None:
            err = torch.zeros(B, ldd, dtype=torch.float64, device=DEV)
            err[:, :Cc] = bnd["dlogits"]
            KC.check(_flat(dl, B * ldd).view(B, ldd), ref["dlogits"], torch.zeros_like(err), chain=0,
                     exact=False, err=err, family=name + "_dlogits", what=what)
        if meter is not None:
            m0 = c.pre["meter"]
            assert float(meter[1]) == float(m0[1]) + float(ref["meter"][1]), what + ": meter[1] not accumulated"
            assert float(meter[2]) == float(m0[2]) + B, what + ": meter[2] not accumulated"
        if name == "head_ce":
            chain = KC.head_chain(h.shape[1], B)
            part = R.head_ce64(h, W, bias, dl_used=_flat(dl, B * ldd).view(B, ldd)[:, :Cc] if dl is not None
                               else torch.zeros(B, Cc, device=DEV), drop_scale=drop_scale, relu=relu)
            KC.check(z, *part["logits"], chain=chain["logits"], exact=False, family="head_logits", what=what)
            if dW is not None:
                KC.check(_flat(dW, Cc * K).view(Cc, K), *part["dW"], chain=chain["dW"], exact=False, family="head_dW",
                         what=what)
                KC.check(db[:Cc], *_plus(c.pre["db"][:Cc], *part["db"]), chain=chain["db"], exact=False,
                         family="head_db", what=what)
            if dh is not None:
                KC.check(_flat(dh, B * K).view(B, K), *part["dh"], chain=chain["dh"], exact=False, family="head_dh",
                         what=what)
        c.footprint(what, **{k: v for k, v in regions.items() if v is not None})
    elif name in ("adam", "sgd"):
        if name == "adam":
            sP, sM, sV, sG32, sG16, sSh, lr, b1, b2, eps, wd, step, gscale, sZero = args
        else:
            sP, sM, sG32, sG16, sSh, lr, mo, wd, first, gscale, sZero = args
        c = _Call(name, g)
        same = sZero is not None and sZero == sG32      # the engine clears the gradient it reads
        p, m = c("p", sP, _gauss(g)), c("m" if name == "adam" else "mom", sM, _gauss(g, 1e-3))
        v = c("v", sV, lambda n, dt: torch.rand(n, device=DEV, generator=g) * 1e-6) if name == "adam" else None
        g32 = c("g32", sG32, _gauss(g, 1e-2), role=UPDATE if same else None)
        g16 = c("g16", sG16, _gauss(g, 1e-2))
        shadow = c("shadow", sSh)
        zero = g32 if same else c("zero", sZero, _gauss(g))
        grad = (g32 if g32 is not None else g16).clone()
        p0, m0 = p.clone(), m.clone()
        c.seal()
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
            KC.check(got, r, torch.zeros_like(r), chain=0, exact=False, err=e, family="%s_%s" % (name, key), what=what)
        if shadow is not None:
            KC.check(shadow, p.double(), p.double(), chain=0, exact=True, family=name + "_shadow", what=what)
        if zero is not None:
            assert torch.count_nonzero(zero) == 0, what
        c.footprint(what)
    elif name == "cast_to_bf16":
        c = _Call(name, g)
        x, y = c("x", args[0], _gauss(g)), c("y", args[1])
        c.seal()
        C.cast_to_bf16(x, y)
        KC.check(y, x.double(), x.double(), chain=0, exact=True, family="cast_to_bf16", what=what)
        c.footprint(what)
    elif name == "nchw_to_nhwc":
        c = _Call(name, g)
        x, y = c("x", args[0], _gauss(g)), c("y", args[1])
        c.seal()
        C.nchw_to_nhwc(x, y)
        ref, mag = R.nchw_to_nhwc64(x, y.shape[3])
        KC.check(y, ref, mag, chain=0, exact=True, family="nchw_to_nhwc", what=what)
        c.footprint(what)
    elif name == "augment":
        _replay_augment(C, sig, g)
    else:
        raise AssertionError("no replay for %s" % name)


def _replay_augment(C, sig, g):
    """augment is a pure function of each output pixel: the guarded launch must equal the same launch
    on tightly allocated tensors bit for bit, and stay within the tolerance of
    test_kernels_gpu.py::test_augment_matches_reference against augment_reference."""
    from distributed_vgg_f_b200.data import transforms as T
    from distributed_vgg_f_b200.data.synthetic import synthetic_uint8_batch

    sSrc, sPrm, sOut, RH, RW, OH, OW, mode, pad, mean, std = sig[1:]
    what = str(sig)
    N, SH, SW, _ = sSrc[1]
    assert SH == SW and OH == OW and mode == 0, what
    imgs = torch.from_numpy(synthetic_uint8_batch(N, SH, seed=N)[0]).to(DEV)
    prm = T.sample_train_params(N, SH, SW, torch.Generator().manual_seed(N)).to(DEV)
    c = _Call("augment", g)
    src = c("src", sSrc, lambda n, dt: imgs, poison=255)
    params = c("params", sPrm, lambda n, dt: prm, poison=CROP_POISON)
    out = c("out", sOut)
    c.seal()
    C.augment(src, params, out, RH, RW, OH, OW, mode, pad, list(mean), list(std))
    tight = torch.zeros(sOut[1], dtype=torch.bfloat16, device=DEV)
    C.augment(imgs, prm, tight, RH, RW, OH, OW, mode, pad, list(mean), list(std))
    assert torch.equal(out.view(torch.int16), tight.view(torch.int16)), what + ": differs from the tight launch"
    assert not bool(out[..., 3:].view(torch.int16).any()), what + ": padding channels not stored as +0"
    ref = T.augment_reference(imgs, prm, (RH, RW), out_hw=OH, mean=mean, std=std)
    diff = (out[..., :3].float().permute(0, 3, 1, 2) - ref).abs()
    assert float(diff.median()) < 5e-3 and float((diff > 0.05).float().mean()) < 2e-3, what
    c.footprint(what)


def replay_all(C, sigs, g, sms):
    """Replay every signature; returns the number replayed per kernel."""
    kinds = {}
    for sig in sigs:
        _replay(C, sig, g, sms)
        torch.cuda.empty_cache()
        kinds[sig[0]] = kinds.get(sig[0], 0) + 1
    return kinds
