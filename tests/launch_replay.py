"""Record the native kernel launches of the engine and replay each call signature on guarded operands.

``_record`` swaps ``ops._C`` for a recording proxy during training and evaluation steps of several
engine configurations and keeps each distinct call signature of a ``RECORDED`` kernel (shapes,
strides, dtypes, storage offset mod 16 elements, scalars, which optional tensors are present).
``_replay`` runs one signature once more in exact mode, on fresh guarded operands laid out the same
way (guarded.py), and checks both:

* the values, against the float64 references of ops.ref (exact where the arithmetic allows it, else
  against kernel_check's bound), through ``verify``, which the step audit (step_audit.py) shares;
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
import math
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
# The positional arguments of each recorded kernel, in call order (head_ce's last, ``accumulate``, is
# optional).  The names of tensor arguments are those of CONTRACT.
ARGS = {
    "gemm": ("A", "a_mn", "B", "b_mn", "M", "N", "K", "out", "ldo", "code", "bias", "alpha", "ksplit", "bn"),
    "conv_fprop": ("x", "w", "bias", "y", "relu", "bn"),
    "conv_fprop_pool": ("x", "w", "bias", "pooled", "mask", "bn"),
    "conv_dgrad": ("dz", "w", "mask_src", "dx", "colsum", "bn"),
    "conv_wgrad": ("dz", "x", "dw", "scale", "ksplit", "bn"),
    "conv0_fprop": ("x4", "w0", "bias", "y"),
    "conv0_wgrad": ("dz", "x4", "dw0"),
    "unpool2x2": ("dp", "mask", "dz", "colsum"),
    "maxpool_fwd": ("x", "y"),
    "maxpool_relu_bwd": ("y", "dp", "dz", "colsum"),
    "avgpool_fwd": ("x", "y"),
    "avgpool_bwd": ("dy", "dx"),
    "bias_grad": ("dz", "db", "rows", "C", "ld", "scale"),
    "fc_bias_act": ("acc", "bias", "y", "y_f32", "B", "N", "relu", "p", "seed", "offset", "clear"),
    "fc_grad_act": ("acc", "act", "dz", "B", "N", "relu", "p", "clear"),
    "cross_entropy": ("logits", "target", "dlogits", "ldd", "meter", "loss", "grad_scale", "class_weights"),
    "head_ce": ("h", "W", "bias", "target", "logits", "dlogits", "ldd", "dW", "db", "dh", "drop_scale", "relu",
                "meter", "loss", "class_weights", "accumulate"),
    "adam": ("p", "m", "v", "g32", "g16", "shadow", "lr", "b1", "b2", "eps", "wd", "step", "gscale", "zero"),
    "sgd": ("p", "mom", "g32", "g16", "shadow", "lr", "mo", "wd", "first", "gscale", "zero"),
    "cast_to_bf16": ("x", "y"),
    "nchw_to_nhwc": ("x", "y"),
    "augment": ("src", "params", "out", "RH", "RW", "OH", "OW", "mode", "pad", "mean", "std"),
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


def _batch(spec, eng, b, fused, seed=None):
    seed = b if seed is None else seed
    if not fused:
        g = torch.Generator(device=DEV).manual_seed(seed)
        x = torch.randn(b, 3, eng.HW, eng.HW, device=DEV, generator=g)
        return x, torch.randint(0, spec.num_classes, (b,), device=DEV, generator=g)
    from distributed_vgg_f_b200.data import transforms as T
    from distributed_vgg_f_b200.data.loader import FusedBatch
    from distributed_vgg_f_b200.data.synthetic import synthetic_uint8_batch

    imgs, labels = synthetic_uint8_batch(b, 128, spec.num_classes, seed=seed)
    return FusedBatch(torch.from_numpy(imgs), T.sample_train_params(b, 128, 128, torch.Generator().manual_seed(seed)),
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


def _pow2(v):
    return float(v) == 2.0 ** round(math.log2(v))


def _epi(code):
    from distributed_vgg_f_b200 import ops

    C = ops.require()
    return {C.EPI_F32_STORE: "f32_store", C.EPI_F32_ATOMIC: "f32_atomic", C.EPI_F32_ATOMIC_T: "f32_atomic_t",
            C.EPI_BF16_BIAS_RELU: "bf16_bias_relu", C.EPI_F32_STORE_T: "f32_store_t",
            C.EPI_BF16_STORE: "bf16_store"}[code]


def _ftz(depth, exact):
    """Absolute error allowance on real data: each of the ``depth`` products (and the result) below
    fp32's normal range, 2^-126, may be flushed to zero.  None in exact mode."""
    return None if exact else (depth + 1) * 2.0 ** -126


def split_args(name, args):
    """The positional arguments of a recorded call -> (tensor arguments, scalars), keyed by ARGS."""
    keys = ARGS[name]
    assert len(keys) - (name == "head_ce") <= len(args) <= len(keys), (name, len(args))
    named = dict(zip(keys, args))
    tensors = {k: v for k, v in named.items() if k in CONTRACT[name]}
    return tensors, {k: v for k, v in named.items() if k not in CONTRACT[name]}


def verify(name, before, after, sc, sms, exact=False, what=""):
    """Check one launch of ``name`` against the float64 reference of ops.ref.

    ``before``: the tensor arguments as they were before the launch (snapshots, keyed by ARGS; None
    for an absent optional tensor); ``after``: the same arguments after it; ``sc``: the scalars.
    ``exact``: the operands were chosen so that the arithmetic is exact (the replay's integer fills);
    otherwise every output is held to kernel_check's bound.  Accumulation targets are checked as
    their value before plus the launch's contribution.  Returns the written region of each argument
    whose region is narrower than the whole tensor (views of ``after``), for the footprint check."""
    b, a = before, after
    if name == "gemm":
        M, N, K, ldo, ksplit = sc["M"], sc["N"], sc["K"], sc["ldo"], sc["ksplit"]
        epi = _epi(sc["code"])
        ref, mag = R.gemm64(b["A"], b["B"], M=M, N=N, K=K, a_mn=sc["a_mn"], b_mn=sc["b_mn"], epi=epi,
                            bias=b["bias"], alpha=sc["alpha"])
        got = a["out"].as_strided(tuple(ref.shape), (ldo, 1), a["out"].storage_offset())
        if "atomic" in epi:
            ref, mag = _plus(b["out"].contiguous().as_strided(tuple(ref.shape), (ldo, 1), 0), ref, mag)
        KC.check(got, ref, mag, chain=KC.gemm_chain(K, ksplit) + 1, exact=exact, family="gemm", what=what,
                 err=_ftz(K, exact))
        return {"out": got}
    if name in ("conv_fprop", "conv_fprop_pool"):
        x, w = b["x"], b["w"]
        N, H, W, Cin = x.shape
        Cout = w.numel() // (9 * Cin)
        pool = name == "conv_fprop_pool"
        ref, mag = R.conv3x3_fprop64(x, w.reshape(Cout, 3, 3, Cin), b["bias"], relu=True if pool else sc["relu"])
        if not pool:
            KC.check(a["y"].reshape(N, H, W, Cout), ref, mag, chain=KC.conv_chain(Cin), exact=exact,
                     family="conv_fprop", what=what, err=_ftz(9 * Cin, exact))
        else:
            KC.check_pool(a["pooled"], a["mask"], ref, mag, chain=KC.conv_chain(Cin), exact=exact, what=what)
            assert not bool(a["mask"].reshape(-1, 4)[:, 3].any()), what + ": mask word 3 not written as 0"
        return {}
    if name == "conv_dgrad":
        dz, w, dx, cs = b["dz"], b["w"], a["dx"], a["colsum"]
        N, H, W, Cout = dz.shape
        Cin = dx.shape[-1]
        ref, mag = R.conv3x3_dgrad64(dz, w.reshape(Cout, 3, 3, Cin), mask_src=b["mask_src"])
        KC.check(dx, ref, mag, chain=KC.conv_chain(Cout), exact=exact, family="conv_dgrad", what=what,
                 err=_ftz(9 * Cout, exact))
        if cs is None:
            return {}
        st = dx.to(torch.float64).reshape(-1, Cin)
        KC.check(cs[:Cin], *_plus(b["colsum"][:Cin], st.sum(0), st.abs().sum(0)),
                 chain=KC.conv_colsum_chain(N * H * W, Cin, sms) + 1, exact=False, family="conv_colsum", what=what)
        return {"colsum": cs[:Cin]}
    if name == "conv_wgrad":
        dz, x = b["dz"], b["x"]
        N, H, W, Cout = dz.shape
        Cin = x.shape[-1]
        ref, mag = R.conv3x3_wgrad64(dz, x, sc["scale"])
        KC.check(a["dw"].reshape(ref.shape), *_plus(b["dw"], ref, mag),
                 chain=KC.wgrad_chain(N, H, W, Cin, Cout, sms) + 1, exact=exact, family="conv_wgrad", what=what,
                 err=_ftz(N * H * W, exact))
        return {}
    if name == "conv0_fprop":
        ref, mag = R.conv0_fprop64(b["x4"], b["w0"].reshape(64, 64), b["bias"])
        KC.check(a["y"].reshape(ref.shape), ref, mag, chain=KC.gemm_chain(64), exact=exact, family="conv0_fprop",
                 what=what, err=_ftz(27, exact))
        return {}
    if name == "conv0_wgrad":
        N, H, W, _ = b["x4"].shape
        ref, mag = R.conv0_wgrad64(b["dz"], b["x4"])
        KC.check(a["dw0"].reshape(64, 64), *_plus(b["dw0"], ref, mag), chain=KC.conv0_wgrad_chain(N * H * W, sms) + 1,
                 exact=exact, family="conv0_wgrad", what=what, err=_ftz(N * H * W, exact))
        return {}
    if name in ("unpool2x2", "maxpool_relu_bwd"):
        dp, cs = b["dp"], a["colsum"]
        N, OH, OW, Cc = dp.shape
        if name == "unpool2x2":
            want, want_cs, cs_mag = R.unpool2x2_64(dp, *R.pool_mask_decode(b["mask"], Cc))
            cs_exact, chain = False, KC.unpool_colsum_chain(N * OH * OW, Cc, sms) + 1
        else:
            want, want_cs, cs_mag = R.maxpool2x2_relu_bwd64(b["y"], dp)
            cs_exact, chain = exact, KC.unpool_colsum_chain(N * OH * OW, Cc, sms) + 1
        KC.check(a["dz"], want, want, chain=0, exact=True, family=name, what=what)
        if cs is None:
            return {}
        KC.check(cs[:Cc], *_plus(b["colsum"][:Cc], want_cs, cs_mag), chain=chain, exact=cs_exact,
                 family="unpool_colsum" if name == "unpool2x2" else "maxpool_colsum", what=what)
        return {"colsum": cs[:Cc]}
    if name == "maxpool_fwd":
        val, _ = R.maxpool2x2_64(b["x"])
        KC.check(a["y"], val, val, chain=0, exact=True, family="maxpool_fwd", what=what)
        return {}
    if name in ("avgpool_fwd", "avgpool_bwd"):
        if name == "avgpool_fwd":
            src, dst = b["x"], a["y"]
            (H, OH), ref = (src.shape[1], dst.shape[1]), R.adaptive_avgpool64(src, dst.shape[1], dst.shape[2])
            terms = R.ap_max_window(H, OH) ** 2
        else:
            src, dst = b["dy"], a["dx"]
            (H, OH), ref = (dst.shape[1], src.shape[1]), R.adaptive_avgpool_bwd64(src, dst.shape[1], dst.shape[2])
            terms = R.ap_max_cover(H, OH) ** 2
        sizes = {hi - lo for lo, hi in R._ap_windows(H, OH)}
        KC.check(dst, *ref, chain=KC.avgpool_chain(terms), exact=exact and all(v & (v - 1) == 0 for v in sizes),
                 family=name, what=what)
        return {}
    if name == "bias_grad":
        rows, Cc, ld, scale = sc["rows"], sc["C"], sc["ld"], sc["scale"]
        db = a["db"]
        ref, mag = R.bias_grad64(b["dz"].reshape(-1)[:rows * ld].view(rows, ld), Cc, scale)
        KC.check(db[:Cc], *_plus(b["db"][:Cc], ref, mag), chain=KC.bias_grad_chain(rows, Cc, sms, ld) + 1,
                 exact=exact and _pow2(scale), family="bias_grad", what=what)
        return {"db": db[:Cc]}
    if name == "fc_bias_act":
        # fc_bias_act64 reproduces the kernel's fp32 rounding points: bit-exact on any data
        B, N = sc["B"], sc["N"]
        y, yf, acc, bias = a["y"], a["y_f32"], a["acc"], b["bias"]
        ref, mag = R.fc_bias_act64(_flat(b["acc"], B * N).view(B, N), None if bias is None else bias[:N],
                                   relu=sc["relu"], drop_p=sc["p"], seed=sc["seed"], offset=sc["offset"])
        for out in (y, yf):
            if out is not None:
                KC.check(_flat(out, B * N).view(B, N), ref, mag, chain=0, exact=True, family="fc_bias_act", what=what)
        if sc["clear"]:
            assert torch.count_nonzero(_flat(acc, B * N)) == 0, what + ": acc not cleared"
        return {"acc": _flat(acc, B * N), "y": None if y is None else _flat(y, B * N),
                "y_f32": None if yf is None else _flat(yf, B * N)}
    if name == "fc_grad_act":
        B, N = sc["B"], sc["N"]
        act, acc, dz = b["act"], a["acc"], a["dz"]
        ref, mag = R.fc_grad_act64(_flat(b["acc"], B * N).view(B, N), None if act is None else
                                   _flat(act, B * N).view(B, N), relu=sc["relu"], drop_p=sc["p"])
        KC.check(_flat(dz, B * N).view(B, N), ref, mag, chain=0, exact=True, family="fc_grad_act", what=what)
        if sc["clear"]:
            assert torch.count_nonzero(_flat(acc, B * N)) == 0, what + ": acc not cleared"
        return {"acc": _flat(acc, B * N), "dz": _flat(dz, B * N)}
    if name in ("cross_entropy", "head_ce"):
        return _verify_ce(name, b, a, sc, what, exact)
    if name in ("adam", "sgd"):
        grad = b["g32"] if b["g32"] is not None else b["g16"]
        p, shadow, zero = a["p"], a["shadow"], a["zero"]
        if name == "adam":
            ref = R.adam_step64(b["p"], b["m"], b["v"], grad, lr=R._f32(sc["lr"]), beta1=R._f32(sc["b1"]),
                                beta2=R._f32(sc["b2"]), eps=R._f32(sc["eps"]), weight_decay=R._f32(sc["wd"]),
                                step=sc["step"], grad_scale=R._f32(sc["gscale"]))
            outs = ((p, "p"), (a["m"], "m"), (a["v"], "v"))
        else:
            ref = R.sgd_step64(b["p"], b["mom"], grad, lr=R._f32(sc["lr"]), momentum=R._f32(sc["mo"]),
                               weight_decay=R._f32(sc["wd"]), first=sc["first"], grad_scale=R._f32(sc["gscale"]))
            outs = ((p, "p"), (a["mom"], "buf"))
        for got, key in outs:
            r, e = ref[key]
            # on real data the moments reach fp32's subnormal range, which the kernel flushes to zero
            floor = _ftz(7, exact)
            KC.check(got, r, torch.zeros_like(r), chain=0, exact=False, err=e if floor is None else e + floor,
                     family="%s_%s" % (name, key), what=what)
        if shadow is not None:
            KC.check(shadow, p.double(), p.double(), chain=0, exact=True, family=name + "_shadow", what=what)
        if zero is not None:
            assert torch.count_nonzero(zero) == 0, what + ": gradient range not cleared"
        return {}
    if name == "cast_to_bf16":
        KC.check(a["y"], b["x"].double(), b["x"].double(), chain=0, exact=True, family="cast_to_bf16", what=what)
        return {}
    if name == "nchw_to_nhwc":
        ref, mag = R.nchw_to_nhwc64(b["x"], a["y"].shape[3])
        KC.check(a["y"], ref, mag, chain=0, exact=True, family="nchw_to_nhwc", what=what)
        return {}
    if name == "augment":
        # a pure function of each output pixel: the tolerance of
        # test_kernels_gpu.py::test_augment_matches_reference against augment_reference
        from distributed_vgg_f_b200.data import transforms as T

        out, OH = a["out"], sc["OH"]
        assert sc["OW"] == OH and sc["mode"] == 0, what
        ref = T.augment_reference(b["src"], b["params"], (sc["RH"], sc["RW"]), out_hw=OH, mean=sc["mean"],
                                  std=sc["std"])
        diff = (out[..., :3].float().permute(0, 3, 1, 2) - ref).abs()
        assert float(diff.median()) < 5e-3 and float((diff > 0.05).float().mean()) < 2e-3, what
        assert not bool(out[..., 3:].view(torch.int16).any()), what + ": padding channels not stored as +0"
        return {}
    raise AssertionError("no reference for %s" % name)


def _verify_ce(name, b, a, sc, what, exact):
    """cross_entropy / head_ce: the loss and dlogits against cross_entropy64 within ce_bound, head_ce's
    GEMM parts within their chains, the meter's count and batch size exactly."""
    t, cw, dl, meter, loss = b["target"], b["class_weights"], a["dlogits"], a["meter"], a["loss"]
    ldd = sc["ldd"]
    if name == "cross_entropy":
        z = b["logits"]
        B, Cc = z.shape
        grad_scale = sc["grad_scale"]
    else:
        h, W, bias, z = b["h"], b["W"], b["bias"], a["logits"]
        B, Cc = z.shape
        K = h.shape[1]
        grad_scale = None
    regions = {"meter": None if meter is None else meter[:3], "loss": None if loss is None else loss[:1],
               "dlogits": None if dl is None else _flat(dl, B * ldd)}
    ref = R.cross_entropy64(z, t, ldd=ldd, class_weights=cw, grad_scale=grad_scale)
    bnd = KC.ce_bound(z, t, class_weights=cw, grad_scale=None if cw is not None else
                      (1.0 / B if grad_scale is None else grad_scale), se_chain=-(-Cc // 32) + 5
                      if name == "cross_entropy" else Cc, warps=32 if name == "cross_entropy" else 16)
    if loss is not None:
        KC.check(loss[:1], ref["loss"].view(1), torch.zeros(1, dtype=torch.float64, device=loss.device), chain=0,
                 exact=False, err=bnd["loss"].view(1), family=name + "_loss", what=what)
    if dl is not None:
        err = torch.zeros(B, ldd, dtype=torch.float64, device=dl.device)
        err[:, :Cc] = bnd["dlogits"]
        KC.check(_flat(dl, B * ldd).view(B, ldd), ref["dlogits"], torch.zeros_like(err), chain=0,
                 exact=False, err=err, family=name + "_dlogits", what=what)
    if meter is not None:
        m0 = b["meter"]
        assert float(meter[1]) == float(m0[1]) + float(ref["meter"][1]), what + ": meter[1] not accumulated"
        assert float(meter[2]) == float(m0[2]) + B, what + ": meter[2] not accumulated"
    if name == "head_ce":
        chain = KC.head_chain(K, B)
        dW, db, dh = a["dW"], a["db"], a["dh"]
        part = R.head_ce64(h, W, bias, dl_used=_flat(dl, B * ldd).view(B, ldd)[:, :Cc] if dl is not None
                           else torch.zeros(B, Cc, device=z.device), drop_scale=sc["drop_scale"], relu=sc["relu"])
        KC.check(z, *part["logits"], chain=chain["logits"], exact=False, family="head_logits", what=what,
                 err=_ftz(K, exact))
        if dW is not None:
            want, chain_dW = part["dW"], chain["dW"]
            if sc.get("accumulate"):                 # a later micro-batch of a group: dW += the batch's gradient
                want, chain_dW = _plus(_flat(b["dW"], Cc * K), *want), chain_dW + 1
            KC.check(_flat(dW, Cc * K).view(Cc, K), *want, chain=chain_dW, exact=False, family="head_dW", what=what,
                     err=_ftz(B, exact))
            KC.check(db[:Cc], *_plus(b["db"][:Cc], *part["db"]), chain=chain["db"], exact=False,
                     family="head_db", what=what)
        if dh is not None:
            KC.check(_flat(dh, B * K).view(B, K), *part["dh"], chain=chain["dh"], exact=False, family="head_dh",
                     what=what, err=_ftz(Cc, exact))
        regions.update(logits=_flat(z, B * Cc), dW=None if dW is None else _flat(dW, Cc * K),
                       db=None if db is None else db[:Cc], dh=None if dh is None else _flat(dh, B * K))
    return {k: v for k, v in regions.items() if v is not None}


def _operands(c, name, s, g):
    """Guarded operands of one replayed call: ``s`` holds the signature of each tensor argument."""
    if name == "gemm":
        K = s["K"]
        return {"A": c("A", s["A"], _ints(K, g)), "B": c("B", s["B"], _ints(K, g)), "out": c("out", s["out"]),
                "bias": c("bias", s["bias"], _bias(g))}
    if name in ("conv_fprop", "conv_fprop_pool"):
        Cin = s["x"][1][3]
        t = {"x": c("x", s["x"], _ints(9 * Cin, g)), "w": c("w", s["w"], _ints(9 * Cin, g)),
             "bias": c("bias", s["bias"], _bias(g))}
        outs = ("y",) if name == "conv_fprop" else ("pooled", "mask")
        t.update({k: c(k, s[k]) for k in outs})
        return t
    if name == "conv_dgrad":
        Cout = s["dz"][1][3]
        return {"dz": c("dz", s["dz"], _ints(9 * Cout, g)), "w": c("w", s["w"], _ints(9 * Cout, g)),
                "mask_src": c("mask_src", s["mask_src"], _ints(1, g)), "dx": c("dx", s["dx"]),
                "colsum": c("colsum", s["colsum"])}
    if name == "conv_wgrad":
        N, H, W, _ = s["dz"][1]
        P = N * H * W
        return {"dz": c("dz", s["dz"], _ints(P, g)), "x": c("x", s["x"], _ints(P, g)), "dw": c("dw", s["dw"])}
    if name == "conv0_fprop":
        return {"x4": c("x4", s["x4"], _ints(27, g)), "w0": c("w0", s["w0"], _ints(27, g)),
                "bias": c("bias", s["bias"], _bias(g)), "y": c("y", s["y"])}
    if name == "conv0_wgrad":
        N, H, W, _ = s["x4"][1]
        P = N * H * W
        return {"dz": c("dz", s["dz"], _ints(P, g)), "x4": c("x4", s["x4"], _ints(P, g)), "dw0": c("dw0", s["dw0"])}
    if name == "unpool2x2":
        N, OH, OW, Cc = s["dp"][1]
        idx = torch.randint(0, 4, (N, OH, OW, Cc), device=DEV, generator=g)
        pos = torch.rand(N, OH, OW, Cc, device=DEV, generator=g) < 0.7
        words = R.pool_mask_encode(idx, pos).to(torch.int32)
        return {"dp": c("dp", s["dp"], _ints(1, g)), "mask": c("mask", s["mask"], lambda n, dt: words.reshape(-1),
                                                               poison=-1),
                "dz": c("dz", s["dz"]), "colsum": c("colsum", s["colsum"])}
    if name == "maxpool_fwd":
        return {"x": c("x", s["x"], _relu_ints(g), poison=G.fmax(torch.bfloat16)), "y": c("y", s["y"])}
    if name == "maxpool_relu_bwd":
        return {"y": c("y", s["y"], _relu_ints(g), poison=G.fmax(torch.bfloat16)), "dp": c("dp", s["dp"], _ints(1, g)),
                "dz": c("dz", s["dz"]), "colsum": c("colsum", s["colsum"])}
    if name == "avgpool_fwd":
        return {"x": c("x", s["x"], _ints(16, g)), "y": c("y", s["y"])}
    if name == "avgpool_bwd":
        return {"dy": c("dy", s["dy"], _ints(16, g)), "dx": c("dx", s["dx"])}
    if name == "bias_grad":
        return {"dz": c("dz", s["dz"], _ints(s["rows"], g)), "db": c("db", s["db"])}
    if name == "fc_bias_act":
        return {"acc": c("acc", s["acc"], _ints(1, g)), "bias": c("bias", s["bias"], _bias(g)), "y": c("y", s["y"]),
                "y_f32": c("y_f32", s["y_f32"])}
    if name == "fc_grad_act":
        return {"acc": c("acc", s["acc"], _ints(1, g)), "act": c("act", s["act"], _relu_ints(g)),
                "dz": c("dz", s["dz"])}
    if name in ("cross_entropy", "head_ce"):
        t = {}
        if name == "cross_entropy":
            t["logits"] = c("logits", s["logits"], _gauss(g, 3.0), poison=G.fmax(torch.float32))
            Cc = s["logits"][1][1]
        else:
            t.update(h=c("h", s["h"], _relu_ints(g)), W=c("W", s["W"], _gauss(g, 0.1)),
                     bias=c("bias", s["bias"], _gauss(g, 0.1)))
            Cc = s["logits"][1][1]
        t["target"] = c("target", s["target"], lambda n, dt: torch.randint(0, Cc, (n,), device=DEV, generator=g),
                        poison=Cc - 1)
        t["class_weights"] = c("class_weights", s["class_weights"],
                               lambda n, dt: torch.rand(n, device=DEV, generator=g) + 0.1)
        for k in ("dlogits", "meter", "loss"):
            t[k] = c(k, s[k])
        if name == "head_ce":
            for k in ("logits", "dW", "db", "dh"):
                t[k] = c(k, s[k])
        return t
    if name in ("adam", "sgd"):
        same = s["zero"] is not None and s["zero"] == s["g32"]     # the engine clears the gradient it reads
        mom = "m" if name == "adam" else "mom"
        t = {"p": c("p", s["p"], _gauss(g)), mom: c(mom, s[mom], _gauss(g, 1e-3))}
        if name == "adam":
            t["v"] = c("v", s["v"], lambda n, dt: torch.rand(n, device=DEV, generator=g) * 1e-6)
        t["g32"] = c("g32", s["g32"], _gauss(g, 1e-2), role=UPDATE if same else None)
        t["g16"] = c("g16", s["g16"], _gauss(g, 1e-2))
        t["shadow"] = c("shadow", s["shadow"])
        t["zero"] = t["g32"] if same else c("zero", s["zero"], _gauss(g))
        return t
    if name == "cast_to_bf16":
        return {"x": c("x", s["x"], _gauss(g)), "y": c("y", s["y"])}
    if name == "nchw_to_nhwc":
        return {"x": c("x", s["x"], _gauss(g)), "y": c("y", s["y"])}
    raise AssertionError("no replay for %s" % name)


def _replay(C, sig, g, sms):
    name = sig[0]
    if name == "augment":
        return _replay_augment(C, sig, g)
    what = str(sig)
    s, sc = split_args(name, sig[1:])
    s.update(sc)
    c = _Call(name, g, atomic=name == "gemm" and "atomic" in _epi(sc["code"]), clear=sc.get("clear"))
    t = _operands(c, name, s, g)
    c.seal()
    before = {k: None if v is None else v.clone() for k, v in t.items()}
    getattr(C, name)(*[t[k] if k in t else sc[k] for k in ARGS[name][:len(sig) - 1]])
    regions = verify(name, before, t, sc, sms, exact=True, what=what)
    c.footprint(what, **{k: v for k, v in regions.items() if v is not None})


def _replay_augment(C, sig, g):
    """augment is a pure function of each output pixel: the guarded launch must equal the same launch
    on tightly allocated tensors bit for bit, and pass verify()."""
    from distributed_vgg_f_b200.data import transforms as T
    from distributed_vgg_f_b200.data.synthetic import synthetic_uint8_batch

    s, sc = split_args("augment", sig[1:])
    what = str(sig)
    N, SH, SW, _ = s["src"][1]
    assert SH == SW, what
    imgs = torch.from_numpy(synthetic_uint8_batch(N, SH, seed=N)[0]).to(DEV)
    prm = T.sample_train_params(N, SH, SW, torch.Generator().manual_seed(N)).to(DEV)
    c = _Call("augment", g)
    src = c("src", s["src"], lambda n, dt: imgs, poison=255)
    params = c("params", s["params"], lambda n, dt: prm, poison=CROP_POISON)
    out = c("out", s["out"])
    c.seal()
    scal = [sc[k] for k in ("RH", "RW", "OH", "OW", "mode", "pad")]
    C.augment(src, params, out, *scal, list(sc["mean"]), list(sc["std"]))
    tight = torch.zeros(s["out"][1], dtype=torch.bfloat16, device=DEV)
    C.augment(imgs, prm, tight, *scal, list(sc["mean"]), list(sc["std"]))
    assert torch.equal(out.view(torch.int16), tight.view(torch.int16)), what + ": differs from the tight launch"
    verify("augment", {"src": imgs, "params": prm}, {"out": out}, sc, 0, what=what)
    c.footprint(what)


def replay_all(C, sigs, g, sms):
    """Replay every signature; returns the number replayed per kernel."""
    kinds = {}
    for sig in sigs:
        _replay(C, sig, g, sms)
        torch.cuda.empty_cache()
        kinds[sig[0]] = kinds.get(sig[0], 0) + 1
    return kinds
