"""Weight decay on the GPU: the AdamW instantiations of adam_kernel against adamw_step64, AdamW at zero
decay against Adam, per-tensor decay segments against separate launches, decoupled ZeRO-1 on emulated
ranks, an audited full-size AdamW step, the launch count, and vggf-mini steps against torch's AdamW."""
import pytest
import torch

import kernel_check as KC
import test_collectives_gpu as TC
import test_step_audit_gpu as TA
from guarded import NAN, Guarded
from distributed_vgg_f_b200.ops import ref as R
from distributed_vgg_f_b200.parallel.symm import owned_cells

pytestmark = pytest.mark.gpu
DEV = "cuda"
F32, BF16 = torch.float32, torch.bfloat16
ARENA_OFF = 4 * 37              # the optimizer cases of test_elementwise_gpu.py: a slice inside the arena
OPT_N = 4 * 135_173
LR = 1e-3


def _C():
    from distributed_vgg_f_b200 import ops
    return ops.require()


def _same_bits(got, want, what):
    bad = got.view(torch.int32) != want.view(torch.int32)
    n = int(bad.sum())
    if n:
        i = int(bad.nonzero()[0, 0])
        raise AssertionError("%s: %d of %d elements differ; first at %d: got %r, expected %r" %
                             (what, n, got.numel(), i, float(got.view(-1)[i]), float(want.view(-1)[i])))


def _state(seed, n):
    g = torch.Generator(device=DEV).manual_seed(seed)
    p = torch.randn(n, device=DEV, generator=g)
    m = torch.randn(n, device=DEV, generator=g) * 1e-3
    v = torch.randn(n, device=DEV, generator=g).abs() * 1e-6
    g32 = torch.randn(n, device=DEV, generator=g)
    g16 = torch.randn(n, device=DEV, generator=g).to(BF16)
    return p, m, v, g32, g16


# ------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("ema", [False, True])
@pytest.mark.parametrize("grad", ["g32", "g16"])
def test_adamw_kernel_within_the_float64_bound(grad, ema):
    """AdamW (decay 0.05, grad_scale 1/8, step 3) on guarded operands at the arena-slice shape of the
    optimizer tests: p / m / v within adamw_step64's bound, the shadow the bf16 of p, the gradient
    cleared, the EMA updated from the new p, nothing outside the slices written."""
    C = _C()
    p0, m0, v0, g32, g16 = _state(11 + (grad == "g16") + 2 * ema, OPT_N)
    ops = [Guarded((OPT_N,), (1,), F32, ARENA_OFF, NAN, DEV) for _ in range(3)]
    for gd, x in zip(ops, (p0, m0, v0)):
        gd.t.copy_(x)
    gsrc = Guarded((OPT_N,), (1,), F32 if grad == "g32" else BF16, ARENA_OFF, NAN, DEV)
    gsrc.t.copy_(g32 if grad == "g32" else g16)
    shadow = Guarded((OPT_N,), (1,), BF16, ARENA_OFF, NAN, DEV)
    e = Guarded((OPT_N,), (1,), F32, ARENA_OFF, NAN, DEV) if ema else None
    e0 = torch.randn(OPT_N, device=DEV, generator=torch.Generator(device=DEV).manual_seed(3))
    if ema:
        e.t.copy_(e0)
    for gd in ops + [gsrc, shadow] + ([e] if ema else []):
        gd.seal()
    lr, b1, b2, eps, wd = R._f32(LR), R._f32(0.9), R._f32(0.999), R._f32(1e-8), 0.05
    C.adam(ops[0].t, ops[1].t, ops[2].t, gsrc.t if grad == "g32" else None, gsrc.t if grad == "g16" else None,
           shadow.t, lr, b1, b2, eps, wd, 3, 0.125, gsrc.t if grad == "g32" else None,
           e.t if ema else None, 0.9 if ema else 0.0, False, True)
    torch.cuda.synchronize()
    ref = R.adamw_step64(p0, m0, v0, (g32 if grad == "g32" else g16.float()), lr=lr, beta1=b1, beta2=b2, eps=eps,
                         weight_decay=wd, step=3, grad_scale=0.125)
    for gd, key in zip(ops, ("p", "m", "v")):
        r, err = ref[key]
        over = (gd.t.double() - r).abs() > err
        assert not bool(over.any()), "%s: %s outside adamw_step64's bound at %d elements" % (grad, key, int(over.sum()))
        gd.check([gd.t], key)
    shadow.check([shadow.t], "shadow")
    assert torch.equal(shadow.t.view(torch.int16), ops[0].t.to(BF16).view(torch.int16))
    if grad == "g32":
        assert int(torch.count_nonzero(gsrc.t)) == 0
        gsrc.check([gsrc.t], "g32")
    else:
        gsrc.check([], "g16")
    if ema:
        e.check([e.t], "ema")
        _same_bits(e.t, 0.9 * e0 + (1 - 0.9) * ops[0].t, "EMA from the new weights")
    # not vacuous: the decoupled decay moved the weights by lr * wd * p beyond the Adam step
    adam = R.adam_step64(p0, m0, v0, (g32 if grad == "g32" else g16.float()), lr=lr, beta1=b1, beta2=b2, eps=eps,
                         weight_decay=0.0, step=3, grad_scale=0.125)["p"][0]
    assert float((ops[0].t.double() - adam).abs().max()) > 0.5 * LR * wd * float(p0.abs().max())


@pytest.mark.parametrize("grad", ["g32", "g16"])
def test_adamw_at_zero_decay_is_adam(grad):
    """With weight decay 0 AdamW's keep factor is 1 and its gradient carries no L2 term: every output is
    bit-identical to the Adam launch."""
    C = _C()
    p0, m0, v0, g32, g16 = _state(21, OPT_N)
    outs = []
    for decoupled in (False, True):
        p, m, v, g, sh = p0.clone(), m0.clone(), v0.clone(), g32.clone(), torch.empty(OPT_N, dtype=BF16, device=DEV)
        C.adam(p, m, v, g if grad == "g32" else None, g16 if grad == "g16" else None, sh, LR, 0.9, 0.999, 1e-8, 0.0,
               5, 0.5, g, None, 0.0, False, decoupled)
        outs.append((p, m, v, g, sh.view(torch.int16).float()))
    for a, b, name in zip(outs[0], outs[1], ("p", "m", "v", "grad", "shadow")):
        _same_bits(b, a, "%s: AdamW(0) against Adam" % name)


SEGS = [(0, 0.05), (2048, 0.0), (6144, 0.05), (6144 + 64, 0.0), (8192, 1e-4)]


@pytest.mark.parametrize("opt", ["adam", "adamw", "sgd"])
def test_segment_table_equals_separate_uniform_launches(opt):
    """One launch with a decay table whose bias entries are 0 gives exactly the bits of one uniform launch
    per segment (a table with one entry per tensor of a bucket stays one launch)."""
    C = _C()
    n = 8192 + 4 * 1000
    p0, m0, v0, g32, _ = _state(31, n)
    bounds = [s for s, _ in SEGS] + [n]

    def launch(p, m, v, g, sh, s, e, wd, table=()):
        starts, wds = [a for a, _ in table], [w for _, w in table]
        if opt == "sgd":
            C.sgd(p[s:e], m[s:e], g[s:e], None, sh[s:e], LR, 0.9, wd, False, 1.0, g[s:e], None, 0.0, False,
                  starts, wds)
        else:
            C.adam(p[s:e], m[s:e], v[s:e], g[s:e], None, sh[s:e], LR, 0.9, 0.999, 1e-8, wd, 4, 1.0, g[s:e], None,
                   0.0, False, opt == "adamw", starts, wds)

    one = [x.clone() for x in (p0, m0, v0, g32)] + [torch.empty(n, dtype=BF16, device=DEV)]
    n0 = C.launch_count()
    launch(*one, 0, n, SEGS[0][1], SEGS)
    assert C.launch_count() == n0 + 1
    sep = [x.clone() for x in (p0, m0, v0, g32)] + [torch.empty(n, dtype=BF16, device=DEV)]
    for k, (s, wd) in enumerate(SEGS):
        launch(*sep, s, bounds[k + 1], wd)
    torch.cuda.synchronize()
    for a, b, name in zip(one, sep, ("p", "m", "v", "grad", "shadow")):
        if a.dtype == BF16:
            a, b = a.view(torch.int16).float(), b.view(torch.int16).float()
        _same_bits(a, b, "%s: %s, one launch with the table against one launch per segment" % (opt, name))
    # not vacuous: the segments did decay differently
    uni = [x.clone() for x in (p0, m0, v0, g32)] + [torch.empty(n, dtype=BF16, device=DEV)]
    launch(*uni, 0, n, 0.05)
    assert not torch.equal(uni[0], one[0])


def test_host_refuses_bad_segment_tables():
    C = _C()
    z = lambda n, dt=F32: torch.zeros(n, dtype=dt, device=DEV)      # noqa: E731
    n = 4096
    bad = {"unsorted": ([0, 2048, 1024], [0.1, 0.0, 0.1]), "misaligned": ([0, 1026], [0.1, 0.0]),
           "outside": ([0, 4096], [0.1, 0.0]), "negative": ([0, 2048], [0.1, -0.1]),
           "first not 0": ([4, 2048], [0.1, 0.0]), "lengths": ([0, 2048], [0.1]),
           "too many": (list(range(0, 4 * (C.wd_max_segments() + 1), 4)), [0.0] * (C.wd_max_segments() + 1))}
    for name, (starts, wds) in bad.items():
        n0 = C.launch_count()
        with pytest.raises(RuntimeError):
            C.adam(z(n), z(n), z(n), z(n), None, None, LR, 0.9, 0.999, 1e-8, 0.0, 1, 1.0, None, None, 0.0, False,
                   True, starts, wds)
        with pytest.raises(RuntimeError):
            C.sgd(z(n), z(n), z(n), None, None, LR, 0.9, 0.0, True, 1.0, None, None, 0.0, False, starts, wds)
        assert C.launch_count() == n0, name


# ---------------------------------------------------------------------------------- ZeRO-1, emulated ranks
Z1_CASES = [(1, 4096, 0, 0), (2, 8 * 31, 8, 1), (3, 65536 + 8, 2056, 16), (8, 65536, 2048, 128)]


@pytest.mark.parametrize("case", Z1_CASES, ids=["W%d-n%d-s%d-c%d" % c for c in Z1_CASES])
def test_decoupled_zero1_on_emulated_ranks(case):
    """Two-shot ZeRO-1 with decoupled decay, every rank in turn on the wire-only entry: on the cells a rank
    owns, p / m / v are bit-identical to the replicated AdamW launch on the reduced bf16 gradient;
    elsewhere (and outside the range) untouched."""
    W, n, start, max_ctas = case
    C = _C()
    seed = Z1_CASES.index(case)
    G = int(C.allreduce_grid(n, W, max_ctas, False))
    gen = torch.Generator(device=DEV).manual_seed(700 + seed)
    inv = 1.0 / W
    packed = [(TC._values("gauss", n, gen) * torch.tensor(inv, device=DEV)).to(BF16) for _ in range(W)]
    owner = torch.full((n,), -1, dtype=torch.int8, device=DEV)
    for r in range(W):
        for a, b in owned_cells(start, n, G, W, r):
            owner[a - start:b - start] = r
    acc = torch.zeros(n, dtype=F32, device=DEV)
    for r in range(W):
        sel = owner == r
        a = torch.zeros(int(sel.sum()), dtype=F32, device=DEV)
        for q in range(W):
            a = a + packed[(r + q) % W][sel].float()
        acc[sel] = a
    red = acc.to(BF16)
    L = start + n + TC.TAIL
    rng = slice(start, start + n)
    p0 = torch.randn(L, generator=gen, device=DEV)
    m0 = torch.randn(L, generator=gen, device=DEV) * 1e-3
    v0 = torch.randn(L, generator=gen, device=DEV).abs() * 1e-6
    HP, wd = TC.HP, 0.05
    rp, rm, rv = p0.clone(), m0.clone(), v0.clone()
    rw = torch.empty(L, dtype=BF16, device=DEV)
    C.adam(rp[rng], rm[rng], rv[rng], None, red, rw[rng], HP["lr"], HP["beta1"], HP["beta2"], HP["eps"], wd,
           TC.STEP, 1.0, None, None, 0.0, False, True)
    grp = TC.Group(W, L, BF16)
    state = [[Guarded((L,), (1,), F32, 0, NAN, DEV) for _ in range(3)] for _ in range(W)]
    shadow = [Guarded((L,), (1,), BF16, 0, TC._poison(BF16, TC.SHADOW_POISON), DEV) for _ in range(W)]
    slot = seed % TC.SLOTS
    for q in range(W):
        grp.wires[q].t[rng] = packed[q]
        for gd, x0 in zip(state[q], (p0, m0, v0)):
            gd.t.copy_(x0)
    for r in range(W):
        epoch = TC._next_epoch()
        grp.arm(r, epoch)
        for gd in state[r]:
            gd.seal()
        n0 = C.launch_count()
        C.zero1_step(grp.comms[r], None, *(gd.t for gd in state[r]), shadow[r].t, start, n, inv, C.AR_TWOSHOT,
                     slot, epoch, max_ctas, HP["lr"], HP["beta1"], HP["beta2"], HP["eps"], wd, TC.STEP,
                     None, 0.0, False, True)
        assert C.launch_count() == n0 + 1
        torch.cuda.synchronize()
        mine = owner == r
        for gd, x0, ref, name in zip(state[r], (p0, m0, v0), (rp, rm, rv), ("p", "m", "v")):
            _same_bits(gd.t[rng], torch.where(mine, ref[rng], x0[rng]),
                       "W%d: %s of rank %d (owned cells: replicated AdamW bit for bit)" % (W, name, r))
            gd.check([gd.t[rng]], "W%d: %s of rank %d" % (W, name, r))


# ------------------------------------------------------------------------------------------- engine
# The arguments an AdamW launch adds after the 14 the replay helper names (ops.adam_step passes all of them
# once the decoupled form or a segment table is used).
ADAM_TAIL = ("ema", "ema_decay", "ema_first", "decoupled", "wd_starts", "wd_values")


def _decay_per_element(sc, p):
    """The launch's weight decay for every element of p (float64): the segment table, or the scalar."""
    starts, values = list(sc["wd_starts"]) or [0], list(sc["wd_values"]) or [sc["wd"]]
    wd = torch.empty(p.numel(), dtype=torch.float64, device=p.device)
    for k, (a, v) in enumerate(zip(starts, values)):
        wd[a:starts[k + 1] if k + 1 < len(starts) else p.numel()] = v
    return wd.view(p.shape)


def _verify_adamw(real_verify):
    """launch_replay.verify, with AdamW launches checked against adamw_step64 as it checks Adam launches
    against adam_step64: p, m and v within the float64 bound (plus the flush-to-zero allowance of real
    data), the shadow the bf16 of p, the gradient range cleared."""
    import kernel_check as KC
    import launch_replay as LR

    def verify(name, before, after, sc, sms, exact=False, what=""):
        if name != "adam" or not sc.get("decoupled"):
            return real_verify(name, before, after, sc, sms, exact=exact, what=what)
        assert sc["ema"] is None, what + ": the audit does not follow the EMA"
        b, a = before, after
        grad = b["g32"] if b["g32"] is not None else b["g16"]
        ref = R.adamw_step64(b["p"], b["m"], b["v"], grad, lr=R._f32(sc["lr"]), beta1=R._f32(sc["b1"]),
                             beta2=R._f32(sc["b2"]), eps=R._f32(sc["eps"]), weight_decay=_decay_per_element(sc, b["p"]),
                             step=sc["step"], grad_scale=R._f32(sc["gscale"]), keep_lr=sc["lr"])
        floor = LR._ftz(7, exact)
        for got, key in ((a["p"], "p"), (a["m"], "m"), (a["v"], "v")):
            r, e = ref[key]
            KC.check(got, r, torch.zeros_like(r), chain=0, exact=False, err=e if floor is None else e + floor,
                     family="adamw_" + key, what=what)
        if a["shadow"] is not None:
            KC.check(a["shadow"], a["p"].double(), a["p"].double(), chain=0, exact=True, family="adamw_shadow",
                     what=what)
        if a["zero"] is not None:
            assert torch.count_nonzero(a["zero"]) == 0, what + ": gradient range not cleared"
        return {}
    return verify


def test_audit_vggf_adamw_bias_decay_zero(capsys, monkeypatch):
    """One full-size VGG-F step (224^2, batch 64) with AdamW, decay 0.05 and the biases at 0: every launch
    against its float64 reference (AdamW: adamw_step64 with per-element decays), its footprint and its links."""
    import launch_replay as LR
    from distributed_vgg_f_b200.models.vggf import vggf_spec

    monkeypatch.setitem(LR.ARGS, "adam", LR.ARGS["adam"] + ADAM_TAIL)
    monkeypatch.setattr(LR, "verify", _verify_adamw(LR.verify))
    eng, aud = TA._run(capsys, "vggf 224 b64 adamw wd 0.05 bias 0", vggf_spec(3), 64, [("train", 64, True)],
                       optimizer="adamw", weight_decay=0.05, bias_weight_decay=0.0)
    assert aud.counts["adam"] == len(eng.plan.buckets)
    assert max(len(s) for s in eng._wd_segments.values()) > 1, "no bucket mixed weights and biases"
    assert {"adamw_p", "adamw_m", "adamw_v"} <= {k.split(":")[0] for k in KC.worst_ratio}, "no AdamW launch checked"


def _batch(b=64, seed=0):
    from distributed_vgg_f_b200.data import transforms as T
    from distributed_vgg_f_b200.data.loader import FusedBatch
    from distributed_vgg_f_b200.data.synthetic import synthetic_uint8_batch

    imgs, labels = synthetic_uint8_batch(b, 128, 3, seed=seed)
    return FusedBatch(torch.from_numpy(imgs), T.sample_train_params(b, 128, 128, torch.Generator().manual_seed(seed)),
                      torch.from_numpy(labels), (256, 256), None)


def test_launch_count_per_step_is_the_defaults():
    """VGG-F: AdamW with the biases at 0 launches exactly as many kernels per step as the default Adam, one
    optimizer launch per bucket, although the tail bucket holds ten tensors of two decays."""
    from distributed_vgg_f_b200 import ops
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine
    from distributed_vgg_f_b200.models.vggf import vggf_spec

    batch = _batch()
    counts = []
    for kw in ({}, dict(optimizer="adamw", weight_decay=0.05, bias_weight_decay=0.0)):
        eng = NativeEngine(vggf_spec(3), device=torch.device(DEV), batch=64, seed=0, distributed=False, **kw)
        per = []
        for _ in range(2):
            n0 = ops.launch_count()
            eng.train_step(batch)
            eng.sync()
            per.append(ops.launch_count() - n0)
        counts.append(per)
        if kw:
            tail = eng._wd_segments[eng.plan.buckets[-1].start]
            assert len(eng.plan.buckets[-1].tensors) == 10 and len(tail) == 10
        del eng
        torch.cuda.empty_cache()
    assert counts[0] == counts[1]


def test_vggf_mini_adamw_steps_match_torch_adamw():
    """vggf-mini steps with AdamW (a large decay, so that the decay dominates the Adam step) and the biases
    at 0: from the engine's own state, torch.optim.AdamW with torchvision's two parameter groups, stepped
    with the bf16-emulating chain's gradients (ops.ref.emulated_step), lands within 4 lr of every weight;
    torch's Adam without decay does not."""
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine
    from distributed_vgg_f_b200.models.vggf import build_oracle, vggf_mini_spec

    spec = vggf_mini_spec(3)
    wd = 100.0                                # keep = 1 - lr * wd = 0.9
    eng = NativeEngine(spec, device=torch.device(DEV), batch=4, lr=LR, seed=0, input_hw=64, distributed=False,
                       optimizer="adamw", weight_decay=wd, bias_weight_decay=0.0,
                       init_state=build_oracle(spec, seed=0).state_dict())
    eng.train_dropout = False
    torch.manual_seed(4)
    for k in range(3):
        x = torch.randn(4, 3, 64, 64, device=DEV).to(BF16).float()
        y = torch.randint(0, 3, (4,), device=DEV)
        state = {n: t.to(DEV) for n, t in eng.export_state().items()}
        st = eng.export_optimizer_state()
        _, _, grads = R.emulated_step(spec, state, x, y)
        refs = {}
        for cls, kw in ((torch.optim.AdamW, dict(weight_decay=wd)), (torch.optim.Adam, {})):
            params = {n: t.clone().requires_grad_(True) for n, t in state.items()}
            groups = [{"params": [params[n] for n in spec.param_names if not n.endswith(".bias")],
                       "weight_decay": kw.get("weight_decay", 0.0)},
                      {"params": [params[n] for n in spec.param_names if n.endswith(".bias")], "weight_decay": 0.0}]
            opt = cls(groups, lr=LR)
            for n in spec.param_names:
                params[n].grad = grads[n].to(DEV).float()
                if st["step"]:
                    opt.state[params[n]] = {"step": torch.tensor(float(st["step"])),
                                            "exp_avg": st["exp_avg"][n].to(DEV),
                                            "exp_avg_sq": st["exp_avg_sq"][n].to(DEV)}
            opt.step()
            refs[cls] = {n: t.detach() for n, t in params.items()}
        eng.train_step((x, y))
        eng.sync()
        got = {n: t.to(DEV) for n, t in eng.export_state().items()}
        for n in spec.param_names:
            err = float((got[n] - refs[torch.optim.AdamW][n]).abs().max())
            assert err <= 4 * LR, "step %d: %s is %.3g from torch's AdamW" % (k, n, err)
        worst = max(float((got[n] - refs[torch.optim.Adam][n]).abs().max()) for n in spec.param_names
                    if not n.endswith(".bias"))
        assert worst > 8 * LR, "the decay is invisible next to the tolerance"
