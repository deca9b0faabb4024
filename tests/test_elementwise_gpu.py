"""The memory-bound kernels of elementwise.cu, loss_optim.cu and the input casts against the float64
references of ops.ref, element by element (kernel_check), at the shapes the training step launches
and at the edges where these kernels go wrong: tied maxima, overlapping average-pool windows,
the bias-gradient block cap, scalar tails, the high Philox counter word, argmax ties, and optimizer
slices inside a larger arena.  Also: every host-side argument check refuses before any launch."""
import pytest
import torch

import kernel_check as KC
from distributed_vgg_f_b200.ops import ref as R

pytestmark = pytest.mark.gpu
DEV = "cuda"
MODES = ["exact", "gauss"]
F64 = torch.float64


def _ops():
    from distributed_vgg_f_b200 import ops
    ops.require()
    return ops


def _C():
    from distributed_vgg_f_b200 import ops
    return ops.require()


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _zeros64(t):
    return torch.zeros(t.shape, dtype=F64, device=t.device)


# ----------------------------------------------------------------------------------- max-pool
POOL_LAYERS = [(n, h, c) for n in (64, 37) for h, c in ((224, 64), (112, 128), (56, 256), (28, 512), (14, 512))]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("N,H,C", POOL_LAYERS + [(2, 224, 8), (3, 16, 8)])
def test_maxpool_fwd_relu_bwd_colsum(N, H, C, mode):
    """Forward and the fused ReLU + pool backward with its column sum.  Exact mode: post-ReLU
    integers, so tied windows, all-zero windows and ReLU zeros are frequent."""
    ops = _ops()
    g = _gen(N * 7 + H + C)
    if mode == "exact":
        y = torch.relu(torch.randint(-2, 3, (N, H, H, C), device=DEV, generator=g)).to(torch.bfloat16)
    else:
        y = torch.relu(torch.randn(N, H, H, C, device=DEV, generator=g)).to(torch.bfloat16)
    p = ops.maxpool2x2(y)
    val, _ = R.maxpool2x2_64(y)
    KC.check(p, val, val, chain=0, exact=True, family="maxpool_fwd")
    dp = KC.operand(p.shape, mode, 1, g, DEV)
    cs = torch.zeros(C, device=DEV)
    dz = ops.maxpool2x2_relu_bwd(y, dp, colsum=cs)
    want, want_cs, cs_mag = R.maxpool2x2_relu_bwd64(y, dp)
    KC.check(dz, want, want, chain=0, exact=True, family="maxpool_relu_bwd")
    KC.check(cs, want_cs, cs_mag, chain=KC.unpool_colsum_chain(N * (H // 2) ** 2, C, KC.sm_count()),
             exact=mode == "exact", family="maxpool_colsum")


# ------------------------------------------------------------------------ adaptive average pool
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("N", [1, 37])
@pytest.mark.parametrize("C", [64, 512])
@pytest.mark.parametrize("H", [2, 4, 5, 7, 8, 10, 14])
def test_adaptive_avgpool_fwd_bwd(H, C, N, mode):
    """Forward and backward to 7x7.  H < 7 has overlapping windows; exact mode needs window sizes that
    are powers of two (every H < 7, H = 8 and 14); H = 10 runs in gauss mode only."""
    if mode == "exact" and H == 10:
        pytest.skip("window sizes 2 and 3: 1/6 and 1/9 are not exact")
    ops = _ops()
    g = _gen(H * 100 + C + N)
    exact = mode == "exact"
    x = KC.operand((N, H, H, C), mode, 16, g, DEV)
    y = ops.adaptive_avgpool(x, 7, 7)
    ref, mag = R.adaptive_avgpool64(x, 7, 7)
    KC.check(y, ref, mag, chain=KC.avgpool_chain(R.ap_max_window(H, 7) ** 2), exact=exact, family="avgpool_fwd")
    dy = KC.operand((N, 7, 7, C), mode, 16, g, DEV)
    dx = ops.adaptive_avgpool_bwd(dy, H, H)
    ref, mag = R.adaptive_avgpool_bwd64(dy, H, H)
    KC.check(dx, ref, mag, chain=KC.avgpool_chain(R.ap_max_cover(H, 7) ** 2), exact=exact, family="avgpool_bwd")


# ---------------------------------------------------------------------------------- bias grad
BIAS_CASES = ([(r, c, c) for r in (1, 37, 64) for c in (8, 64, 512, 1000, 2056, 4096)]
              + [(3_000_007, 8, 8), (3_000_007, 64, 64)]                     # hits the block cap
              + [(37, 3, 8), (64, 10, 16), (1, 3, 8), (5000, 10, 16)])       # ld = rup8(C) != C


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("rows,C,ld", BIAS_CASES)
def test_bias_grad(rows, C, ld, mode):
    ops = _ops()
    g = _gen(rows % 1000 + C)
    exact = mode == "exact"
    scale = 0.5 if exact else 0.37
    dz = KC.operand((rows, ld), mode, rows, g, DEV)
    db0 = KC.bias(C, mode, g, DEV)
    db = db0.clone()
    ops.bias_grad(dz, db, rows, C, ld=ld, scale=scale)
    ref, mag = R.bias_grad64(dz, C, scale)
    KC.check(db, ref + db0.double(), mag + db0.double().abs(), chain=KC.bias_grad_chain(rows, C, KC.sm_count(), ld),
             exact=exact, family="bias_grad", what="rows=%d C=%d ld=%d" % (rows, C, ld))


# ------------------------------------------------------------------------------ FC epilogues
def _drop_keys():
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine
    eng = NativeEngine.__new__(NativeEngine)
    eng.seed, eng.rank, eng.same_dropout_all_ranks = 0, 0, False
    return [NativeEngine._drop_key(eng, i) for i in range(3)]


OFFSETS = [1, 2, 2 ** 32 + 1]
FC_CASES = [(B, N, p) for B in (1, 16, 37, 64) for N in (512, 4096, 10) for p in (0.0, 0.5, 0.6)]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("B,N,p", FC_CASES)
def test_fc_bias_act_and_dropout(B, N, p, mode):
    """y = dropout(relu(acc + bias)) bit for bit in both modes: bf16 and fp32 outputs, Philox mask of
    (seed, offset, element), fp32 keep scale, and the accumulator cleared or kept."""
    C = _C()
    i = FC_CASES.index((B, N, p))
    seed, offset = _drop_keys()[i % 3], OFFSETS[i % 3]
    g = _gen(i)
    acc0 = KC.operand((B, N), mode, 1, g, DEV).float()
    bias = KC.bias(N, mode, g, DEV)
    ref, mag = R.fc_bias_act64(acc0, bias, relu=True, drop_p=p, seed=seed, offset=offset)
    for clear in (True, False):
        acc = acc0.clone()
        y = torch.empty(B, N, dtype=torch.bfloat16, device=DEV)
        yf = torch.empty(B, N, device=DEV)
        C.fc_bias_act(acc, bias, y, yf, B, N, True, p, seed, offset, clear)
        KC.check(y, ref, mag, chain=0, exact=True, family="fc_bias_act", what="bf16")
        KC.check(yf, ref, mag, chain=0, exact=True, family="fc_bias_act", what="fp32")
        assert torch.equal(acc, torch.zeros_like(acc) if clear else acc0)
    if p > 0 and B * N >= 4096:
        keep = ref != 0
        frac = 1 - float(R.dropout_mask64(seed, offset, B, N, p)[0].float().mean())
        assert abs(frac - p) < 0.05 and bool(keep.any())


def test_dropout_masks_differ_by_step_and_layer_and_ignore_batch_size():
    C = _C()
    N, p = 4096, 0.5
    k0, k1, _ = _drop_keys()

    def mask(B, seed, offset):
        acc = torch.ones(B, N, device=DEV)
        y = torch.empty(B, N, dtype=torch.bfloat16, device=DEV)
        C.fc_bias_act(acc, None, y, None, B, N, True, p, seed, offset, False)
        return y != 0

    a = mask(64, k0, 1)
    assert not torch.equal(a, mask(64, k0, 2))                 # another step
    assert not torch.equal(a, mask(64, k1, 1))                 # another layer
    assert not torch.equal(a, mask(64, k0, 2 ** 32 + 1))        # the high counter word is used
    assert torch.equal(mask(37, k0, 1), a[:37])                # a ragged last batch draws the same rows
    keep, _ = R.dropout_mask64(k0, 1, 64, N, p, device=DEV)
    assert torch.equal(a, keep)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("B,N,relu,p", [(64, 4096, True, 0.5), (37, 512, True, 0.6), (16, 4096, True, 0.0),
                                         (37, 25088, False, 0.0), (1, 4097, True, 0.5), (37, 10, True, 0.6),
                                         (3, 513, False, 0.0), (1, 5, True, 0.6)])
def test_fc_grad_act(B, N, relu, p, mode):
    """dz = acc * [act > 0] / (1 - p) with the forward's own output as act; B * N % 4 in {1, 2, 3}
    runs the scalar tail."""
    C = _C()
    g = _gen(B * N)
    seed, offset = _drop_keys()[2], 5
    act = torch.empty(B, N, dtype=torch.bfloat16, device=DEV)
    if relu:
        C.fc_bias_act(torch.randn(B, N, device=DEV, generator=g), None, act, None, B, N, True, p, seed, offset, True)
    acc0 = KC.operand((B, N), mode, 1, g, DEV).float()
    ref, mag = R.fc_grad_act64(acc0, act if relu else None, relu=relu, drop_p=p)
    if relu and p > 0:
        keep, _ = R.dropout_mask64(seed, offset, B, N, p, device=DEV)
        assert torch.equal(act != 0, keep & (act != 0)) and not bool((ref[~keep] != 0).any())
    for clear in (True, False):
        acc = acc0.clone()
        dz = torch.empty(B, N, dtype=torch.bfloat16, device=DEV)
        C.fc_grad_act(acc, act if relu else None, dz, B, N, relu, p, clear)
        KC.check(dz, ref, mag, chain=0, exact=True, family="fc_grad_act")
        assert torch.equal(acc, torch.zeros_like(acc) if clear else acc0)


# ------------------------------------------------------------------------------ cross-entropy
def _ce_logits(B, C, g, scale, ties):
    z = torch.randn(B, C, device=DEV, generator=g) * scale
    t = torch.randint(0, C, (B,), device=DEV, generator=g)
    if ties and C > 1:
        # duplicated maxima: in neighbouring lanes (c, c + 1), or 32 apart (same lane, a later stride)
        for r in range(0, B, 3):
            a = r % C
            b = (a + 32) % C if C > 32 and r % 2 == 0 else (a + 1) % C
            if a != b:
                z[r, a] = z[r, b] = z[r].max() + 1
                t[r] = a if r % 2 else b
    return z, t


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("B,C", [(1, 3), (37, 3), (64, 3), (32, 1000), (256, 1000), (7, 10)])
def test_cross_entropy(B, C, weighted):
    """Loss, dlogits (padding zeroed up to ldd > C), meter; __expf / __logf errors bounded by
    kernel_check.ce_bound; logits x30 and tied maxima where the lower index must win."""
    C_ = _C()
    g = _gen(B + C)
    ldd = (C + 7) // 8 * 8 + 8
    for scale, ties in ((3.0, True), (30.0, False)):
        z, t = _ce_logits(B, C, g, scale, ties)
        w = torch.rand(C, device=DEV, generator=g) + 0.1 if weighted else None
        dl = torch.full((B, ldd), 7.0, dtype=torch.bfloat16, device=DEV)
        meter = torch.zeros(4, device=DEV)
        loss = torch.zeros(1, device=DEV)
        C_.cross_entropy(z, t, dl, ldd, meter, loss, 1.0 / B, w)
        ref = R.cross_entropy64(z, t, ldd=ldd, class_weights=w)
        bnd = KC.ce_bound(z, t, class_weights=w, se_chain=-(-C // 32) + 5, warps=32)
        err = torch.zeros(B, ldd, dtype=F64, device=DEV)
        err[:, :C] = bnd["dlogits"]
        KC.check(dl, ref["dlogits"], _zeros64(err), chain=0, exact=False, err=err, family="ce_dlogits")
        KC.check(loss, ref["loss"].view(1), torch.zeros(1, dtype=F64, device=DEV), chain=0, exact=False,
                 err=bnd["loss"].view(1), family="ce_loss")
        KC.check(meter[:1], ref["meter"][:1].to(DEV), torch.zeros(1, dtype=F64, device=DEV), chain=0, exact=False,
                 err=bnd["meter0"].view(1), family="ce_meter")
        assert float(meter[1]) == float(ref["meter"][1]) and float(meter[2]) == B


HEAD_KS = [32, 96, 512, 1000, 1024]
HEAD_CASES = [(B, C) for B in (1, 37, 64, 256) for C in (1, 3, 8)]


@pytest.mark.parametrize("B,C", HEAD_CASES)
def test_head_ce(B, C):
    """The fused head: logits, loss, dlogits, dW, db, dh; ReLU + drop_scale 2.5, class weights on every
    other case, then the evaluation form."""
    C_ = _C()
    i = HEAD_CASES.index((B, C))
    K = HEAD_KS[i % len(HEAD_KS)]
    weighted = i % 2 == 1
    g = _gen(1000 + i)
    h = torch.relu(torch.randn(B, K, device=DEV, generator=g)).to(torch.bfloat16)
    W = (torch.randn(C, K, device=DEV, generator=g) * 0.1).to(torch.bfloat16)
    bias = torch.randn(C, device=DEV, generator=g) * 0.1
    t = torch.randint(0, C, (B,), device=DEV, generator=g)
    cw = torch.rand(C, device=DEV, generator=g) + 0.5 if weighted else None
    ldd = 8
    logits = torch.empty(B, C, device=DEV)
    dl = torch.full((B, ldd), 7.0, dtype=torch.bfloat16, device=DEV)
    dW = torch.empty(C, K, device=DEV)
    db0 = torch.randn(C, device=DEV, generator=g)
    db = db0.clone()
    dh = torch.empty(B, K, dtype=torch.bfloat16, device=DEV)
    meter = torch.zeros(4, device=DEV)
    loss = torch.zeros(1, device=DEV)
    C_.head_ce(h, W, bias, t, logits, dl, ldd, dW, db, dh, 2.5, True, meter, loss, cw)
    chain = KC.head_chain(K, B)
    ref = R.head_ce64(h, W, bias, dl_used=dl[:, :C], drop_scale=2.5, relu=True)
    KC.check(logits, *ref["logits"], chain=chain["logits"], exact=False, family="head_logits")
    # the loss part is judged on the logits the kernel computed
    ce = R.cross_entropy64(logits, t, ldd=ldd, class_weights=cw)
    bnd = KC.ce_bound(logits, t, class_weights=cw, se_chain=C, warps=16)
    err = torch.zeros(B, ldd, dtype=F64, device=DEV)
    err[:, :C] = bnd["dlogits"]
    KC.check(dl, ce["dlogits"], _zeros64(err), chain=0, exact=False, err=err, family="head_dlogits")
    KC.check(loss, ce["loss"].view(1), torch.zeros(1, dtype=F64, device=DEV), chain=0, exact=False,
             err=bnd["loss"].view(1), family="head_loss")
    assert float(meter[1]) == float(ce["meter"][1]) and float(meter[2]) == B
    KC.check(dW, *ref["dW"], chain=chain["dW"], exact=False, family="head_dW")
    KC.check(db, ref["db"][0] + db0.double(), ref["db"][1] + db0.double().abs(), chain=chain["db"], exact=False,
             family="head_db")
    KC.check(dh, *ref["dh"], chain=chain["dh"], exact=False, family="head_dh")
    # evaluation form: forward + metrics only
    logits2 = torch.empty_like(logits)
    C_.head_ce(h, W, bias, t, logits2, None, 0, None, None, None, 1.0, False, None, loss, None)
    assert torch.equal(logits2, logits)
    ce = R.cross_entropy64(logits2, t)
    bnd = KC.ce_bound(logits2, t, se_chain=C, warps=16)
    KC.check(loss, ce["loss"].view(1), torch.zeros(1, dtype=F64, device=DEV), chain=0, exact=False,
             err=bnd["loss"].view(1), family="head_loss")


# ------------------------------------------------------------------------------- optimizers
ARENA_OFF = 4 * 37              # the slice starts inside the arena, 16-byte aligned
OPT_N = 4 * 135_173             # not a multiple of any grid stride (blocks x 256 threads x 4)
F32 = R._f32


def _arena(g, n_total, scale=1.0):
    return torch.randn(n_total, device=DEV, generator=g) * scale


def _check_outside(before, after, s, e, what):
    for b, a in zip(before, after):
        assert torch.equal(b[:s], a[:s]) and torch.equal(b[e:], a[e:]), what + ": elements outside the slice changed"


@pytest.mark.parametrize("g16", [False, True])
def test_adam_steps_on_an_arena_slice(g16):
    """One step at a time against adam_step64 applied to the kernel's previous state: steps 1, 2, 10
    and 10^4, weight decay, grad_scale 1/8, fp32 or bf16 gradients, shadow RNE(p) bit for bit, the
    gradient range zeroed and everything outside the slice untouched."""
    C = _C()
    g = _gen(77 + g16)
    s, e = ARENA_OFF, ARENA_OFF + OPT_N
    tot = e + 64
    p, m, v = _arena(g, tot), _arena(g, tot, 1e-3), _arena(g, tot).abs() * 1e-6
    w16 = p.to(torch.bfloat16)
    g32 = _arena(g, tot)
    gb = torch.randn(tot, device=DEV, generator=g).to(torch.bfloat16)
    hp = dict(lr=F32(1e-3), beta1=F32(0.9), beta2=F32(0.999), eps=F32(1e-8), weight_decay=F32(0.01))
    for step in (1, 2, 10, 10_000):
        if not g16:                  # magnitudes 1 .. 1e-6, so that eps matters in some elements
            g32[s:e] = torch.randn(OPT_N, device=DEV, generator=g) * 10.0 ** (-6 * torch.rand(OPT_N, device=DEV,
                                                                                                generator=g))
        before = [t.clone() for t in (p, m, v, w16, g32)]
        ref = R.adam_step64(p[s:e], m[s:e], v[s:e], gb[s:e] if g16 else g32[s:e], step=step, grad_scale=0.125, **hp)
        C.adam(p[s:e], m[s:e], v[s:e], None if g16 else g32[s:e], gb[s:e] if g16 else None, w16[s:e],
               hp["lr"], hp["beta1"], hp["beta2"], hp["eps"], hp["weight_decay"], step, 0.125, g32[s:e])
        for got, key in ((p, "p"), (m, "m"), (v, "v")):
            r, err = ref[key]
            KC.check(got[s:e], r, _zeros64(r), chain=0, exact=False, err=err, family="adam_" + key,
                     what="step %d" % step)
        KC.check(w16[s:e], p[s:e].double(), p[s:e].double(), chain=0, exact=True, family="adam_shadow")
        assert torch.count_nonzero(g32[s:e]) == 0
        _check_outside(before, (p, m, v, w16, g32), s, e, "adam")


@pytest.mark.parametrize("momentum", [0.9, 0.0])
@pytest.mark.parametrize("g16", [False, True])
def test_sgd_steps_on_an_arena_slice(g16, momentum):
    C = _C()
    g = _gen(88 + g16)
    s, e = ARENA_OFF, ARENA_OFF + OPT_N
    tot = e + 64
    p, mom = _arena(g, tot), _arena(g, tot)
    w16 = p.to(torch.bfloat16)
    g32 = _arena(g, tot)
    gb = torch.randn(tot, device=DEV, generator=g).to(torch.bfloat16)
    lr, mo, wd = F32(0.01), F32(momentum), F32(1e-4)
    for step in (1, 2, 10):
        if not g16:
            g32[s:e] = torch.randn(OPT_N, device=DEV, generator=g)
        before = [t.clone() for t in (p, mom, w16, g32)]
        ref = R.sgd_step64(p[s:e], mom[s:e], gb[s:e] if g16 else g32[s:e], lr=lr, momentum=mo, weight_decay=wd,
                           first=step == 1, grad_scale=0.125)
        C.sgd(p[s:e], mom[s:e], None if g16 else g32[s:e], gb[s:e] if g16 else None, w16[s:e], lr, mo, wd,
              step == 1, 0.125, g32[s:e])
        for got, key in ((p, "p"), (mom, "buf")):
            r, err = ref[key]
            KC.check(got[s:e], r, _zeros64(r), chain=0, exact=False, err=err, family="sgd_" + key)
        KC.check(w16[s:e], p[s:e].double(), p[s:e].double(), chain=0, exact=True, family="sgd_shadow")
        assert torch.count_nonzero(g32[s:e]) == 0
        _check_outside(before, (p, mom, w16, g32), s, e, "sgd")


# ------------------------------------------------------------------------------------ casts
@pytest.mark.parametrize("n", [4096, 4097, 4098, 4099, 1, 2, 3])
def test_casts(n):
    C = _C()
    g = _gen(n)
    x = torch.randn(n, device=DEV, generator=g) * 10.0 ** torch.randint(-3, 4, (n,), device=DEV, generator=g).float()
    y = torch.full((n + 8,), 7.0, dtype=torch.bfloat16, device=DEV)
    C.cast_to_bf16(x, y[:n])
    KC.check(y[:n], x.double(), x.double(), chain=0, exact=True, family="cast_to_bf16")
    assert bool((y[n:] == 7.0).all())
    back = torch.empty(n, device=DEV)
    C.cast_to_f32(y[:n], back)
    assert torch.equal(back, y[:n].float())


@pytest.mark.parametrize("N,Cin,H,W,cpad", [(2, 3, 224, 224, 4), (37, 3, 64, 64, 4), (1, 3, 5, 7, 8)])
def test_nchw_to_nhwc_zero_pads(N, Cin, H, W, cpad):
    C = _C()
    x = torch.randn(N, Cin, H, W, device=DEV, generator=_gen(N))
    y = torch.full((N, H, W, cpad), 7.0, dtype=torch.bfloat16, device=DEV)
    C.nchw_to_nhwc(x, y)
    ref, mag = R.nchw_to_nhwc64(x, cpad)
    KC.check(y, ref, mag, chain=0, exact=True, family="nchw_to_nhwc")


# ---------------------------------------------------------------------- host-side refusals
def _misaligned(shape, dtype, by=1):
    n = 1
    for d in shape:
        n *= d
    return torch.zeros(n + 16, dtype=dtype, device=DEV)[by:by + n].view(shape)


def _refusals():
    bf, f = torch.bfloat16, torch.float32
    z = lambda *s, dt=bf: torch.zeros(*s, dtype=dt, device=DEV)       # noqa: E731
    lz = lambda n: torch.zeros(n, dtype=torch.long, device=DEV)       # noqa: E731
    C = _C()

    def head(target=None, bias=None, ldd=8, dl=None, dW=None, db=None, dh=None, meter=None, cw=None):
        """A valid head_ce call (B 4, C 3, K 32) with one argument replaced."""
        return C.head_ce(z(4, 32), z(3, 32), z(3, dt=f) if bias is None else bias, lz(4) if target is None else target,
                         z(4, 3, dt=f), z(4, 8) if dl is None else dl, ldd, z(3, 32, dt=f) if dW is None else dW,
                         z(3, dt=f) if db is None else db, z(4, 32) if dh is None else dh, 1.0, True,
                         z(4, dt=f) if meter is None else meter, None, cw)

    def aug(params=None, out=None, pad=4):
        """A valid NHWC augment call (2 images of 16 x 16 to 8 x 8) with one argument replaced."""
        return C.augment(torch.zeros(2, 16, 16, 3, dtype=torch.uint8, device=DEV),
                         z(2, 8, dt=f) if params is None else params, z(2, 8, 8, 4) if out is None else out,
                         16, 16, 8, 8, 0, pad, [0.5] * 3, [0.5] * 3)
    return {
        "fc_grad_act dropout without relu": lambda: C.fc_grad_act(z(4, 8, dt=f), None, z(4, 8), 4, 8, False, 0.5, True),
        "head_ce dropout without relu": lambda: C.head_ce(z(4, 32), z(3, 32), z(3, dt=f),
                                                          torch.zeros(4, dtype=torch.long, device=DEV), z(4, 3, dt=f),
                                                          z(4, 8), 8, z(3, 32, dt=f), z(3, dt=f), z(4, 32), 2.0, False,
                                                          None, None, None),
        "fc_grad_act short act": lambda: C.fc_grad_act(z(4, 8, dt=f), z(4, 4), z(4, 8), 4, 8, True, 0.5, True),
        "fc_bias_act short y": lambda: C.fc_bias_act(z(4, 8, dt=f), None, z(4, 4), None, 4, 8, True, 0.0, 0, 0, True),
        "maxpool_fwd y shape": lambda: C.maxpool_fwd(z(2, 8, 8, 64), z(2, 4, 2, 64)),
        "maxpool_fwd misaligned": lambda: C.maxpool_fwd(_misaligned((2, 8, 8, 64), bf), z(2, 4, 4, 64)),
        "maxpool_relu_bwd dp shape": lambda: C.maxpool_relu_bwd(z(2, 8, 8, 64), z(2, 4, 4, 32), z(2, 8, 8, 64), None),
        "maxpool_relu_bwd dtype": lambda: C.maxpool_relu_bwd(z(2, 8, 8, 64), z(2, 4, 4, 64, dt=f), z(2, 8, 8, 64), None),
        "avgpool_fwd batch": lambda: C.avgpool_fwd(z(2, 4, 4, 64), z(3, 7, 7, 64)),
        "avgpool_bwd mismatch": lambda: C.avgpool_bwd(z(3, 7, 7, 64), z(2, 4, 4, 64)),
        "avgpool_bwd non-contiguous": lambda: C.avgpool_bwd(z(2, 7, 7, 128)[..., :64], z(2, 4, 4, 64)),
        "bias_grad misaligned": lambda: C.bias_grad(_misaligned((64, 64), bf), z(64, dt=f), 64, 64, 64, 1.0),
        "bias_grad short dz": lambda: C.bias_grad(z(63, 64), z(64, dt=f), 64, 64, 64, 1.0),
        "adam misaligned": lambda: C.adam(_misaligned((64,), f), z(64, dt=f), z(64, dt=f), z(64, dt=f), None, None,
                                          1e-3, 0.9, 0.999, 1e-8, 0.0, 1, 1.0, None),
        "adam size": lambda: C.adam(z(64, dt=f), z(60, dt=f), z(64, dt=f), z(64, dt=f), None, None,
                                    1e-3, 0.9, 0.999, 1e-8, 0.0, 1, 1.0, None),
        "adam dtype": lambda: C.adam(z(64, dt=f), z(64, dt=f), z(64, dt=f), z(64, dt=f), None, z(64, dt=f),
                                     1e-3, 0.9, 0.999, 1e-8, 0.0, 1, 1.0, None),
        "adam non-contiguous": lambda: C.adam(z(128, dt=f)[::2], z(64, dt=f), z(64, dt=f), z(64, dt=f), None, None,
                                              1e-3, 0.9, 0.999, 1e-8, 0.0, 1, 1.0, None),
        "sgd misaligned shadow": lambda: C.sgd(z(64, dt=f), z(64, dt=f), z(64, dt=f), None, _misaligned((64,), bf),
                                               0.1, 0.9, 0.0, True, 1.0, None),
        "sgd size": lambda: C.sgd(z(64, dt=f), z(64, dt=f), z(68, dt=f), None, None, 0.1, 0.9, 0.0, True, 1.0, None),
        "cast_to_bf16 misaligned": lambda: C.cast_to_bf16(_misaligned((64,), f), z(64)),
        "cast_to_bf16 size": lambda: C.cast_to_bf16(z(64, dt=f), z(60)),
        "nchw_to_nhwc shape": lambda: C.nchw_to_nhwc(z(2, 3, 8, 8, dt=f), z(2, 8, 4, 4)),
        # wgmma entry points: operand extents against M / N / K, ldo and the epilogue
        "gemm short A": lambda: C.gemm(z(8, 64), False, z(16, 64), False, 16, 16, 64, z(16, 16, dt=f), 16, 0, None,
                                       1.0, 1, 0),
        "gemm short B": lambda: C.gemm(z(16, 64), False, z(8, 64), False, 16, 16, 64, z(16, 16, dt=f), 16, 0, None,
                                       1.0, 1, 0),
        "gemm out dtype": lambda: C.gemm(z(16, 64), False, z(16, 64), False, 16, 16, 64, z(16, 16), 16, 0, None,
                                         1.0, 1, 0),
        "gemm short out": lambda: C.gemm(z(16, 64), False, z(16, 64), False, 16, 16, 64, z(15, 16, dt=f), 16, 0,
                                         None, 1.0, 1, 0),
        "gemm ldo": lambda: C.gemm(z(16, 64), False, z(16, 64), False, 16, 16, 64, z(16, 16, dt=f), 8, 0, None,
                                   1.0, 1, 0),
        "gemm short bias": lambda: C.gemm(z(16, 64), False, z(16, 64), False, 16, 16, 64, z(16, 16), 16, 3,
                                          z(8, dt=f), 1.0, 1, 0),
        "gemm missing bias": lambda: C.gemm(z(16, 64), False, z(16, 64), False, 16, 16, 64, z(16, 16), 16, 3, None,
                                            1.0, 1, 0),
        "conv_fprop short bias": lambda: C.conv_fprop(z(1, 8, 8, 64), z(64, 3, 3, 64), z(32, dt=f), z(1, 8, 8, 64),
                                                      True, 0),
        "conv_fprop_pool short bias": lambda: C.conv_fprop_pool(z(1, 8, 8, 64), z(64, 3, 3, 64), z(32, dt=f),
                                                                z(1, 4, 4, 64), z(1, 4, 4, 2, 4, dt=torch.int32), 0),
        "conv_dgrad dx shape": lambda: C.conv_dgrad(z(1, 8, 8, 64), z(64, 3, 3, 64), None, z(1, 8, 4, 64), None, 0),
        "conv_dgrad mask shape": lambda: C.conv_dgrad(z(1, 8, 8, 64), z(64, 3, 3, 64), z(1, 4, 8, 64),
                                                      z(1, 8, 8, 64), None, 0),
        "conv_dgrad short colsum": lambda: C.conv_dgrad(z(1, 8, 8, 64), z(64, 3, 3, 64), None, z(1, 8, 8, 64),
                                                        z(32, dt=f), 0),
        "conv_wgrad x shape": lambda: C.conv_wgrad(z(1, 8, 8, 64), z(1, 4, 8, 64), z(64, 3, 3, 64, dt=f), 1.0, 0, 0),
        "conv0_fprop y shape": lambda: C.conv0_fprop(z(1, 8, 8, 4), z(64, 64), z(64, dt=f), z(1, 8, 4, 64)),
        "conv0_fprop short bias": lambda: C.conv0_fprop(z(1, 8, 8, 4), z(64, 64), z(32, dt=f), z(1, 8, 8, 64)),
        "conv0_wgrad dz shape": lambda: C.conv0_wgrad(z(1, 8, 4, 64), z(1, 8, 8, 4), z(64, 64, dt=f)),
        # loss kernels: targets, dlogits and the optional outputs against B, C and ldd
        "cross_entropy short targets": lambda: C.cross_entropy(z(4, 3, dt=f), lz(2), z(4, 8), 8, None, None, 0.25,
                                                               None),
        "cross_entropy ldd < C": lambda: C.cross_entropy(z(4, 3, dt=f), lz(4), z(4, 8), 2, None, None, 0.25, None),
        "cross_entropy short dlogits": lambda: C.cross_entropy(z(4, 3, dt=f), lz(4), z(2, 8), 8, None, None, 0.25,
                                                               None),
        "cross_entropy short meter": lambda: C.cross_entropy(z(4, 3, dt=f), lz(4), None, 0, z(2, dt=f), None, 0.25,
                                                             None),
        "cross_entropy short class_weights": lambda: C.cross_entropy(z(4, 3, dt=f), lz(4), None, 0, None, None,
                                                                     0.25, z(2, dt=f)),
        "head_ce short targets": lambda: head(target=lz(2)),
        "head_ce short bias": lambda: head(bias=z(2, dt=f)),
        "head_ce ldd < C": lambda: head(ldd=2),
        "head_ce short dlogits": lambda: head(dl=z(2, 8)),
        "head_ce short dW": lambda: head(dW=z(2, 32, dt=f)),
        "head_ce short db": lambda: head(db=z(2, dt=f)),
        "head_ce short dh": lambda: head(dh=z(2, 32)),
        "head_ce short meter": lambda: head(meter=z(2, dt=f)),
        "head_ce short class_weights": lambda: head(cw=z(2, dt=f)),
        # input kernels
        "augment params shape": lambda: aug(params=z(2, 7, dt=f)),
        "augment short params": lambda: aug(params=z(1, 8, dt=f)),
        "augment short out": lambda: aug(out=z(1, 8, 8, 4)),
        "augment pad < 3": lambda: aug(out=z(2, 8, 8, 2), pad=2),
        "im2col_c3 short out": lambda: C.im2col_c3(z(2, 8, 8, 4), z(64, 64), 64),
        "im2col_c3 x channels": lambda: C.im2col_c3(z(2, 8, 8, 3), z(128, 64), 64),
    }


REFUSALS = ["fc_grad_act dropout without relu", "head_ce dropout without relu", "fc_grad_act short act",
            "fc_bias_act short y", "maxpool_fwd y shape", "maxpool_fwd misaligned", "maxpool_relu_bwd dp shape",
            "maxpool_relu_bwd dtype", "avgpool_fwd batch", "avgpool_bwd mismatch", "avgpool_bwd non-contiguous",
            "bias_grad misaligned", "bias_grad short dz", "adam misaligned", "adam size", "adam dtype",
            "adam non-contiguous", "sgd misaligned shadow", "sgd size", "cast_to_bf16 misaligned",
            "cast_to_bf16 size", "nchw_to_nhwc shape",
            "gemm short A", "gemm short B", "gemm out dtype", "gemm short out", "gemm ldo", "gemm short bias",
            "gemm missing bias", "conv_fprop short bias", "conv_fprop_pool short bias", "conv_dgrad dx shape",
            "conv_dgrad mask shape", "conv_dgrad short colsum", "conv_wgrad x shape", "conv0_fprop y shape",
            "conv0_fprop short bias", "conv0_wgrad dz shape", "cross_entropy short targets", "cross_entropy ldd < C",
            "cross_entropy short dlogits", "cross_entropy short meter", "cross_entropy short class_weights",
            "head_ce short targets", "head_ce short bias", "head_ce ldd < C", "head_ce short dlogits",
            "head_ce short dW", "head_ce short db", "head_ce short dh", "head_ce short meter",
            "head_ce short class_weights", "augment params shape", "augment short params", "augment short out",
            "augment pad < 3", "im2col_c3 short out", "im2col_c3 x channels"]


@pytest.mark.parametrize("case", REFUSALS)
def test_host_refuses_before_launching(case):
    """Each argument check raises, and nothing was launched (the native launch counter is unchanged)."""
    ops = _ops()
    fn = _refusals()[case]
    torch.cuda.synchronize()
    n0 = ops.launch_count()
    with pytest.raises(RuntimeError):
        fn()
    assert ops.launch_count() == n0
