"""Per-element acceptance criterion for the wgmma kernels against the float64 references of ops.ref.

Every element must satisfy

    |got - ref| <= eps_out * |ref| + gamma * mag

where ``mag`` is the reference evaluated on |operands|, ``eps_out`` is 2^-8 for bf16 outputs (one
round-to-nearest-even) and 0 for fp32 outputs, and ``gamma = chain * 2^-24 * SAFETY``: ``chain`` is
the longest sequence of fp32 additions the kernel makes to produce one element (k16 wgmma steps of
one split, plus the split-K partials added atomically, plus the epilogue's own operations).  Unlike
an error relative to the tensor's maximum, this bound is as tight for a small border pixel or a late
channel chunk as for the largest output.

Two input modes:

* ``exact``: operands are small integers (|v| <= 4 when the reduction is at most 4608 deep, else
  {-1, 0, 1}) and biases multiples of 1/4, so every partial sum is an fp32 integer below 2^24 in any
  order.  fp32 outputs must then equal the reference exactly and bf16 outputs must equal its RNE
  rounding (+0 and -0 count as equal).  A dropped or doubled k-block, tap or split shows at any depth.
* ``gauss``: Gaussian operands, checked against the bound.
"""
from __future__ import annotations

import torch

U32 = 2.0 ** -24            # unit roundoff of fp32
EPS_BF16 = 2.0 ** -8        # unit roundoff of bf16
# Margin over the chain estimate: wgmma may add the 16 products of a k-step with less than fp32
# precision.  Worst err/bound of the gauss-mode tests on one H100 80GB HBM3 (700 W limit), fp32
# outputs: GEMM 0.11, conv wgrad 0.014, conv0 wgrad 0.007, column sums <= 0.002 -- below 1 / SAFETY.
# bf16 outputs reach 0.99 because their own rounding may use the whole 2^-8 |ref| term.
# Memory-bound kernels (test_elementwise_gpu.py and the replay, H100 80GB HBM3 at a 400 W limit),
# fp32 outputs: Adam p 0.25, m 0.19, v 0.17; SGD p 0.25, momentum 0.24; bias_grad 0.12; head_ce db 0.12,
# dW 0.02, logits 0.04, loss 0.02; cross_entropy loss 0.04; max-pool column sum 6e-5.  The optimizer
# bounds are running bounds without slack of their own, so their worst case sits at 1 / SAFETY.
SAFETY = 4.0
EXACT_DEPTH = 4608          # deepest reduction that gets |v| <= 4 operands (|sum| <= 16 * 4608 < 2^24)

worst_ratio: dict = {}      # family -> worst err/bound seen in gauss mode in this process


def gamma(chain: float) -> float:
    return chain * U32 * SAFETY


def operand(shape, mode: str, depth: int, gen: torch.Generator, device, scale: float = 1.0) -> torch.Tensor:
    """bf16 operand of a reduction of ``depth`` terms."""
    if mode == "exact":
        a = 4 if depth <= EXACT_DEPTH else 1
        return torch.randint(-a, a + 1, tuple(shape), generator=gen, device=device).to(torch.bfloat16)
    return (torch.randn(tuple(shape), generator=gen, device=device) * scale).to(torch.bfloat16)


def bias(n: int, mode: str, gen: torch.Generator, device) -> torch.Tensor:
    """fp32 bias: multiples of 1/4 in [-8, 8] (exact) or N(0, 0.1^2)."""
    if mode == "exact":
        return torch.randint(-32, 33, (n,), generator=gen, device=device).float() / 4
    return torch.randn(n, generator=gen, device=device) * 0.1


def check(got: torch.Tensor, ref: torch.Tensor, mag: torch.Tensor, *, chain: float, exact: bool,
          family: str = "", what: str = "", err=None) -> float:
    """Assert the criterion on every element; returns the worst err/bound ratio (0 in exact mode).
    ``err`` (optional, absolute units) is a derived error bound of arithmetic that is not a chain of
    additions (ce_bound, the optimizer references); it is added to the bound times SAFETY."""
    assert got.shape == ref.shape == mag.shape, (what, tuple(got.shape), tuple(ref.shape), tuple(mag.shape))
    bf = got.dtype == torch.bfloat16
    g = got.to(torch.float64)
    if exact:
        want = ref.to(torch.bfloat16 if bf else torch.float32).to(torch.float64)
        bad = ~(g == want)
        n = int(bad.sum())
        if n:
            i = int((g - want).abs().nan_to_num(float("inf")).argmax())
            idx = tuple(int(v) for v in torch.unravel_index(torch.tensor(i), got.shape))
            raise AssertionError("%s %s: %d of %d elements differ from the exact result; worst at %s: got %r, "
                                 "expected %r" % (family, what, n, got.numel(), idx, float(g.flatten()[i]),
                                                  float(want.flatten()[i])))
        return 0.0
    bound = (EPS_BF16 if bf else 0.0) * ref.abs() + gamma(chain) * mag
    if err is not None:
        bound = bound + SAFETY * err
    err = (g - ref).abs()
    ratio = torch.where(err == 0, torch.zeros_like(err), err / bound).nan_to_num(float("inf"))
    i = int(ratio.argmax())
    worst = float(ratio.flatten()[i])
    if family:
        key = "%s:%s" % (family, "bf16" if bf else "f32")
        worst_ratio[key] = max(worst_ratio.get(key, 0.0), worst)
        print("[kernel_check] %s %s worst err/bound %.3g" % (key, what, worst))
    if not worst <= 1.0:
        idx = tuple(int(v) for v in torch.unravel_index(torch.tensor(i), got.shape))
        raise AssertionError("%s %s: err/bound %.3g at %s (got %r, ref %r, mag %r, chain %g); %d elements over" %
                             (family, what, worst, idx, float(g.flatten()[i]), float(ref.flatten()[i]),
                              float(mag.flatten()[i]), chain, int((ratio > 1).sum())))
    return worst


def check_pool(pooled: torch.Tensor, mask: torch.Tensor, y_ref: torch.Tensor, y_mag: torch.Tensor, *,
               chain: float, exact: bool, family: str = "conv_fprop_pool", what: str = "") -> float:
    """The fused conv + ReLU + 2x2 pool against the un-pooled float64 reference y_ref (post-ReLU):
    the pooled bf16 value, the argmax (first maximum in window order) and the "max > 0" bit.  The
    argmax only matters where the maximum is positive (elsewhere the gradient is zero whatever it
    says) and is checked there; in gauss mode only in windows whose top two values are further
    apart than the error bound allows them to swap, and "max > 0" only where the maximum exceeds
    its bound."""
    from distributed_vgg_f_b200.ops import ref as R

    C = y_ref.shape[-1]
    idx, pos = R.pool_mask_decode(mask, C)
    if exact:
        val, ridx, rpos = R.pool2x2_select(y_ref.to(torch.bfloat16).to(torch.float64))
        check(pooled, val, val, chain=0, exact=True, family=family, what=what + " pooled")
        sure_pos, sure_idx = torch.ones_like(rpos), rpos
        worst = 0.0
    else:
        win = R.pool_windows(y_ref)
        bnd = R.pool_windows(EPS_BF16 * y_ref.abs() + gamma(chain) * y_mag).amax(-1)
        top2, ridx = win.topk(2, dim=-1)
        ridx = ridx[..., 0]
        val = top2[..., 0]
        rpos = val > 0
        worst = check(pooled, val, R.pool_windows(y_mag).amax(-1), chain=chain, exact=False, family=family,
                      what=what + " pooled")
        sure_pos = (val.abs() > bnd)
        sure_idx = rpos & (top2[..., 0] - top2[..., 1] > 2 * bnd)
    bad = sure_pos & (pos != rpos)
    if bool(bad.any()):
        i = tuple(int(v) for v in bad.nonzero()[0])
        raise AssertionError("%s %s: 'max > 0' bit wrong at %s (got %s)" % (family, what, i, bool(pos[i])))
    bad = sure_idx & (idx != ridx)
    if bool(bad.any()):
        i = tuple(int(v) for v in bad.nonzero()[0])
        raise AssertionError("%s %s: %d argmax entries wrong, first at %s: got %d, expected %d" %
                             (family, what, int(bad.sum()), i, int(idx[i]), int(ridx[i])))
    return worst


# ---------------------------------------------------------------- chains of the kernel families
def _cdiv(a: int, b: int) -> int:
    return -(-a // b)


def gemm_chain(K: int, ksplit: int = 1) -> int:
    """umma GEMM: k16 steps of one split + the splits added atomically + the epilogue operation."""
    iters = _cdiv(K, 64)
    per = _cdiv(iters, max(ksplit, 1))
    return 4 * per + _cdiv(iters, per) + 1


def conv_chain(depth_channels: int) -> int:
    """Implicit-GEMM conv fprop / dgrad: 9 taps x C/16 k16 steps, then bias (fprop)."""
    return 9 * depth_channels // 16 + 2


def split_chain(tiles_per_split: int, ksplit: int) -> int:
    """Split-K wgrad: k16 steps over one split's 64-pixel tiles + the splits added + the epilogue operation."""
    return 4 * tiles_per_split + ksplit + 1


def wgrad_chain(N: int, H: int, W: int, Cin: int, Cout: int, sms: int, kind: str = "wgrad", bn: int = 0) -> int:
    """conv3x3_wgrad (``kind`` "wgrad_partial": conv3x3_wgrad_partial + the reduce) with its default split, at
    tile width ``bn`` (0: the launcher's own), as the launcher plans it (conv_plan: needs the extension)."""
    from distributed_vgg_f_b200 import ops

    p = ops.require().conv_plan(kind, N, H, W, Cin, Cout, sms, bn)
    return split_chain(p["tiles_per_split"], p["ksplit"])


def conv0_wgrad_chain(pixels: int, sms: int) -> int:
    """conv0_wgrad: k-blocks of 64 pixels spread over at most one CTA per SM, two accumulators each."""
    tiles = _cdiv(pixels, 64)
    grid = min(tiles, sms)
    return 4 * _cdiv(tiles, grid) + 2 * grid


def conv_colsum_chain(pixels: int, channels: int, sms: int, tiles: int = None) -> int:
    """Fused column sum of conv dgrad: a 5-level warp reduction, at most four warp sums per tile into
    the CTA's shared-memory sums, one global atomic per CTA.  ``tiles``: the launch's pixel tiles times
    its 64-channel blocks, where the pixel box does not fill the 128-row tile (default: full tiles)."""
    if tiles is None:
        tiles = _cdiv(pixels, 128) * _cdiv(channels, 64)
    return 5 + 4 * _cdiv(tiles, min(tiles, sms)) + sms


def unpool_colsum_chain(pooled_pixels: int, channels: int, sms: int) -> int:
    """unpool2x2 / maxpool2x2_relu_bwd column sum: a grid-stride loop per thread, shared-memory atomics
    of the threads that own the channel, one global atomic per block."""
    c8 = channels // 8
    total = pooled_pixels * c8
    blocks = min(_cdiv(total, 256), 16 * sms)
    return _cdiv(total, blocks * 256) + 256 // c8 + blocks


def sm_count() -> int:
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def generator(seed: int, device) -> torch.Generator:
    return torch.Generator(device=device).manual_seed(seed)



# ------------------------------------------------- chains and bounds of the memory-bound kernels
def avgpool_chain(terms: int) -> int:
    """adaptive_avgpool_fwd / _bwd: ``terms`` is the most window elements one output sums (forward:
    ops.ref.ap_max_window squared) or the most windows one input lies in (backward: ap_max_cover
    squared).  Each term costs at most an fp32 1/count, a product and an add."""
    return 3 * terms


def bias_grad_chain(rows: int, C: int, sms: int, ld: int = None) -> int:
    """bias_grad with the launch geometry of elementwise.cu::bias_grad(): CG column groups of 8
    channels (<= 256) x RL = 256 / CG row lanes; blocks of RL * 16 rows, capped at 8 blocks per SM per
    column-group slice; each lane adds every RL-th row of its block's rows_per_block, lane 0 adds the
    other RL - 1 lanes, multiplies by scale, and each block adds its sum atomically.  C % 8 != 0 or
    ld != C takes bias_grad_ld: one thread adds all rows."""
    if C % 8 or (ld is not None and ld != C):
        return rows + 2
    c8 = C // 8
    CG = min(c8, 256)
    RL = max(256 // CG, 1)
    nblk = _cdiv(rows, RL * 16)
    nblk = max(min(nblk, sms * 8 // _cdiv(c8, CG)), 1)
    rpb = _cdiv(rows, nblk)
    return _cdiv(rpb, RL) + RL + 1 + _cdiv(rows, rpb)


def head_chain(K: int, B: int) -> dict:
    """head_ce: logits = fmas over one lane's K / 32 inputs, 5 shuffle adds and the bias; dW[c][k] and
    db[c] are serial sums over the B rows (db added to the buffer's value); dh = at most 8 fmas over the
    classes, times drop_scale."""
    return {"logits": _cdiv(K, 32) + 6, "dW": B, "db": B + 1, "dh": 9}


# CUDA C++ Programming Guide, table of intrinsic functions (single precision):
#   __expf(x): at most 2 + floor(|1.173 x|) ulp;
#   __logf(x): at most 2^-21.41 absolute for x in [0.5, 2], else 3 ulp.
# One ulp of a normal fp32 value y is at most 2^-23 |y|.
def _expf_rel(x: torch.Tensor) -> torch.Tensor:
    return (2 + torch.floor((1.173 * x).abs())) * 2.0 ** -23


def _logf_abs(s: torch.Tensor) -> torch.Tensor:
    L = s.log()
    inner = (s >= 0.5) & (s <= 2.0)
    return torch.where(inner, torch.full_like(s, 2.0 ** -21.41), 3 * 2.0 ** -23 * L.abs())


def ce_bound(logits: torch.Tensor, target: torch.Tensor, *, class_weights=None, grad_scale=None,
             se_chain: int, warps: int) -> dict:
    """First-order bound of what cross_entropy_kernel / head_ce_kernel may get wrong, per output, in
    absolute units, for the fp32 logits z the kernel saw (u = 2^-24 per fp32 operation):

      x_c = z_c - max            rounded:          |dx_c| <= u |x_c|
      e_c = __expf(x_c)          relative error    r(x_c) = (2 + floor|1.173 x_c|) 2^-23, plus |dx_c|
      se  = sum_c e_c            se_chain adds of positive terms (lanes, then 5 shuffles, or serial)
                                 |dse| <= sum_c e_c (r(x_c) + u|x_c|) + se_chain u se
      lse = max + __logf(se)     |dlse| <= |dse| / se + logf_abs(se) + u |lse|
      nll = w (lse - z_t)        |dnll| <= w (|dlse| + 2u |lse - z_t|)
      loss = sum nll / D         rows / warps per warp, then the warps: |dsum| <= sum|dnll| + chain u sum|nll|;
                                 D = B exact, or sum w with its own chain; one division
      a_c = z_c - lse            |da_c| <= |dlse| + u |a_c|
      g_c = (__expf(a_c) - [c == t]) w norm
                                 |dg_c| <= w norm (p_c (|da_c| + r(a_c)) + u |p_c - [c == t]|) + 3u |g_c| + |g_c| dnorm
    The bf16 rounding of dlogits is check()'s own 2^-8 |ref| term; results below 2^-126 may be flushed
    to zero, hence an absolute 2^-126 more.  Returns {"loss", "dlogits" [B][C],
    "meter0"}."""
    u = U32
    z = logits.to(torch.float64)
    B, C = z.shape
    t = target.to(torch.int64).view(-1)
    mx = z.amax(1, keepdim=True)
    x = z - mx
    e = x.exp()
    se = e.sum(1)
    dse = (e * (_expf_rel(x) + u * x.abs())).sum(1) + se_chain * u * se
    L = se.log()
    lse = mx.view(-1) + L
    dlse = dse / se + _logf_abs(se) + u * lse.abs()
    if class_weights is not None:
        w = class_weights.to(torch.float64)[t]
        D = w.sum()
        dD = (_cdiv(B, 1024) + 5 + warps) * u * D
        norm, dnorm = 1.0 / D, dD / D + u
    else:
        w = torch.ones(B, dtype=torch.float64, device=z.device)
        D, dD = float(B), 0.0
        norm, dnorm = (1.0 / B if grad_scale is None else grad_scale), 0.0
    zt = z.gather(1, t.view(-1, 1)).view(-1)
    nll = w * (lse - zt)
    dnll = w * (dlse + 2 * u * (lse - zt).abs())
    tl = nll.sum()
    dtl = dnll.sum() + (_cdiv(B, warps) + warps) * u * nll.abs().sum()
    loss = tl / D
    dloss = dtl / D + tl.abs() * dD / D ** 2 + u * loss.abs()
    a = z - lse[:, None]
    p = a.exp()
    onehot = torch.nn.functional.one_hot(t, C).to(torch.float64)
    g = (p - onehot) * (w * norm)[:, None]
    dg = (w * norm)[:, None] * (p * (dlse[:, None] + u * a.abs() + _expf_rel(a)) + u * (p - onehot).abs()) \
        + g.abs() * (3 * u + dnorm) + (w * norm)[:, None] * 2.0 ** -126 + 2.0 ** -126
    return {"loss": dloss, "dlogits": dg, "meter0": B * dloss + u * B * loss.abs()}
