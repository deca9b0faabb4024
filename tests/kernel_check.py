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
          family: str = "", what: str = "") -> float:
    """Assert the criterion on every element; returns the worst err/bound ratio (0 in exact mode)."""
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
    err = (g - ref).abs()
    bound = (EPS_BF16 if bf else 0.0) * ref.abs() + gamma(chain) * mag
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


def _pow2_div(x: int, cap: int) -> int:
    p = 1
    while p * 2 <= cap and x % (p * 2) == 0:
        p *= 2
    return p


def wgrad_chain(N: int, H: int, W: int, Cin: int, Cout: int, sms: int) -> int:
    """conv3x3_wgrad with its default split: k16 steps over one split's pixel tiles + the splits."""
    if Cin == 64 and H % 8 == 0 and W % 8 == 0 and W >= 16:          # wgrad_halo64: 8 x 8 pixel tiles
        tiles = N * (H // 8) * (W // 8)
        ks = max(1, min(sms // _cdiv(Cout, 64), tiles))
    else:                                                            # WgradPolicy: 64-pixel boxes
        wb = _pow2_div(W, 32)
        hb = _pow2_div(H, 64 // wb)
        nb = 64 // (wb * hb)
        tiles = _cdiv(W, wb) * _cdiv(H, hb) * _cdiv(N, nb)
        base = _cdiv(Cout, 128) * _cdiv(Cin, 64 if Cin <= 64 else 128) * 9
        ks = min(max(_cdiv(tiles, 64), _cdiv(4 * sms, base)), tiles)
    per = _cdiv(tiles, ks)
    return 4 * per + _cdiv(tiles, per) + 1


def conv0_wgrad_chain(pixels: int, sms: int) -> int:
    """conv0_wgrad: k-blocks of 64 pixels spread over at most one CTA per SM, two accumulators each."""
    tiles = _cdiv(pixels, 64)
    grid = min(tiles, sms)
    return 4 * _cdiv(tiles, grid) + 2 * grid


def conv_colsum_chain(pixels: int, channels: int, sms: int) -> int:
    """Fused column sum of conv dgrad: a 5-level warp reduction, at most four warp sums per tile into
    the CTA's shared-memory sums, one global atomic per CTA."""
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

