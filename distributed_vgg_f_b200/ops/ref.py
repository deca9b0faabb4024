"""Plain-PyTorch fp32 references of the engine's ops, chained exactly like the engine chains its
kernels -- including *where* tensors are rounded to bf16 (activations, activation gradients) --
so that an engine step can be checked layer by layer with tight tolerances.  Also the building
blocks used as oracles in tests/test_kernels_gpu.py.

All functions take/return NCHW fp32 tensors holding bf16-representable values where the engine
stores bf16.
"""
from __future__ import annotations

from typing import Dict, List

import torch
import torch.nn.functional as F

from ..models.vggf import VGGSpec


def rb(t: torch.Tensor) -> torch.Tensor:
    """Round to bf16 and back (what storing a tensor as bf16 does)."""
    return t.to(torch.bfloat16).to(torch.float32)


def pool_relu_bwd(y: torch.Tensor, dp: torch.Tensor) -> torch.Tensor:
    """Backward of [ReLU -> maxpool2x2] given the post-ReLU map y: first maximal element wins."""
    with torch.enable_grad():
        yr = y.detach().clone().requires_grad_(True)
        F.max_pool2d(yr, 2, 2).backward(dp)
    return yr.grad * (y > 0)


@torch.no_grad()
def emulated_step(spec: VGGSpec, state: Dict[str, torch.Tensor], x: torch.Tensor, target: torch.Tensor,
                  dropout_masks: bool = False, return_intermediates: bool = False,
                  override: dict = None, soft_target: torch.Tensor = None, label_smoothing: float = 0.0,
                  teacher_logits: torch.Tensor = None, distill_alpha: float = 0.5, distill_temperature: float = 4.0):
    """Forward + backward of the network on fp32 torch ops with the engine's rounding points.

    state: torch-layout fp32 tensors (weights are rounded to bf16 here, biases stay fp32).
    Returns (logits, mean loss, grads in torch layout).  Dropout is treated as identity.

    ``soft_target`` (probability targets [B][C], e.g. MixUp / CutMix) and ``label_smoothing``: the loss
    is F.cross_entropy(logits, soft_target or target, label_smoothing=) and its gradient
    (softmax - t) / B with t the smoothed target.

    ``teacher_logits`` ([B][C], optional): knowledge distillation with weight ``distill_alpha`` and temperature
    ``distill_temperature`` -- the loss is (1 - a) CE + a T^2 KL(softmax(u / T) || softmax(z / T)) / B and its
    gradient (1 - a) (the CE gradient) + a T (softmax(z / T) - softmax(u / T)) / B, rounded to bf16 once.

    ``override`` (optional) pins the forward state to tensors observed elsewhere -- keys ``acts``
    (post-ReLU conv outputs, NCHW), ``feat`` (pooled feature map), ``fc_y`` (hidden FC outputs),
    ``logits``.  ReLU / max-pool gating is discontinuous: a 1-ulp difference in a near-zero
    activation flips a mask and moves a whole gradient row, so a *backward* check is only tight
    when both sides gate on the same forward values.
    """
    override = override or {}
    w = {k: (rb(v) if v.dim() > 1 else v.float()) for k, v in state.items()}
    acts: List[torch.Tensor] = []
    pools: List[torch.Tensor] = []
    a = rb(x)
    conv_in: List[torch.Tensor] = []
    for c in spec.convs:
        conv_in.append(a)
        y = rb(torch.relu(F.conv2d(a, w[c.name + ".weight"], w[c.name + ".bias"], padding=1)))
        if "acts" in override:
            y = override["acts"][len(acts)].float()
        acts.append(y)
        a = y
        if c.pool_after:
            a = F.max_pool2d(y, 2, 2)
        pools.append(a)
    feat_hw = a.shape[-1]
    feat = a
    if feat_hw != spec.pooled_hw:
        feat = rb(F.adaptive_avg_pool2d(a, (spec.pooled_hw, spec.pooled_hw)))
    if "feat" in override:
        feat = override["feat"].float()
    # the engine flattens NHWC; torch-layout FC-1 weights expect NCHW flatten -- same values
    h = torch.flatten(feat, 1)
    fc_in: List[torch.Tensor] = []
    last = len(spec.fcs) - 1
    for i, f in enumerate(spec.fcs):
        fc_in.append(h)
        z = h @ w[f.name + ".weight"].t() + w[f.name + ".bias"]
        if i == last:
            logits = override["logits"].float() if "logits" in override else z
        else:
            h = rb(torch.relu(z) if f.relu else z)
            if "fc_y" in override:
                h = override["fc_y"][i].float()
    B = x.shape[0]
    logp = torch.log_softmax(logits, dim=1)
    if soft_target is None and not label_smoothing:
        loss = -logp.gather(1, target.view(-1, 1)).mean()
        dz = rb((torch.softmax(logits, 1) - F.one_hot(target, logits.shape[1]).float()) / B)
    else:
        t = soft_target.float() if soft_target is not None else F.one_hot(target, logits.shape[1]).float()
        t = t * (1.0 - label_smoothing) + label_smoothing / logits.shape[1]
        loss = -(t * logp).sum(1).mean()
        dz = rb((torch.softmax(logits, 1) - t) / B)
    if teacher_logits is not None:
        a, T = float(distill_alpha), float(distill_temperature)
        t = F.one_hot(target, logits.shape[1]).float() if soft_target is None else soft_target.float()
        t = t * (1.0 - label_smoothing) + label_smoothing / logits.shape[1]
        lps, lpt = torch.log_softmax(logits / T, 1), torch.log_softmax(teacher_logits.float() / T, 1)
        kl = (lpt.exp() * (lpt - lps)).sum() / B
        loss = (1.0 - a) * loss + a * T * T * kl
        dz = rb((1.0 - a) * (torch.softmax(logits, 1) - t) / B + a * T * (lps.exp() - lpt.exp()) / B)

    grads: Dict[str, torch.Tensor] = {}
    inter = {"fc_dz": {}, "fc_y": {i: fc_in[i + 1] for i in range(last)}, "conv_dz": {}}
    for i in range(last, -1, -1):
        f = spec.fcs[i]
        inter["fc_dz"][i] = dz
        grads[f.name + ".bias"] = dz.sum(0)
        grads[f.name + ".weight"] = dz.t() @ fc_in[i]
        dacc = dz @ w[f.name + ".weight"]
        if i > 0:
            prev = spec.fcs[i - 1]
            dz = rb(dacc * (fc_in[i] > 0)) if prev.relu else rb(dacc)
        else:
            g = rb(dacc).view_as(feat)
            inter["dfeat"] = g
    if feat_hw != spec.pooled_hw:
        src = pools[-1].detach().clone().requires_grad_(True)
        with torch.enable_grad():
            F.adaptive_avg_pool2d(src, (spec.pooled_hw, spec.pooled_hw)).backward(g)
        g = rb(src.grad)
    for i in range(len(spec.convs) - 1, -1, -1):
        c = spec.convs[i]
        y = acts[i]
        if c.pool_after:
            with torch.enable_grad():
                dzc = rb(pool_relu_bwd(y, g))
        else:
            dzc = g
        inter["conv_dz"][i] = dzc
        grads[c.name + ".bias"] = dzc.sum((0, 2, 3))
        xin = conv_in[i]
        grads[c.name + ".weight"] = torch.nn.grad.conv2d_weight(xin, w[c.name + ".weight"].shape, dzc, padding=1)
        if i == 0:
            break
        dx = F.conv_transpose2d(dzc, w[c.name + ".weight"], padding=1)
        if spec.convs[i - 1].pool_after:
            g = rb(dx)
        else:
            g = rb(dx * (xin > 0))
    if return_intermediates:
        return logits, loss, grads, inter
    return logits, loss, grads


# -------------------------------------------------------------------- float64 kernel references
# One reference per wgmma kernel family, in the kernel's own layouts (NHWC activations, OHWI conv
# weights).  Each returns (ref, mag): the exact result of the operation on the (bf16) inputs in
# float64, and the same operation on |inputs| -- the scale of the rounding errors an fp32
# accumulation of that sum can make, element by element.  Nothing here picks an algorithm: the
# convolutions are nine shifted GEMMs.

def _f64(t: torch.Tensor) -> torch.Tensor:
    return t.to(torch.float64)


def gemm64(a: torch.Tensor, b: torch.Tensor, *, M: int, N: int, K: int, a_mn: bool = False,
           b_mn: bool = False, epi: str = "f32_store", bias=None, alpha: float = 1.0):
    """ops.gemm: out = alpha * A B^T (A [M][K] or, a_mn, [K][M]; B [N][K] or, b_mn, [K][N]).
    Returned [M][N], or [N][M] for the transposed stores (*_t); f32_atomic* are the sum the
    kernel adds to a zeroed output; bf16_bias_relu is relu(A B^T + bias) (no alpha)."""
    A = _f64(a[:K, :M].t() if a_mn else a[:M, :K])
    B = _f64(b[:K, :N].t() if b_mn else b[:N, :K])
    ref, mag = A @ B.t(), A.abs() @ B.abs().t()
    if epi == "bf16_bias_relu":
        if bias is not None:
            ref, mag = ref + _f64(bias[:N]), mag + _f64(bias[:N]).abs()
        ref = torch.relu(ref)
    else:
        ref, mag = alpha * ref, abs(alpha) * mag
    if epi.endswith("_t"):
        ref, mag = ref.t(), mag.t()
    return ref.contiguous(), mag.contiguous()


def _taps(x: torch.Tensor):
    """The nine (kh, kw) shifted views x[n, h + kh - 1, w + kw - 1, :] of an NHWC tensor, zero padded,
    as [pixels][C] matrices."""
    N, H, W, C = x.shape
    xp = torch.zeros(N, H + 2, W + 2, C, dtype=torch.float64, device=x.device)
    xp[:, 1:H + 1, 1:W + 1] = _f64(x)
    for kh in range(3):
        for kw in range(3):
            yield kh, kw, xp[:, kh:kh + H, kw:kw + W].reshape(-1, C)


def conv3x3_fprop64(x: torch.Tensor, w: torch.Tensor, bias=None, relu: bool = True):
    """3x3/s1/p1 conv: x NHWC [N,H,W,Cin], w [Cout][3][3][Cin] -> [N,H,W,Cout]."""
    N, H, W, _ = x.shape
    w64 = _f64(w)
    ref = torch.zeros(N * H * W, w.shape[0], dtype=torch.float64, device=x.device)
    mag = torch.zeros_like(ref)
    for kh, kw, xs in _taps(x):
        wt = w64[:, kh, kw, :]
        ref += xs @ wt.t()
        mag += xs.abs() @ wt.abs().t()
    if bias is not None:
        ref, mag = ref + _f64(bias), mag + _f64(bias).abs()
    if relu:
        ref = torch.relu(ref)
    return ref.view(N, H, W, -1), mag.view(N, H, W, -1)


def conv3x3_dgrad64(dz: torch.Tensor, w: torch.Tensor, mask_src=None):
    """dx[n,h,w,ci] = sum_{kh,kw,co} dz[n, h-kh+1, w-kw+1, co] w[co,kh,kw,ci], times (mask_src > 0)."""
    N, H, W, _ = dz.shape
    w64 = _f64(w)
    ref = torch.zeros(N * H * W, w.shape[3], dtype=torch.float64, device=dz.device)
    mag = torch.zeros_like(ref)
    for kh, kw, dzs in _taps(dz):
        wt = w64[:, 2 - kh, 2 - kw, :]                    # dz shifted by (kh-1, kw-1) meets the mirrored tap
        ref += dzs @ wt
        mag += dzs.abs() @ wt.abs()
    ref, mag = ref.view(N, H, W, -1), mag.view(N, H, W, -1)
    if mask_src is not None:
        keep = (mask_src.float() > 0).to(torch.float64)
        ref, mag = ref * keep, mag * keep
    return ref, mag


def conv3x3_wgrad64(dz: torch.Tensor, x: torch.Tensor, scale: float = 1.0):
    """dw[co,kh,kw,ci] = scale * sum_{n,h,w} dz[n,h,w,co] x[n, h+kh-1, w+kw-1, ci]."""
    Cout, Cin = dz.shape[3], x.shape[3]
    dz2 = _f64(dz).reshape(-1, Cout)
    ref = torch.zeros(Cout, 3, 3, Cin, dtype=torch.float64, device=dz.device)
    mag = torch.zeros_like(ref)
    for kh, kw, xs in _taps(x):
        ref[:, kh, kw] = dz2.t() @ xs
        mag[:, kh, kw] = dz2.abs().t() @ xs.abs()
    return scale * ref, abs(scale) * mag


def conv0_fprop64(x4: torch.Tensor, w0: torch.Tensor, bias):
    """First conv on NHWC4 pixels (channel 3 unused): w0 [64][64] holds the [kh][kw][c] taps in
    columns 0..26 -> relu(conv + bias) [N,H,W,64]."""
    return conv3x3_fprop64(x4[..., :3], w0[:, :27].reshape(-1, 3, 3, 3), bias, relu=True)


def conv0_wgrad64(dz: torch.Tensor, x4: torch.Tensor):
    """Weight gradient of conv0 in the [64][64] layout of w0: columns 27..63 are zero."""
    r, m = conv3x3_wgrad64(dz, x4[..., :3])
    ref = torch.zeros(dz.shape[3], 64, dtype=torch.float64, device=dz.device)
    mag = torch.zeros_like(ref)
    ref[:, :27], mag[:, :27] = r.reshape(-1, 27), m.reshape(-1, 27)
    return ref, mag


def pool_windows(t: torch.Tensor) -> torch.Tensor:
    """[N,H,W,C] -> [N,H/2,W/2,C,4]: the 2x2 windows in the order (0,0), (0,1), (1,0), (1,1).  Floor mode:
    an odd last row / column lies in no window."""
    N, H, W, C = t.shape
    v = t[:, :H // 2 * 2, :W // 2 * 2].reshape(N, H // 2, 2, W // 2, 2, C)
    return v.permute(0, 1, 3, 5, 2, 4).reshape(N, H // 2, W // 2, C, 4)


def pool2x2_select(y: torch.Tensor):
    """The fused pool on a stored (bf16) post-ReLU map y: (pooled max, argmax 0..3 = first maximum in
    window order, max > 0).  torch.max returns the first maximal index, like the kernel."""
    win = pool_windows(y)
    val, idx = win.max(dim=-1)
    return val, idx, val > 0


def pool_mask_decode(mask: torch.Tensor, C: int):
    """Mask words [N,OH,OW,C/32,4] int32 = {argmax bit 0, argmax bit 1, max > 0, 0} per 32 channels
    -> (argmax [N,OH,OW,C] in 0..3, positive [N,OH,OW,C] bool)."""
    m = mask.to(torch.int64) & 0xFFFFFFFF
    bits = torch.arange(32, device=mask.device)
    per = (m[..., None] >> bits) & 1                                      # [N,OH,OW,C/32,4,32]
    b0, b1, pos = per[..., 0, :], per[..., 1, :], per[..., 2, :]
    sh = mask.shape[:3] + (C,)
    return (b0 | (b1 << 1)).reshape(sh), pos.reshape(sh).bool()


def pool_mask_encode(idx: torch.Tensor, pos: torch.Tensor) -> torch.Tensor:
    """Inverse of pool_mask_decode."""
    N, OH, OW, C = idx.shape
    bits = (1 << torch.arange(32, device=idx.device, dtype=torch.int64))
    i, p = idx.to(torch.int64).view(N, OH, OW, C // 32, 32), pos.to(torch.int64).view(N, OH, OW, C // 32, 32)
    words = torch.stack([((i & 1) * bits).sum(-1), (((i >> 1) & 1) * bits).sum(-1), (p * bits).sum(-1),
                         torch.zeros_like(i[..., 0])], dim=-1)
    return torch.where(words >= 2 ** 31, words - 2 ** 32, words).to(torch.int32)


def unpool2x2_64(dp: torch.Tensor, idx: torch.Tensor, pos: torch.Tensor):
    """Backward of the fused pool: dp goes to the recorded argmax of each window where the max was > 0.
    Returns (dz [N,2*OH,2*OW,C], column sum of dz, column sum of |dz|)."""
    N, OH, OW, C = dp.shape
    g = _f64(dp) * pos
    win = torch.zeros(N, OH, OW, C, 4, dtype=torch.float64, device=dp.device)
    win.scatter_(-1, idx.to(torch.int64)[..., None], g[..., None])
    dz = win.view(N, OH, OW, C, 2, 2).permute(0, 1, 4, 2, 5, 3).reshape(N, 2 * OH, 2 * OW, C)
    return dz, g.sum((0, 1, 2)), g.abs().sum((0, 1, 2))


# ----------------------------------------------------- float64 references of the memory-bound kernels
# elementwise.cu and loss_optim.cu.  Where a kernel's fp32 arithmetic is at most one add and one
# multiply of fp32 operands, the reference reproduces its rounding points (``_r32``): float64 holds
# such a sum or product exactly (barring a 30-bit exponent gap in a sum), so rounding it once to fp32
# gives the kernel's value and the tests compare bit for bit.

def _r32(t: torch.Tensor) -> torch.Tensor:
    """Round float64 values to fp32 and back: one fp32 operation's result."""
    return t.to(torch.float32).to(torch.float64)


def _f32(x: float) -> float:
    """A Python scalar as the fp32 value the kernel receives."""
    return float(torch.tensor(x, dtype=torch.float32))


def _first_max(win: torch.Tensor):
    """(max, index of its first occurrence) over the last dimension."""
    val = win.amax(-1)
    pos = torch.arange(win.shape[-1], device=win.device)
    idx = torch.where(win == val[..., None], pos, win.shape[-1]).amin(-1)
    return val, idx


def maxpool2x2_64(x: torch.Tensor):
    """maxpool2x2_fwd on NHWC x: (pooled max [N,H/2,W/2,C], first maximum 0..3 in window order)."""
    return _first_max(pool_windows(_f64(x)))


def maxpool2x2_relu_bwd64(y: torch.Tensor, dp: torch.Tensor):
    """Backward of [ReLU -> maxpool2x2] from the stored post-ReLU map y: dp goes to the first maximum
    of each window whose maximum is > 0.  Returns (dz, column sum of dz, column sum of |dz|)."""
    val, idx = maxpool2x2_64(y)
    dz, cs, mag = unpool2x2_64(dp, idx, val > 0)
    H, W = y.shape[1], y.shape[2]
    if (H, W) != dz.shape[1:3]:         # floor mode: the odd last row / column gets dz = 0
        dz = F.pad(dz, (0, 0, 0, W - dz.shape[2], 0, H - dz.shape[1]))
    return dz, cs, mag


def _ap_windows(n_in: int, n_out: int):
    """torch's adaptive-pool windows: [floor(o*in/out), ceil((o+1)*in/out)) -- they overlap when in < out."""
    return [((o * n_in) // n_out, -(-((o + 1) * n_in) // n_out)) for o in range(n_out)]


def adaptive_avgpool64(x: torch.Tensor, OH: int, OW: int):
    """adaptive_avgpool_fwd on NHWC x -> (mean of each window [N,OH,OW,C], mean of |x|)."""
    N, H, W, C = x.shape
    x64 = _f64(x)
    ref = torch.zeros(N, OH, OW, C, dtype=torch.float64, device=x.device)
    mag = torch.zeros_like(ref)
    for oh, (h0, h1) in enumerate(_ap_windows(H, OH)):
        for ow, (w0, w1) in enumerate(_ap_windows(W, OW)):
            win = x64[:, h0:h1, w0:w1]
            ref[:, oh, ow] = win.mean((1, 2))
            mag[:, oh, ow] = win.abs().mean((1, 2))
    return ref, mag


def adaptive_avgpool_bwd64(dy: torch.Tensor, H: int, W: int):
    """adaptive_avgpool_bwd: every input pixel gets dy / (window size) of each window it lies in."""
    N, OH, OW, C = dy.shape
    dy64 = _f64(dy)
    ref = torch.zeros(N, H, W, C, dtype=torch.float64, device=dy.device)
    mag = torch.zeros_like(ref)
    for oh, (h0, h1) in enumerate(_ap_windows(H, OH)):
        for ow, (w0, w1) in enumerate(_ap_windows(W, OW)):
            g = dy64[:, oh, ow][:, None, None] / ((h1 - h0) * (w1 - w0))
            ref[:, h0:h1, w0:w1] += g
            mag[:, h0:h1, w0:w1] += g.abs()
    return ref, mag


def ap_max_window(n_in: int, n_out: int) -> int:
    """Largest window of adaptive pooling along one dimension."""
    return max(b - a for a, b in _ap_windows(n_in, n_out))


def ap_max_cover(n_in: int, n_out: int) -> int:
    """Most windows one input position lies in, along one dimension."""
    return max(sum(a <= i < b for a, b in _ap_windows(n_in, n_out)) for i in range(n_in))


def bias_grad64(dz: torch.Tensor, C: int, scale: float = 1.0, rows=None):
    """bias_grad / bias_grad_ld: scale * sum over rows of dz[:rows, :C] for a row stride ld >= C."""
    d = _f64(dz.reshape(dz.shape[0], -1)[:rows, :C])
    return scale * d.sum(0), abs(scale) * d.abs().sum(0)


# ---- Philox4x32-10 (Random123), vectorised over int64 tensors holding 32-bit words
_PHILOX_M = (0xD2511F53, 0xCD9E8D57)
_PHILOX_W = (0x9E3779B9, 0xBB67AE85)
_MASK32 = 0xFFFFFFFF


def _mulhilo(a: int, b: torch.Tensor):
    # 32 x 32 -> 64-bit product in int64 without overflow: split b into 16-bit halves
    lo16, hi16 = b & 0xFFFF, b >> 16
    p_lo = a * lo16                                   # < 2^48
    p_hi = a * hi16                                   # < 2^48
    lo = (p_lo + ((p_hi & 0xFFFF) << 16)) & _MASK32
    hi = ((p_hi + (p_lo >> 16)) >> 16) & _MASK32
    return hi, lo


def philox4x32_10(key, ctr):
    """Philox4x32-10 of 32-bit words (Python ints or int64 tensors): key (k0, k1), counter (c0..c3)
    -> the four output words, as int64 tensors."""
    k0, k1 = (torch.as_tensor(k, dtype=torch.int64) for k in key)
    c0, c1, c2, c3 = (torch.as_tensor(c, dtype=torch.int64) for c in ctr)
    for _ in range(10):
        hi0, lo0 = _mulhilo(_PHILOX_M[0], c0)
        hi1, lo1 = _mulhilo(_PHILOX_M[1], c2)
        c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
        k0, k1 = (k0 + _PHILOX_W[0]) & _MASK32, (k1 + _PHILOX_W[1]) & _MASK32
    return c0, c1, c2, c3


def dropout_mask64(seed: int, offset: int, B: int, N: int, p: float, device=None):
    """The dropout of fc_bias_act: (keep [B][N] bool, keep_scale).  Word j of Philox quad q, keyed by
    (seed lo, seed hi) with counter (q lo, q hi, offset lo, offset hi), decides element 4q + j of the
    flattened [B][N]: u = (word >> 8) * 2^-24 and the element is dropped iff u < fp32(p).
    keep_scale = fp32(1 / (1 - fp32(p)))."""
    total = B * N
    q = torch.arange((total + 3) // 4, dtype=torch.int64, device=device)
    words = philox4x32_10((seed & _MASK32, (seed >> 32) & _MASK32),
                          (q & _MASK32, q >> 32, offset & _MASK32, (offset >> 32) & _MASK32))
    r = torch.stack(words, dim=1).reshape(-1)[:total]
    u = (r >> 8).to(torch.float64) * 2.0 ** -24
    p32 = torch.tensor(p, dtype=torch.float32)
    one = torch.tensor(1.0, dtype=torch.float32)
    keep_scale = float(one / (one - p32)) if p > 0 else 1.0
    keep = ~(u < float(p32)) if p > 0 else torch.ones_like(u, dtype=torch.bool)
    return keep.view(B, N), keep_scale


def fc_bias_act64(acc: torch.Tensor, bias, *, relu: bool, drop_p: float = 0.0, seed: int = 0, offset: int = 0):
    """fc_bias_act on fp32 acc [B][N]: dropout(relu(acc + bias)) with the kernel's rounding points
    (fp32 add, fp32 multiply by keep_scale).  Returns (y [B][N], mag)."""
    B, N = acc.shape
    a = _f64(acc)
    b = _f64(bias).view(1, N) if bias is not None else torch.zeros(1, N, dtype=torch.float64, device=acc.device)
    v = _r32(a + b)
    mag = a.abs() + b.abs()
    if relu:
        v = torch.relu(v)
    if drop_p > 0:
        keep, ks = dropout_mask64(seed, offset, B, N, drop_p, device=acc.device)
        v = torch.where(keep, _r32(v * ks), torch.zeros_like(v))
        mag = mag * keep * ks
    return v, mag


def fc_grad_act64(acc: torch.Tensor, act, *, relu: bool, drop_p: float = 0.0):
    """fc_grad_act: dz = acc * [act > 0] * fp32(1 / (1 - p)), or acc unchanged without ReLU."""
    a = _f64(acc)
    if not relu:
        return a, a.abs()
    ks = dropout_mask64(0, 0, 1, 1, drop_p)[1]
    v = torch.where(act.to(torch.float64) > 0, _r32(a * ks), torch.zeros_like(a))
    return v, v.abs()


def _first_argmax(z: torch.Tensor) -> torch.Tensor:
    return _first_max(z)[1]


def cross_entropy64(logits: torch.Tensor, target: torch.Tensor, *, ldd: int = 0, class_weights=None,
                    grad_scale=None):
    """cross_entropy on fp32 logits [B][C] -> dict with
    loss: mean nll, or sum_i w_i nll_i / sum_i w_i with class weights;
    dlogits [B][ldd]: (softmax - onehot) * w_i / sum w (or * grad_scale, default 1/B), columns >= C zero;
    meter: (loss * B, count of first-maximum argmax == target, B)."""
    z = _f64(logits)
    B, C = z.shape
    t = target.to(torch.int64).view(-1)
    lse = torch.logsumexp(z, dim=1)
    nll = lse - z.gather(1, t.view(-1, 1)).view(-1)
    if class_weights is not None:
        w = _f64(class_weights)[t]
        norm = 1.0 / w.sum()
        loss = (w * nll).sum() * norm
    else:
        w = torch.ones(B, dtype=torch.float64, device=z.device)
        norm = _f32(1.0 / B if grad_scale is None else grad_scale)
        loss = nll.mean()
    dl = torch.zeros(B, max(ldd, C), dtype=torch.float64, device=z.device)
    dl[:, :C] = (torch.softmax(z, 1) - torch.nn.functional.one_hot(t, C).to(torch.float64)) * (w * norm)[:, None]
    correct = float((_first_argmax(z) == t).sum())
    meter = torch.tensor([float(loss) * B, correct, float(B)], dtype=torch.float64)
    return {"loss": loss, "dlogits": dl, "meter": meter}


def tta_reduce64(view_logits: torch.Tensor, target: torch.Tensor):
    """The --val-tta score of logits [V][B][C], one slice per view, in float64 -> dict with
    probs [B][C]: mean over the views of softmax(logits); loss: the batch mean of -log probs[y];
    meter: (loss * B, count of first-maximum argmax(probs) == target, B)."""
    z = _f64(view_logits)
    V, B, C = z.shape
    t = target.to(torch.int64).view(-1)
    probs = torch.softmax(z, 2).sum(0) / V
    loss = -torch.log(probs.gather(1, t.view(-1, 1))).mean()
    correct = float((_first_argmax(probs) == t).sum())
    meter = torch.tensor([float(loss) * B, correct, float(B)], dtype=torch.float64)
    return {"probs": probs, "loss": loss, "meter": meter}


def class_metrics(scores: torch.Tensor, target: torch.Tensor, views: int = 1):
    """The per-class evaluation counts of scores [B][C] (fp32 logits, or tta_accumulate's sums with ``views`` = V) ->
    (confusion int64 [C][C], rows labels and columns predictions; top-5 count).  A row's scores are the fp32 quotient
    s = scores / V, rounded to nearest as __fdiv_rn; its prediction is the first maximum, NaN never one; the label y
    ranks #{c : s_c > s_y} + #{c < y : s_c == s_y} and counts toward top-5 below 5.  A row without a maximum (every
    score NaN or -inf) or with a label outside [0, C) is counted nowhere."""
    s = scores.detach().to("cpu", torch.float32) / float(views)
    B, C = s.shape
    t = target.detach().to("cpu", torch.int64).view(-1)[:B]
    finite = torch.where(torch.isnan(s), torch.full_like(s, -float("inf")), s)
    best, pred = _first_max(finite)
    keep = (best > -float("inf")) & (t >= 0) & (t < C)
    s, t, pred = s[keep], t[keep], pred[keep]
    sy = s.gather(1, t.view(-1, 1))
    pos = torch.arange(C)
    rank = ((s > sy) | ((s == sy) & (pos < t.view(-1, 1)))).sum(1)
    confusion = torch.bincount(t * C + pred, minlength=C * C).view(C, C)
    return confusion, int((rank < 5).sum())


def kd_cross_entropy64(logits: torch.Tensor, teacher: torch.Tensor, target: torch.Tensor, *, alpha: float,
                       temperature: float, class_weights=None, label_smoothing: float = 0.0, soft_target=None,
                       ldd: int = 0):
    """The distillation loss in float64, in closed form -> dict with
    loss: (1 - alpha) CE + alpha T^2 sum_r KL(softmax(u_r / T) || softmax(z_r / T)) / B, where CE is
    F.cross_entropy(z, soft_target or target, weight=class_weights, label_smoothing=);
    dlogits [B][ldd]: (1 - alpha) dCE + alpha T (softmax(z / T) - softmax(u / T)) / B, columns >= C zero;
    meter: (loss * B, count of first-maximum argmax == target (or the soft target's first maximum), B)."""
    z, u = _f64(logits), _f64(teacher)
    B, C = z.shape
    t = target.to(torch.int64).view(-1)
    a, T = float(alpha), float(temperature)
    q = torch.nn.functional.one_hot(t, C).to(torch.float64) if soft_target is None else _f64(soft_target)
    cls = t if soft_target is None else _first_argmax(_f64(soft_target))
    q = q * (1.0 - label_smoothing) + label_smoothing / C
    norm = 1.0 / B
    if class_weights is not None:
        cw = _f64(class_weights)
        q = q * cw[None, :]
        if soft_target is None:          # integer targets: torch divides by the targets' weights
            norm = 1.0 / float(cw[t].sum())
    logp = torch.log_softmax(z, 1)
    ce = -(q * logp).sum() * norm
    dce = (torch.softmax(z, 1) * q.sum(1, keepdim=True) - q) * norm
    lps, lpt = torch.log_softmax(z / T, 1), torch.log_softmax(u / T, 1)
    kl = (lpt.exp() * (lpt - lps)).sum() / B
    loss = (1.0 - a) * ce + a * T * T * kl
    dl = torch.zeros(B, max(ldd, C), dtype=torch.float64, device=z.device)
    dl[:, :C] = (1.0 - a) * dce + a * T * (lps.exp() - lpt.exp()) / B
    correct = float((_first_argmax(z) == cls).sum())
    meter = torch.tensor([float(loss) * B, correct, float(B)], dtype=torch.float64)
    return {"loss": loss, "dlogits": dl, "meter": meter}


def head_ce64(h: torch.Tensor, W: torch.Tensor, bias: torch.Tensor, *, dl_used: torch.Tensor,
              drop_scale: float = 1.0, relu: bool = True):
    """head_ce's GEMM parts, each (ref, mag).  logits = h W^T + bias; the backward takes the dlogits
    the kernel rounded to bf16 (dl_used [B][C]), because that rounding point is part of the kernel:
    dW = dl^T h, db = sum_r dl, dh = (dl W) * [h > 0 if relu] * drop_scale.  The loss and dlogits are
    cross_entropy64 of the logits."""
    h64, W64, b64, dl = _f64(h), _f64(W), _f64(bias), _f64(dl_used)
    out = {"logits": (h64 @ W64.t() + b64, h64.abs() @ W64.abs().t() + b64.abs()),
           "dW": (dl.t() @ h64, dl.abs().t() @ h64.abs()),
           "db": (dl.sum(0), dl.abs().sum(0))}
    keep = (h64 > 0).to(torch.float64) if relu else torch.ones_like(h64)
    out["dh"] = ((dl @ W64) * keep * drop_scale, (dl.abs() @ W64.abs()) * keep * abs(drop_scale))
    return out


_U = 2.0 ** -24


def _sqrt_err(s, e_v):
    # |sqrt(a) - sqrt(b)| <= min(|a - b| / (2 sqrt(a)), sqrt(|a - b|))
    return torch.minimum(e_v / (2 * s).clamp_min(1e-300), e_v.sqrt())


def adam_step64(p, m, v, g, *, lr: float, beta1: float, beta2: float, eps: float, weight_decay: float,
                step: int, grad_scale: float = 1.0):
    """One step of adam_kernel (torch.optim.Adam with L2 weight decay, bias correction of step ``step``,
    the gradient scaled by grad_scale) from the given state.  Hyperparameters are taken as given: pass
    their fp32 values to compare with the kernel.  Returns {"p", "m", "v": (ref, err)}: err is a
    first-order running bound, in absolute units, of what the kernel's fp32 operations may add to
    each result (u per operation, the inputs taken as exact, the fp32 rounding of the bias
    corrections included)."""
    u = _U
    p, m, v, g = _f64(p), _f64(m), _f64(v), _f64(g)
    gs, wdp = g * grad_scale, weight_decay * p
    gk = gs + wdp
    e_gk = u * (gs.abs() + wdp.abs() + gk.abs())
    return _adam_moments_step64(p, torch.zeros_like(p), m, v, gk, e_gk, lr=lr, beta1=beta1, beta2=beta2, eps=eps,
                                step=step)


def _adam_moments_step64(p, e_p0, m, v, gk, e_gk, *, lr, beta1, beta2, eps, step):
    """The moments and step of adam_update (adam.cuh) from the gradient gk (error e_gk) and the weight p
    (error e_p0 that p carries in already)."""
    u = _U
    b1, b2 = beta1, beta2
    bc1i, bc2i = 1.0 / (1.0 - b1 ** step), 1.0 / (1.0 - b2 ** step) ** 0.5
    m1 = b1 * m + (1 - b1) * gk
    e_m = u * (b1 * m.abs() + m1.abs()) + (1 - b1) * (e_gk + u * gk.abs())
    t = (1 - b2) * gk
    e_t = (1 - b2) * e_gk + u * t.abs()
    t2 = t * gk
    e_t2 = gk.abs() * e_t + t.abs() * e_gk + u * t2.abs()
    v1 = b2 * v + t2
    e_v = u * (b2 * v.abs() + v1.abs()) + e_t2
    s = v1.sqrt()
    e_s = _sqrt_err(s, e_v) + u * s
    d = s * bc2i + eps
    e_d = bc2i * e_s + 3 * u * s * bc2i + u * d
    a = lr * bc1i
    num = a * m1
    e_num = a * e_m + 3 * u * num.abs()
    q = num / d
    e_q = e_num / d + num.abs() * e_d / d ** 2 + u * q.abs()
    p1 = p - q
    e_p = e_p0 + e_q + u * p1.abs()
    return {"p": (p1, e_p), "m": (m1, e_m), "v": (v1, e_v)}


def adamw_keep(lr: float, weight_decay):
    """AdamW's weight factor as the kernels take it: fp32(1 - lr * wd), the product in double (torch's
    Python scalar).  ``weight_decay`` may be a float64 tensor (one decay per element)."""
    if isinstance(weight_decay, torch.Tensor):
        return (1.0 - lr * weight_decay.to(torch.float64)).to(torch.float32).to(torch.float64)
    return _f32(1.0 - lr * weight_decay)


def adamw_step64(p, m, v, g, *, lr: float, beta1: float, beta2: float, eps: float, weight_decay,
                 step: int, grad_scale: float = 1.0, keep_lr: float = None):
    """One step of adam_kernel's decoupled form (torch.optim.AdamW): p' = p * keep with keep =
    adamw_keep(keep_lr or lr, weight_decay), then Adam on g * grad_scale with no L2 term.  ``lr`` is
    taken as given, like adam_step64's (pass the fp32 value the kernel receives); ``keep_lr`` is the
    double-precision rate the host forms keep from (default ``lr``).  ``weight_decay``: a float or a
    tensor of per-element decays.  Returns {"p", "m", "v": (ref, err)} as adam_step64; the error of
    keep itself is not counted: the kernel receives the same fp32 factor."""
    u = _U
    p, m, v, g = _f64(p), _f64(m), _f64(v), _f64(g)
    keep = adamw_keep(lr if keep_lr is None else keep_lr, weight_decay)
    p0 = p * keep
    gk = g * grad_scale
    return _adam_moments_step64(p0, u * p0.abs(), m, v, gk, u * gk.abs(), lr=lr, beta1=beta1, beta2=beta2,
                                eps=eps, step=step)


def sgd_step64(p, buf, g, *, lr: float, momentum: float, weight_decay: float, first: bool,
               grad_scale: float = 1.0):
    """One step of sgd_kernel (torch.optim.SGD with momentum, no dampening, L2 weight decay):
    d = g * grad_scale + wd * p; buf = d on the first step, else momentum * buf + d; p -= lr * buf.
    Returns {"p", "buf": (ref, err)} like adam_step64."""
    u = _U
    p, buf, g = _f64(p), _f64(buf), _f64(g)
    gs, wdp = g * grad_scale, weight_decay * p
    gk = gs + wdp
    e_gk = u * (gs.abs() + wdp.abs() + gk.abs())
    if first:
        b1, e_b = gk, e_gk
    else:
        mb = momentum * buf
        b1 = mb + gk
        e_b = u * (mb.abs() + b1.abs()) + e_gk
    q = lr * b1
    p1 = p - q
    e_p = lr * e_b + u * (q.abs() + p1.abs())
    return {"p": (p1, e_p), "buf": (b1, e_b)}


def ema_step64(ema, p, *, decay: float, first: bool):
    """One update of the weights' moving average as the optimizer kernels apply it from the new weights
    p: ema * d + p * a with d = fp32(decay), a = fp32(1 - decay) (1 - decay taken in double), or a copy
    of p on the first update.  Returns (ref, err) like adam_step64: two rounded products and one
    rounded sum."""
    u = _U
    e64, p64 = _f64(ema), _f64(p)
    if first:
        return p64, torch.zeros_like(p64)
    de, ap = _f32(decay) * e64, _f32(1.0 - decay) * p64
    r = de + ap
    return r, u * (de.abs() + ap.abs() + r.abs())


def nchw_to_nhwc64(x: torch.Tensor, cpad: int):
    """nchw_to_nhwc: fp32 NCHW -> NHWC with channels zero-padded to cpad (the kernel rounds to bf16)."""
    N, C, H, W = x.shape
    y = torch.zeros(N, H, W, cpad, dtype=torch.float64, device=x.device)
    y[..., :C] = _f64(x).permute(0, 2, 3, 1)
    return y, y.abs()


# ------------------------------------------------------------------ split-K without atomics
def splitk_reduce64(slices: torch.Tensor, dst=None, alpha: float = 1.0):
    """splitk_reduce in float64: (dst or 0) + alpha * sum over slices [splits, n].  Returns (ref, err)
    with err the fp32 rounding of the kernel's splits - 1 ordered adds, its product and its final add."""
    s64 = _f64(slices)
    tot = s64.sum(0)
    mag = s64.abs().sum(0)
    r = _f32(alpha) * tot
    err = _U * abs(_f32(alpha)) * mag * slices.shape[0]
    if dst is not None:
        r = r + _f64(dst)
        err = err + _U * r.abs()
    return r, err


def splitk_reduce_ordered(slices: torch.Tensor, dst=None, alpha: float = 1.0) -> torch.Tensor:
    """splitk_reduce bit for bit: fp32 adds in slice order, one rounded product by fp32(alpha), one
    rounded add onto dst.  (fp32 tensor arithmetic on the CPU rounds every operation: no FMA.)"""
    acc = slices[0].to("cpu", torch.float32).clone()
    for k in range(1, slices.shape[0]):
        acc = acc + slices[k].to("cpu", torch.float32)
    acc = acc * torch.tensor(alpha, dtype=torch.float32)
    if dst is not None:
        acc = dst.to("cpu", torch.float32) + acc
    return acc
