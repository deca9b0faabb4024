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
                  override: dict = None):
    """Forward + backward of the network on fp32 torch ops with the engine's rounding points.

    state: torch-layout fp32 tensors (weights are rounded to bf16 here, biases stay fp32).
    Returns (logits, mean loss, grads in torch layout).  Dropout is treated as identity.

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
    loss = -logp.gather(1, target.view(-1, 1)).mean()
    dz = rb((torch.softmax(logits, 1) - F.one_hot(target, logits.shape[1]).float()) / B)

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
    """[N,H,W,C] -> [N,H/2,W/2,C,4]: the 2x2 windows in the order (0,0), (0,1), (1,0), (1,1)."""
    N, H, W, C = t.shape
    v = t.reshape(N, H // 2, 2, W // 2, 2, C)
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
