"""Python face of the native sm_90a kernels (csrc/*.cu -> distributed_vgg_f_b200/_C*.so).

The extension is built in-tree by ``build_native.py`` (``__graft_entry__.build()``).  On a machine
with a CUDA device the ops FAIL LOUDLY when the extension is missing -- there is no silent torch
fallback on the GPU path; ``ops.ref`` holds the torch reference implementations used as the
numerical oracle in the tests and as the CPU path.

Layout conventions: activations NHWC bf16; conv weights [Cout][3][3][Cin] bf16 (OHWI);
FC weights [out][in] bf16; gradients fp32.
"""
from __future__ import annotations

import importlib
from typing import Optional, Tuple

import torch

from ..config import DATA

_C = None
_IMPORT_ERROR: Optional[BaseException] = None
try:
    _C = importlib.import_module("distributed_vgg_f_b200._C")
except BaseException as e:           # noqa: BLE001 - keep the reason for the loud failure below
    _IMPORT_ERROR = e


def available() -> bool:
    return _C is not None


def require() -> "module":
    """Return the extension module or raise with build instructions."""
    if _C is None:
        raise RuntimeError(
            "distributed_vgg_f_b200._C (the sm_90a kernel library) is not built/importable: %r.\n"
            "Run `python build_native.py` (or __graft_entry__.build()) in the repo root. "
            "The GPU path has no torch fallback by design." % (_IMPORT_ERROR,))
    return _C


def launch_count() -> int:
    return int(require().launch_count())


# ----------------------------------------------------------------------------------- GEMM / conv
def gemm(a: torch.Tensor, b: torch.Tensor, out: torch.Tensor, *, M: int, N: int, K: int,
         a_mn: bool = False, b_mn: bool = False, epi: str = "f32_store", ldo: Optional[int] = None,
         bias: Optional[torch.Tensor] = None, alpha: float = 1.0, ksplit: int = 1, bn: int = 0) -> None:
    """out = alpha * A @ B^T on wgmma.  a_mn/b_mn: the operand is stored [K][M|N]."""
    C = require()
    code = {"f32_store": C.EPI_F32_STORE, "f32_atomic": C.EPI_F32_ATOMIC,
            "f32_atomic_t": C.EPI_F32_ATOMIC_T, "bf16_bias_relu": C.EPI_BF16_BIAS_RELU,
            "f32_store_t": C.EPI_F32_STORE_T, "bf16_store": C.EPI_BF16_STORE}[epi]
    if ldo is None:
        ldo = out.stride(0)
    C.gemm(a, a_mn, b, b_mn, M, N, K, out, ldo, code, bias, alpha, ksplit, bn)


def conv3x3_fprop(x, w, bias, relu: bool = True, bn: int = 0, out=None):
    N, H, W, _ = x.shape
    y = out if out is not None else torch.empty(N, H, W, w.shape[0], dtype=torch.bfloat16, device=x.device)
    require().conv_fprop(x, w, bias, y, relu, bn)
    return y


def pool_mask_like(n: int, h: int, w: int, c: int, device) -> torch.Tensor:
    """Mask buffer of conv3x3_fprop_pool for an un-pooled [n,h,w,c] activation."""
    return torch.zeros(n, h // 2, w // 2, c // 32, 4, dtype=torch.int32, device=device)


def conv3x3_fprop_pool(x, w, bias, bn: int = 0, out=None, mask=None):
    """maxpool2x2(relu(conv(x) + bias)) without materialising the un-pooled tensor (the engine's
    default for pooled layers; B200_FUSE_POOL=0 turns it off).
    Returns (pooled bf16 [N,H/2,W/2,Cout], mask int32 [N,H/2,W/2,Cout/32,4])."""
    N, H, W, _ = x.shape
    cout = w.shape[0]
    p = out if out is not None else torch.empty(N, H // 2, W // 2, cout, dtype=torch.bfloat16, device=x.device)
    m = mask if mask is not None else pool_mask_like(N, H, W, cout, x.device)
    require().conv_fprop_pool(x, w, bias, p, m, bn)
    return p, m


def unpool2x2(dp, mask, out=None, colsum=None):
    """Backward of the fused pool: route dp to the recorded argmax where the maximum was > 0."""
    N, OH, OW, Cc = dp.shape
    dz = out if out is not None else torch.empty(N, OH * 2, OW * 2, Cc, dtype=dp.dtype, device=dp.device)
    require().unpool2x2(dp, mask, dz, colsum)
    return dz


def conv3x3_dgrad(dz, w, cin: int, mask_src=None, bn: int = 0, out=None, colsum=None):
    """dx = conv_transpose(dz, w) [* (mask_src > 0)]; colsum (fp32 [cin]) += dx.sum(pixels)."""
    N, H, W, _ = dz.shape
    dx = out if out is not None else torch.empty(N, H, W, cin, dtype=torch.bfloat16, device=dz.device)
    require().conv_dgrad(dz, w, mask_src, dx, colsum, bn)
    return dx


def conv3x3_wgrad(dz, x, dw, scale: float = 1.0, ksplit: int = 0, bn: int = 0):
    """dw (fp32 [Cout][3][3][Cin]) += scale * dz^T (*) x -- accumulates, caller zeroes."""
    require().conv_wgrad(dz, x, dw, scale, ksplit, bn)
    return dw


# --------------------------------------------------------- split-K without atomics (--deterministic)
# Each function runs the PARTIAL form of a split-K kernel (every split stores its own slice of the
# workspace ``ws``, a flat fp32 tensor) and then ``splitk_reduce``, which adds the slices in split
# order: the result is a function of the operands alone, not of the order the CTAs finish in.
def splitk_reduce(ws, dst, n: int, splits: int, *, slice_elems: Optional[int] = None, alpha: float = 1.0,
                  accumulate: bool = False):
    """dst[:n] = (dst[:n] if accumulate else 0) + alpha * (((ws[0] + ws[1]) + ws[2]) + ...), slices
    ``slice_elems`` apart (default: n rounded up to whole float4s), each operation rounded to fp32."""
    C = require()
    C.splitk_reduce(ws, dst, n, C.workspace_slice(n) if slice_elems is None else slice_elems, splits, alpha,
                    accumulate)


def gemm_det(a, b, out, ws, *, M: int, N: int, K: int, a_mn: bool = False, b_mn: bool = False,
             transposed: bool = False, alpha: float = 1.0, ksplit: int = 1, bn: int = 0,
             accumulate: bool = False) -> int:
    """``gemm`` with epi f32_atomic (f32_atomic_t when ``transposed``) and split-K, reproducibly: ``out``
    is dense ([M][N], transposed [N][M]) and is overwritten unless ``accumulate``.  Returns the splits."""
    n = M * N
    splits = int(require().gemm_partial(a, a_mn, b, b_mn, M, N, K, ws, M if transposed else N, transposed, alpha,
                                        ksplit, bn))
    splitk_reduce(ws, out, n, splits, accumulate=accumulate)
    return splits


def conv3x3_wgrad_det(dz, x, dw, ws, scale: float = 1.0, accumulate: bool = False) -> int:
    """dw (fp32 [Cout][3][3][Cin]) = (dw if accumulate else 0) + scale * dz^T (*) x, reproducibly."""
    splits = int(require().conv_wgrad_partial(dz, x, ws, scale))
    splitk_reduce(ws, dw, dw.numel(), splits, accumulate=accumulate)
    return splits


def conv0_wgrad_det(dz, x4, dw0, ws, accumulate: bool = False) -> int:
    """Layer-0 weight gradient (``conv0_wgrad``), reproducibly."""
    splits = int(require().conv0_wgrad_partial(dz, x4, ws))
    splitk_reduce(ws, dw0, 64 * 64, splits, accumulate=accumulate)
    return splits


def colsum_det(dz2d, db, ws, rows: int, C: int, scale: float = 1.0, accumulate: bool = False) -> int:
    """db[:C] = (db if accumulate else 0) + scale * dz2d[:rows].sum(0) with C % 8 == 0: ``bias_grad``'s
    per-block sums stored as rows of ``ws`` and added in block order."""
    blocks = int(require().colsum_partial(dz2d, ws, rows, C, scale))
    splitk_reduce(ws, db, C, blocks, slice_elems=C, accumulate=accumulate)
    return blocks


# ---------------------------------------------------------------------------------- element-wise
def maxpool2x2(x, out=None):
    N, H, W, Cc = x.shape
    y = out if out is not None else torch.empty(N, H // 2, W // 2, Cc, dtype=x.dtype, device=x.device)
    require().maxpool_fwd(x, y)
    return y


def maxpool2x2_relu_bwd(y, dp, out=None, colsum=None):
    dz = out if out is not None else torch.empty_like(y)
    require().maxpool_relu_bwd(y, dp, dz, colsum)
    return dz


def adaptive_avgpool(x, oh: int, ow: int, out=None):
    N, _, _, Cc = x.shape
    y = out if out is not None else torch.empty(N, oh, ow, Cc, dtype=x.dtype, device=x.device)
    require().avgpool_fwd(x, y)
    return y


def adaptive_avgpool_bwd(dy, h: int, w: int, out=None):
    N, _, _, Cc = dy.shape
    dx = out if out is not None else torch.empty(N, h, w, Cc, dtype=dy.dtype, device=dy.device)
    require().avgpool_bwd(dy, dx)
    return dx


def bias_grad(dz2d, db, rows: int, C: int, ld: Optional[int] = None, scale: float = 1.0):
    require().bias_grad(dz2d, db, rows, C, ld if ld is not None else C, scale)
    return db


def fc_bias_act(acc, bias, y=None, y_f32=None, *, B: int, N: int, relu: bool, drop_p: float = 0.0,
                seed: int = 0, offset: int = 0, clear: bool = True):
    require().fc_bias_act(acc, bias, y, y_f32, B, N, relu, drop_p, seed, offset, clear)


def fc_grad_act(acc, act, dz, *, B: int, N: int, relu: bool, drop_p: float = 0.0, clear: bool = True):
    require().fc_grad_act(acc, act, dz, B, N, relu, drop_p, clear)


def cross_entropy(logits, target, dlogits=None, ldd: int = 0, meter=None, loss_out=None,
                  grad_scale: Optional[float] = None, class_weights=None, label_smoothing: float = 0.0,
                  mix=None):
    """Fused cross-entropy.  ``label_smoothing`` and ``mix`` (a ``data.transforms.MixDraw``: row r's
    target is lam e_{target[r]} + (1 - lam) e_{target[r-1 mod B]}) give F.cross_entropy's soft-target
    loss; without them the integer-label kernel runs."""
    if grad_scale is None:
        grad_scale = 1.0 / logits.shape[0]
    if label_smoothing == 0.0 and mix is None:
        require().cross_entropy(logits, target, dlogits, ldd or logits.shape[1], meter, loss_out,
                                grad_scale, class_weights)
        return
    require().cross_entropy_soft(logits, target, dlogits, ldd or logits.shape[1], meter, loss_out, grad_scale,
                                 class_weights, float(label_smoothing), mix.lam if mix is not None else 1.0,
                                 mix is not None)


def soft_targets(label_smoothing: float = 0.0, mix=None):
    """``head_ce``'s ``soft`` argument: None for integer labels without smoothing."""
    if label_smoothing == 0.0 and mix is None:
        return None
    return [float(label_smoothing), mix.lam if mix is not None else 1.0, 1.0 if mix is not None else 0.0]


def cross_entropy_kd(logits, target, teacher, *, alpha: float, temperature: float, dlogits=None, ldd: int = 0,
                     meter=None, loss_out=None, grad_scale: Optional[float] = None, class_weights=None,
                     label_smoothing: float = 0.0, mix=None):
    """``cross_entropy`` with knowledge distillation against fp32 ``teacher`` logits [B][C]: the loss is
    (1 - alpha) CE + alpha T^2 KL(softmax(teacher / T) || softmax(logits / T)) / B with CE the loss ``cross_entropy``
    computes (class weights, smoothing and mixing apply to it alone); meter and loss_out receive that loss."""
    if grad_scale is None:
        grad_scale = 1.0 / logits.shape[0]
    require().cross_entropy_kd(logits, target, dlogits, ldd or logits.shape[1], meter, loss_out, grad_scale,
                               class_weights, teacher, float(alpha), float(temperature),
                               soft_targets(label_smoothing, mix))


def _ema_args(ema, ema_decay: float, ema_first: bool) -> tuple:
    """Trailing arguments of the optimizer entries: none at all without a moving average."""
    return () if ema is None else (ema, float(ema_decay), bool(ema_first))


def wd_max_segments() -> int:
    """Weight-decay segments one optimizer launch can take (``wd_segments``)."""
    return int(require().wd_max_segments())


def _wd_args(wd_segments) -> tuple:
    """(starts, decays) of a segment table [(start, weight decay), ...], ordered as given."""
    return [int(s) for s, _ in wd_segments], [float(w) for _, w in wd_segments]


def adam_step(p, m, v, *, g32=None, g16=None, shadow=None, lr, beta1=0.9, beta2=0.999, eps=1e-8,
              weight_decay=0.0, step: int, grad_scale: float = 1.0, zero=None, ema=None, ema_decay: float = 0.0,
              ema_first: bool = False, decoupled: bool = False, wd_segments=None):
    """Fused Adam over a flat range.  ``ema`` (fp32, p's size): the same pass also updates the weights'
    moving average, ema = decay * ema + (1 - decay) * p_new, or ema = p_new with ``ema_first``.
    ``decoupled``: AdamW (torch.optim.AdamW: p *= 1 - lr * wd, then Adam without the L2 term).
    ``wd_segments`` [(start, wd), ...] (starts in elements of the range, the first 0, increasing,
    multiples of 4): a per-segment weight decay in the same launch, in place of ``weight_decay``."""
    args = (p, m, v, g32, g16, shadow, lr, beta1, beta2, eps, weight_decay, step, grad_scale, zero)
    if not decoupled and wd_segments is None:
        require().adam(*args, *_ema_args(ema, ema_decay, ema_first))
        return
    require().adam(*args, ema, float(ema_decay), bool(ema_first), bool(decoupled),
                   *_wd_args(wd_segments or ()))


def sgd_step(p, mom, *, g32=None, g16=None, shadow=None, lr, momentum=0.9, weight_decay=0.0,
             first: bool, grad_scale: float = 1.0, zero=None, ema=None, ema_decay: float = 0.0,
             ema_first: bool = False, wd_segments=None):
    """Fused SGD (momentum, L2 weight decay) over a flat range; ``ema`` and ``wd_segments`` as for
    ``adam_step``."""
    args = (p, mom, g32, g16, shadow, lr, momentum, weight_decay, first, grad_scale, zero)
    if wd_segments is None:
        require().sgd(*args, *_ema_args(ema, ema_decay, ema_first))
        return
    require().sgd(*args, ema, float(ema_decay), bool(ema_first), *_wd_args(wd_segments))


def layerwise_step(phase: int, kind: str, p, m, v=None, *, g32=None, g16=None, shadow=None, zero=None, ema=None,
                   ema_decay: float = 0.0, ema_first: bool = False, ws, ratio=None, lr: float, beta1: float = 0.9,
                   beta2: float = 0.999, eps: float = 1e-6, momentum: float = 0.0, step: int = 0, first: bool = False,
                   grad_scale: float = 1.0, segments, trust_coeff: float = 1e-3, trust_eps: float = 1e-8):
    """One launch of LAMB or LARS (``kind``), phase 1 or 2 (parallel/layerwise.py), over the flat range of ``p``.
    ``segments``: the launch's parallel.layerwise.Segment rows.  Phase 1 writes each CTA's partial sums into ``ws``;
    phase 2 reads them, writes each tensor's ratio into ``ratio`` (when given) and updates ``p`` (+ ``shadow``,
    ``ema``).  ``zero``: the gradient range to clear (LAMB: phase 1, LARS: phase 2)."""
    cols = [[s.start for s in segments], [s.ctas for s in segments], [s.slot for s in segments],
            [s.nslots for s in segments], [s.tensor for s in segments], [float(s.wd) for s in segments]]
    require().layerwise(int(phase), kind, p, m, v, g32, g16, shadow, zero, ema, ws, ratio, float(lr), float(beta1),
                        float(beta2), float(eps), float(momentum), int(step), bool(first), float(grad_scale),
                        float(ema_decay), bool(ema_first), *cols, float(trust_coeff), float(trust_eps))


def ema_update(p, ema, *, decay: float, first: bool = False):
    """ema = decay * ema + (1 - decay) * p (fp32, each operation rounded, no FMA), or ema = p with ``first``:
    the EMA update of ``adam_step`` / ``sgd_step`` for weights no optimizer launch covers (frozen layers)."""
    require().ema_update(p, ema, float(decay), bool(first))


# ---------------------------------------------------------------------------------------- PowerSGD
# One compressed tensor is an n x m row-major fp32 matrix (m % 4 == 0); P is [n][rank], Q is [m][rank].
def psgd_project(g, e, q, p, *, n: int, m: int, rank: int, scale: float = 1.0) -> None:
    """M = g * scale + e written over ``e``, and P = M Q into ``p``."""
    require().psgd_project(g, e, q, p, n, m, rank, float(scale))


def psgd_backproject(M, p, q, ws, *, n: int, m: int, rank: int) -> None:
    """Q = M^T P into ``q``; per-row-split partial sums go to ``ws`` and are added in split order."""
    require().psgd_backproject(M, p, q, ws, n, m, rank)


def psgd_workspace_elems(n: int, m: int, rank: int, sms: Optional[int] = None) -> int:
    C = require()
    return int(C.psgd_workspace_elems(n, m, rank, C.sm_count() if sms is None else sms))


def psgd_orthogonalize(x, *, rows: int, rank: int, count: int = 1) -> None:
    """Modified Gram-Schmidt of ``count`` consecutive [rows][rank] matrices in place; zero columns stay zero."""
    require().psgd_orthogonalize(x, rows, rank, count)


def psgd_decompress(p, q, g, e, *, n: int, m: int, rank: int, alpha: float = 1.0) -> None:
    """G = alpha P Q^T written over ``g``; e = M - G (``e`` holds M from psgd_project)."""
    require().psgd_decompress(p, q, g, e, n, m, rank, float(alpha))


_MIX_KIND = {"mixup": 1, "cutmix": 2}


def augment(src_u8, params, out, resized_hw: Tuple[int, int], out_hw: int = DATA.crop,
            mode: str = "im2col", pad: int = 64, mix=None):
    """uint8 [N,H,W,3] + params [N,8] -> normalised bf16 (NHWC padded, or layer-0 im2col rows).
    ``mix`` (a ``data.transforms.MixDraw``, NHWC only): MixUp / CutMix the batch in the same pass,
    sample i with sample i-1 mod N."""
    if mix is None:
        require().augment(src_u8, params, out, resized_hw[0], resized_hw[1], out_hw, out_hw,
                          1 if mode == "im2col" else 0, pad, list(DATA.mean), list(DATA.std))
        return out
    if mode != "nhwc":
        raise ValueError("augment: MixUp / CutMix are fused into the NHWC mode only")
    require().augment_mixed(src_u8, params, out, resized_hw[0], resized_hw[1], out_hw, out_hw, pad,
                            list(DATA.mean), list(DATA.std), _MIX_KIND[mix.kind], mix.lam, list(mix.box))
    return out


def augment_ragged(data_u8, geom, params, inter, out, geom_host, params_host, out_hw: int = DATA.crop,
                   mix=None):
    """Images of any sizes (data/loader.py::RaggedBatch on the device) -> normalised bf16 NHWC4
    ``out``, resampled as Pillow does.  ``geom_host`` / ``params_host``: the CPU tensors the device
    ``geom`` / ``params`` were copied from; ``inter`` holds ``ragged_inter_bytes(geom_host)``.
    ``mix``: as for ``augment``."""
    if mix is None:
        require().augment_ragged(data_u8, geom, params, inter, out, geom_host, params_host, out_hw, out_hw,
                                 list(DATA.mean), list(DATA.std))
        return out
    require().augment_ragged_mixed(data_u8, geom, params, inter, out, geom_host, params_host, out_hw, out_hw,
                                   list(DATA.mean), list(DATA.std), _MIX_KIND[mix.kind], mix.lam, list(mix.box))
    return out


def augment_view(src_u8, params, out, resized_hw: Tuple[int, int], view: int, out_hw: int = DATA.crop):
    """``augment`` (NHWC4) for one test-time augmentation view (``data.transforms.TTA_VIEWS``) of the resized image."""
    require().augment_view(src_u8, params, out, resized_hw[0], resized_hw[1], out_hw, out_hw, int(view),
                           list(DATA.mean), list(DATA.std))
    return out


def augment_ragged_view(data_u8, geom, params, inter, out, geom_host, params_host, view: int,
                        out_hw: int = DATA.crop, pass1=()):
    """``augment_ragged`` for one view.  ``pass1``: every view of the batch, to run the horizontal pass once for all
    of them first (its rows and columns are the union of what they read); empty: ``inter`` already holds it."""
    require().augment_ragged_view(data_u8, geom, params, inter, out, geom_host, params_host, out_hw, out_hw,
                                  list(DATA.mean), list(DATA.std), int(view), [int(v) for v in pass1])
    return out


def tta_accumulate(logits, target, acc, *, view: int, views: int, meter=None, loss_out=None) -> None:
    """Add view ``view`` of ``views`` to the view-mean reduction: acc[:B] = softmax(logits) at view 0, += at the
    later ones; the last view adds (sum of -log(acc[y] / V), count of argmax(acc / V) == y, B) into ``meter``."""
    require().tta_accumulate(logits, target, acc, meter, loss_out, int(view), int(views))


def class_metrics(scores, target, confusion, top5, *, views: int = 1) -> None:
    """Add one batch to the per-class evaluation counts: for each row of the fp32 ``scores`` [b][C] divided by ``views``
    (logits: 1; tta_accumulate's acc: V), confusion[y][first maximum] += 1 (int64 [C][C], rows labels) and, when the
    label ranks among the first five, top5 += 1 (``ref.class_metrics`` has the rule)."""
    require().class_metrics(scores, target, confusion, top5, int(views))


def ragged_inter_bytes(geom_host) -> int:
    """Bytes of the intermediate ``augment_ragged`` needs for these geometry rows."""
    return int(require().ragged_inter_bytes(geom_host))


def native_decode_pngs(paths, threads: int = 8):
    """Multi-threaded native PNG decode (csrc/png_decode.cpp) -> uint8 tensor [N,H,W,3], or None when
    a file is not a plain 8-bit PNG / sizes differ / the extension is absent (caller uses PIL)."""
    if _C is None or not hasattr(_C, "decode_pngs"):
        return None
    paths = list(paths)
    if not paths or not all(p.lower().endswith(".png") for p in paths):
        return None
    try:
        return _C.decode_pngs(paths, threads)
    except Exception:
        return None
