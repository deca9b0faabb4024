"""CPU reference of the streaming JPEG decode (csrc/jpeg.cu): quantised coefficients -> RGB, bit for bit
what Pillow's libjpeg(-turbo) gives for ``Image.open(f).convert("RGB")``.

The arithmetic is libjpeg's: the ``JDCT_ISLOW`` integer IDCT (``jidctint.c``) with its range-limit table,
"fancy" triangle upsampling of 1x1 chroma under 2x1 / 2x2 luma (``jdsample.c``; components at most two
samples wide are replicated instead), edges that repeat the last real sample, and the 16-bit fixed-point
YCbCr -> RGB tables of ``jdcolor.c``.  It is ``JpegBatch.to_float``'s decoder and the tests' oracle.

A batch (``JpegBatch``) carries, per image, one int32 descriptor row (``csrc/include/jpeg.h``):
``[ncomp, hmax, vmax, first block, raw offset, bw0..2, bh0..2, quant row 0..2, 0, 0]``.
"""
from __future__ import annotations

import numpy as np

DESC_DIM = 16

_CONST_BITS, _PASS1_BITS = 13, 2
_F = {k: int(v * (1 << _CONST_BITS) + 0.5) for k, v in dict(
    c0298=0.298631336, c0390=0.390180644, c0541=0.541196100, c0765=0.765366865, c0899=0.899976223,
    c1175=1.175875602, c1501=1.501321110, c1847=1.847759065, c1961=1.961570560, c2053=2.053119869,
    c2562=2.562915447, c3072=3.072711026).items()}


def _idct_1d(x, shift):
    """One jidctint pass along the last axis of int64 ``x`` [..., 8]; returns the 8 outputs descaled by ``shift``
    (rounded as libjpeg's DESCALE)."""
    F = _F
    z2, z3 = x[..., 2], x[..., 6]
    z1 = (z2 + z3) * F["c0541"]
    tmp2 = z1 - z3 * F["c1847"]
    tmp3 = z1 + z2 * F["c0765"]
    tmp0 = (x[..., 0] + x[..., 4]) << _CONST_BITS
    tmp1 = (x[..., 0] - x[..., 4]) << _CONST_BITS
    tmp10, tmp13, tmp11, tmp12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    t0, t1, t2, t3 = x[..., 7], x[..., 5], x[..., 3], x[..., 1]
    z1, z2, z3, z4 = t0 + t3, t1 + t2, t0 + t2, t1 + t3
    z5 = (z3 + z4) * F["c1175"]
    t0, t1, t2, t3 = t0 * F["c0298"], t1 * F["c2053"], t2 * F["c3072"], t3 * F["c1501"]
    z1, z2 = z1 * -F["c0899"], z2 * -F["c2562"]
    z3, z4 = z3 * -F["c1961"] + z5, z4 * -F["c0390"] + z5
    t0, t1, t2, t3 = t0 + z1 + z3, t1 + z2 + z4, t2 + z2 + z3, t3 + z1 + z4
    r = 1 << (shift - 1)
    out = [tmp10 + t3, tmp11 + t2, tmp12 + t1, tmp13 + t0, tmp13 - t0, tmp12 - t1, tmp11 - t2, tmp10 - t3]
    return np.stack([(o + r) >> shift for o in out], axis=-1)


def _range_limit(x):
    """libjpeg's post-IDCT range-limit table indexed with ``x & 1023`` (x: the descaled sample before +128)."""
    t = x & 1023
    return np.where(t < 128, t + 128, np.where(t < 512, 255, np.where(t < 896, 0, t - 896))).astype(np.uint8)


def idct_islow(coef: np.ndarray, quant: np.ndarray) -> np.ndarray:
    """Blocks of quantised coefficients [n, 64] (natural order) and their tables [n, 64] -> samples uint8 [n, 8, 8]."""
    x = (coef.astype(np.int64) * quant.astype(np.int64)).reshape(-1, 8, 8)
    ws = _idct_1d(x.transpose(0, 2, 1), _CONST_BITS - _PASS1_BITS).transpose(0, 2, 1)    # columns
    return _range_limit(_idct_1d(ws, _CONST_BITS + _PASS1_BITS + 3))                       # rows


def _plane(samples: np.ndarray, bw: int, bh: int) -> np.ndarray:
    """Blocks [bw*bh, 8, 8] of one component, row by row -> the component's sample plane [8 bh, 8 bw]."""
    return samples.reshape(bh, bw, 8, 8).transpose(0, 2, 1, 3).reshape(bh * 8, bw * 8)


def _upsample(c: np.ndarray, H: int, W: int, hmax: int, vmax: int) -> np.ndarray:
    """Chroma plane (its real ceil(W/hmax) x ceil(H/vmax) part) -> H x W, as libjpeg's h2v1 / h2v2 upsamplers."""
    cw, ch = -(-W // hmax), -(-H // vmax)
    c = c[:ch, :cw].astype(np.int32)
    if hmax == 1:
        return c
    if cw <= 2:                                     # jdsample.c: no fancy upsampling this narrow
        return np.repeat(np.repeat(c, 2, axis=1), vmax, axis=0)[:H, :W]
    if vmax == 1:
        prev = np.concatenate([c[:, :1], c[:, :-1]], axis=1)
        nxt = np.concatenate([c[:, 1:], c[:, -1:]], axis=1)
        even = (3 * c + prev + 1) >> 2
        odd = (3 * c + nxt + 2) >> 2
        even[:, 0] = c[:, 0]
        odd[:, -1] = c[:, -1]
        out = np.stack([even, odd], axis=2).reshape(ch, 2 * cw)
        return out[:, :W]
    up = np.concatenate([c[:1], c[:-1]], axis=0)    # the row above (first row: itself)
    dn = np.concatenate([c[1:], c[-1:]], axis=0)    # the row below (last real row: itself)
    rows = np.stack([3 * c + up, 3 * c + dn], axis=1).reshape(2 * ch, cw)
    prev = np.concatenate([rows[:, :1], rows[:, :-1]], axis=1)
    nxt = np.concatenate([rows[:, 1:], rows[:, -1:]], axis=1)
    even = (3 * rows + prev + 8) >> 4
    odd = (3 * rows + nxt + 7) >> 4
    even[:, 0] = (rows[:, 0] * 4 + 8) >> 4
    odd[:, -1] = (rows[:, -1] * 4 + 7) >> 4
    out = np.stack([even, odd], axis=2).reshape(2 * ch, 2 * cw)
    return out[:H, :W]


def _ycc_to_rgb(y, cb, cr) -> np.ndarray:
    """jdcolor.c's ycc_rgb_convert: 16-bit fixed-point tables, results clamped to [0, 255]."""
    y, cb, cr = (a.astype(np.int64) for a in (y, cb, cr))
    cb, cr = cb - 128, cr - 128
    r = y + ((91881 * cr + 32768) >> 16)
    g = y + ((-22554 * cb + 32768 - 46802 * cr) >> 16)
    b = y + ((116130 * cb + 32768) >> 16)
    return np.clip(np.stack([r, g, b], axis=-1), 0, 255).astype(np.uint8)


def decode_image(desc: np.ndarray, H: int, W: int, coef: np.ndarray, quant: np.ndarray,
                 raw: np.ndarray) -> np.ndarray:
    """One image of a batch -> uint8 [H, W, 3].  ``coef``: the batch's int16 [blocks, 64]; ``quant``: its int32
    [rows, 64] tables; ``raw``: its uint8 raw-RGB bytes."""
    d = [int(v) for v in desc]
    n = d[0]
    if n == 0:
        return raw[d[4]:d[4] + H * W * 3].reshape(H, W, 3).copy()
    at, planes = d[3], []
    for c in range(n):
        bw, bh, q = d[5 + c], d[8 + c], d[11 + c]
        blocks = coef[at:at + bw * bh]
        at += bw * bh
        planes.append(_plane(idct_islow(blocks, np.broadcast_to(quant[q], blocks.shape)), bw, bh))
    if n == 1:
        return np.repeat(planes[0][:H, :W, None], 3, axis=2)
    hmax, vmax = d[1], d[2]
    return _ycc_to_rgb(planes[0][:H, :W], _upsample(planes[1], H, W, hmax, vmax),
                       _upsample(planes[2], H, W, hmax, vmax))


def decode_batch(coef, quant, raw, desc, geom) -> np.ndarray:
    """Every image of a batch at its ``geom`` offset, back to back: the flat uint8 RGB buffer a ``RaggedBatch``
    would carry."""
    coef = np.asarray(coef).reshape(-1, 64)
    quant = np.asarray(quant).reshape(-1, 64)
    raw, desc, geom = np.asarray(raw), np.asarray(desc), np.asarray(geom)
    k = geom.shape[0]
    out = np.empty(int(geom[k - 1, 0] + geom[k - 1, 1] * geom[k - 1, 2] * 3), dtype=np.uint8)
    for i in range(k):
        off, H, W = (int(v) for v in geom[i, :3])
        out[off:off + H * W * 3] = decode_image(desc[i], H, W, coef, quant, raw).reshape(-1)
    return out
