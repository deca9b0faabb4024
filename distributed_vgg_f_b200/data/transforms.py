"""Input transforms as *parameters + one fused sampling op*.

Reference pipelines (distributedVggf.py:88-95 train, :103-108 val), all on PIL images in the
training process:
  train: RandomResizedCrop(256, scale=(.8,1)) -> RandomRotation(10) -> RandomHorizontalFlip ->
         CenterCrop(224) -> ToTensor -> Normalize(ImageNet mean/std)
  val:   Resize(256) -> CenterCrop(224) -> ToTensor -> Normalize
Every stage is a coordinate map, so the whole chain collapses into "for each of the 224x224 output
pixels: undo centre-crop, undo flip, undo rotation (nearest, zero fill), bilinear-sample the crop
box of the source".  We draw the random parameters on the host with torchvision's exact
distributions (``sample_train_params``) and evaluate the chain in one pass:
``augment_reference`` (torch ops; CPU path and oracle) and ``ops.augment`` (sm_90a kernel that
reads uint8 HWC and writes normalised bf16 NHWC / the layer-0 im2col matrix directly).
``reference_transforms`` returns the literal torchvision pipeline for bit-level parity runs.
"""
from __future__ import annotations

import math
from typing import NamedTuple, Optional, Tuple

import torch

from ..config import DATA

# params row: [top, left, crop_h, crop_w, cos(theta), sin(theta), flip, _]
PARAM_DIM = 8


def sample_train_params(n: int, src_h: int, src_w: int,
                        generator: Optional[torch.Generator] = None,
                        scale=DATA.crop_scale, ratio=DATA.crop_ratio,
                        degrees: float = DATA.rotation_deg) -> torch.Tensor:
    """Random crop box / angle / flip per sample, distributed as torchvision's get_params.

    Vectorised over the batch (the loader thread must keep up with ~8k images/s per GPU):
    RandomResizedCrop's "up to 10 attempts, else centre crop" becomes a first-valid-attempt select.
    """
    out = torch.zeros(n, PARAM_DIM, dtype=torch.float32)
    area = float(src_h * src_w)
    log_lo, log_hi = math.log(ratio[0]), math.log(ratio[1])
    u = torch.rand(n, 10, 2, generator=generator, dtype=torch.float64)
    pos = torch.rand(n, 2, generator=generator, dtype=torch.float64)
    misc = torch.rand(n, 2, generator=generator, dtype=torch.float64)
    target_area = area * (scale[0] + (scale[1] - scale[0]) * u[..., 0])
    aspect = torch.exp(log_lo + (log_hi - log_lo) * u[..., 1])
    w = torch.round(torch.sqrt(target_area * aspect))                     # [n, 10]
    h = torch.round(torch.sqrt(target_area / aspect))
    ok = (w > 0) & (w <= src_w) & (h > 0) & (h <= src_h)
    first = torch.argmax(ok.to(torch.int8), dim=1)                        # first valid attempt
    any_ok = ok.any(dim=1)
    rows = torch.arange(n)
    cw, ch = w[rows, first], h[rows, first]
    # torchvision's centre-crop fallback when all 10 attempts fail
    in_ratio = src_w / src_h
    if in_ratio < min(ratio):
        fw, fh = float(src_w), float(round(src_w / min(ratio)))
    elif in_ratio > max(ratio):
        fh, fw = float(src_h), float(round(src_h * max(ratio)))
    else:
        fw, fh = float(src_w), float(src_h)
    cw = torch.where(any_ok, cw, torch.full_like(cw, fw))
    ch = torch.where(any_ok, ch, torch.full_like(ch, fh))
    top = torch.minimum(torch.floor(pos[:, 0] * (src_h - ch + 1)), src_h - ch)
    left = torch.minimum(torch.floor(pos[:, 1] * (src_w - cw + 1)), src_w - cw)
    top = torch.where(any_ok, top, torch.floor((src_h - ch) / 2))
    left = torch.where(any_ok, left, torch.floor((src_w - cw) / 2))
    theta = torch.deg2rad(-degrees + 2.0 * degrees * misc[:, 0])
    out[:, 0], out[:, 1], out[:, 2], out[:, 3] = top.float(), left.float(), ch.float(), cw.float()
    out[:, 4], out[:, 5] = torch.cos(theta).float(), torch.sin(theta).float()
    out[:, 6] = (misc[:, 1] < 0.5).float()
    return out


def val_params(n: int, src_h: int, src_w: int) -> torch.Tensor:
    out = torch.zeros(n, PARAM_DIM, dtype=torch.float32)
    out[:, 2], out[:, 3], out[:, 4] = src_h, src_w, 1.0
    return out


def resized_dims(train: bool, src_h: int, src_w: int, resize: int = DATA.resize) -> Tuple[int, int]:
    """Size of the intermediate 'resized' image: 256x256 for train, shorter-side-256 for val."""
    if train:
        return resize, resize
    if src_h <= src_w:
        return resize, max(int(resize * src_w / src_h), 1)
    return max(int(resize * src_h / src_w), 1), resize


# ------------------------------------------------------------------- test-time augmentation views
# --val-tta: the views of an evaluation image, each an out_hw x out_hw crop of the Resize(R') image.  A view code
# is a position (torchvision's five_crop order, then the centre crop's mirror image) or'ed with TTA_FLIP to take
# the crop from the image's horizontal mirror; csrc/include/api.h (TtaPosition) uses the same codes.
TTA_TOP_LEFT, TTA_TOP_RIGHT, TTA_BOTTOM_LEFT, TTA_BOTTOM_RIGHT, TTA_CENTRE, TTA_CENTRE_MIRROR = range(6)
TTA_FLIP = 8
_FIVE = (TTA_TOP_LEFT, TTA_TOP_RIGHT, TTA_BOTTOM_LEFT, TTA_BOTTOM_RIGHT, TTA_CENTRE)
TTA_VIEWS = {
    "none": (TTA_CENTRE,),
    # the centre crop and its mirror image: hflip(center_crop(img)) is the crop of hflip(img) at the mirrored origin
    "flip": (TTA_CENTRE, TTA_CENTRE_MIRROR | TTA_FLIP),
    "five-crop": _FIVE,                                      # torchvision's five_crop
    "ten-crop": _FIVE + tuple(v | TTA_FLIP for v in _FIVE),  # ten_crop(vertical_flip=False)
}
TTA_MODES = tuple(TTA_VIEWS)


def tta_views(mode: str) -> Tuple[int, ...]:
    """The view codes of a --val-tta mode, in the order their probabilities are added."""
    if mode not in TTA_VIEWS:
        raise ValueError("val_tta must be one of %s (got %r)" % (", ".join(TTA_MODES), mode))
    return TTA_VIEWS[mode]


def view_origin(view: int, RH: int, RW: int, OH: int, OW: int) -> Tuple[int, int, bool]:
    """(top, left, mirrored) of view ``view``'s OH x OW crop of an RH x RW image; centre origins round half to
    even, as torchvision's center_crop."""
    pos = view & ~TTA_FLIP
    if not 0 <= pos <= TTA_CENTRE_MIRROR or view < 0:
        raise ValueError("bad view code %r" % view)
    if OH > RH or OW > RW:
        raise ValueError("a %d x %d view does not fit a %d x %d image" % (OH, OW, RH, RW))
    cy, cx = int(round((RH - OH) / 2.0)), int(round((RW - OW) / 2.0))
    y0 = {TTA_TOP_LEFT: 0, TTA_TOP_RIGHT: 0, TTA_BOTTOM_LEFT: RH - OH, TTA_BOTTOM_RIGHT: RH - OH}.get(pos, cy)
    x0 = {TTA_TOP_LEFT: 0, TTA_BOTTOM_LEFT: 0, TTA_TOP_RIGHT: RW - OW, TTA_BOTTOM_RIGHT: RW - OW,
          TTA_CENTRE_MIRROR: RW - OW - cx}.get(pos, cx)
    return y0, x0, bool(view & TTA_FLIP)


def augment_reference(src: torch.Tensor, params: torch.Tensor, resized_hw: Tuple[int, int],
                      out_hw: int = DATA.crop, mean=DATA.mean, std=DATA.std, view: Optional[int] = None) -> torch.Tensor:
    """Torch evaluation of the fused transform.  src: uint8 [n,H,W,3] -> float32 [n,3,out,out].
    ``view`` (a TTA view code): that view's crop instead of the centre crop, its flip combined with each
    sample's flip bit."""
    n, H, W, _ = src.shape
    RH, RW = resized_hw
    dev = src.device
    p = params.to(dev, torch.float32)
    ys, xs = torch.meshgrid(torch.arange(out_hw, device=dev, dtype=torch.float32),
                            torch.arange(out_hw, device=dev, dtype=torch.float32), indexing="ij")
    # undo CenterCrop(out_hw) on the RH x RW image (torchvision rounds the offset)
    off_y = int(round((RH - out_hw) / 2.0))
    off_x = int(round((RW - out_hw) / 2.0))
    vflip = False
    if view is not None:
        off_y, off_x, vflip = view_origin(view, RH, RW, out_hw, out_hw)
    ay = (ys + off_y).expand(n, -1, -1)
    ax = (xs + off_x).expand(n, -1, -1)
    flip = (p[:, 6].view(n, 1, 1) > 0.5) != vflip
    bx = torch.where(flip, (RW - 1) - ax, ax)
    by = ay
    # undo rotation: PIL affine, output pixel centre -> input coordinate, nearest = floor
    c, s = p[:, 4].view(n, 1, 1), p[:, 5].view(n, 1, 1)
    cx, cy = RW / 2.0, RH / 2.0
    dx, dy = bx + 0.5 - cx, by + 0.5 - cy
    rx = torch.floor(c * dx - s * dy + cx)
    ry = torch.floor(s * dx + c * dy + cy)
    inside = (rx >= 0) & (rx < RW) & (ry >= 0) & (ry < RH)
    # bilinear sample of the crop box (clamped to the box == resize of the cropped image)
    top, left = p[:, 0].view(n, 1, 1), p[:, 1].view(n, 1, 1)
    ch, cw = p[:, 2].view(n, 1, 1), p[:, 3].view(n, 1, 1)
    sy = (ry + 0.5) * (ch / RH) - 0.5
    sx = (rx + 0.5) * (cw / RW) - 0.5
    sy = torch.minimum(torch.clamp(sy, min=0.0), ch - 1)
    sx = torch.minimum(torch.clamp(sx, min=0.0), cw - 1)
    y0, x0 = torch.floor(sy), torch.floor(sx)
    wy, wx = (sy - y0), (sx - x0)
    y1 = torch.minimum(y0 + 1, ch - 1)
    x1 = torch.minimum(x0 + 1, cw - 1)
    srcf = src.to(torch.float32)
    bidx = torch.arange(n, device=dev).view(n, 1, 1).expand(-1, out_hw, out_hw)

    def g(yy, xx):
        return srcf[bidx, (yy + top).long().clamp_(0, H - 1), (xx + left).long().clamp_(0, W - 1)]

    wy, wx = wy.unsqueeze(-1), wx.unsqueeze(-1)
    val = (g(y0, x0) * (1 - wy) * (1 - wx) + g(y0, x1) * (1 - wy) * wx +
           g(y1, x0) * wy * (1 - wx) + g(y1, x1) * wy * wx)
    val = torch.where(inside.unsqueeze(-1), val, torch.zeros_like(val)) / 255.0
    m = torch.tensor(mean, device=dev).view(1, 1, 1, 3)
    sd = torch.tensor(std, device=dev).view(1, 1, 1, 3)
    return ((val - m) / sd).permute(0, 3, 1, 2).contiguous()


# ------------------------------------------------------------------------------ ragged (any size)
# Pillow's 8-bit resampler (libImaging/Resample.c) keeps 22 fractional bits in its fixed-point weights.
PIL_PRECISION_BITS = 22
# geometry row of a ragged batch: [byte offset into the batch's flat uint8 buffer, H, W, RH, RW]
GEOM_DIM = 5


def _pil_bilinear_coeffs(in_size: int, out_size: int):
    """Pillow's BILINEAR coefficients for one axis: (lo [out], k int64 [out, taps]) with k = 0 past
    each row's window.  Every operation is the fp64 one of precompute_coeffs / normalize_coeffs_8bpc."""
    import numpy as np

    scale = in_size / out_size
    fs = max(scale, 1.0)
    support, ss = fs, 1.0 / fs
    taps = int(math.ceil(support)) * 2 + 1
    lo = np.zeros(out_size, np.int64)
    k = np.zeros((out_size, taps), np.int64)
    for i in range(out_size):
        center = (i + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), in_size) - xmin
        w = [max(0.0, 1.0 - abs((x + xmin - center + 0.5) * ss)) for x in range(xmax)]
        ww = 0.0
        for v in w:
            ww += v
        for x, v in enumerate(w):
            v = v / ww if ww != 0.0 else v
            k[i, x] = int(-0.5 + v * (1 << PIL_PRECISION_BITS)) if v < 0 else int(0.5 + v * (1 << PIL_PRECISION_BITS))
        lo[i] = xmin
    return lo, k


def pil_resize_reference(img_u8, out_h: int, out_w: int):
    """``Image.fromarray(img).resize((out_w, out_h), Image.BILINEAR)`` bit for bit, for uint8 HWC RGB:
    the horizontal pass first, rounded to uint8, then the vertical pass; an unchanged axis is skipped.
    Accepts and returns a numpy array (a torch tensor in gives a torch tensor out)."""
    import numpy as np

    as_torch = isinstance(img_u8, torch.Tensor)
    src = (img_u8.numpy() if as_torch else np.asarray(img_u8)).astype(np.int64)
    half, shift = 1 << (PIL_PRECISION_BITS - 1), PIL_PRECISION_BITS
    H, W = src.shape[:2]
    if out_w != W:
        lo, k = _pil_bilinear_coeffs(W, out_w)
        idx = np.minimum(lo[:, None] + np.arange(k.shape[1])[None, :], W - 1)       # k = 0 past the window
        src = np.clip((half + (src[:, idx, :] * k[None, :, :, None]).sum(2)) >> shift, 0, 255)
    if out_h != H:
        lo, k = _pil_bilinear_coeffs(H, out_h)
        idx = np.minimum(lo[:, None] + np.arange(k.shape[1])[None, :], H - 1)
        src = np.clip((half + (src[idx, :, :] * k[:, :, None, None]).sum(1)) >> shift, 0, 255)
    out = src.astype(np.uint8)
    return torch.from_numpy(out) if as_torch else out


def ragged_geometry(hw, train: bool, resize: int = DATA.resize) -> torch.Tensor:
    """Geometry rows [k, GEOM_DIM] of images of sizes ``hw`` ([k, 2]) gathered back to back."""
    g = torch.zeros(len(hw), GEOM_DIM, dtype=torch.int64)
    off = 0
    for i, (h, w) in enumerate(hw):
        h, w = int(h), int(w)
        g[i, 0], g[i, 1], g[i, 2] = off, h, w
        g[i, 3], g[i, 4] = resized_dims(train, h, w, resize)
        off += h * w * 3
    return g


def ragged_reference(data_u8: torch.Tensor, geom: torch.Tensor, params: torch.Tensor,
                     out_hw: int = DATA.crop, mean=DATA.mean, std=DATA.std, view: Optional[int] = None) -> torch.Tensor:
    """The reference chain for images of any size, with Pillow's resampling.  data_u8: the flat uint8
    buffer the geometry rows point into; params rows as ``sample_train_params`` / ``val_params``.
    Per image: crop box -> Pillow BILINEAR resize to (RH, RW) -> nearest rotation with zero fill ->
    flip -> centre crop -> normalise (float32, as ToTensor + Normalize).  Val rows (box = the whole
    image, no rotation, no flip) are Resize + CenterCrop.  -> float32 [k, 3, out_hw, out_hw].
    ``view``: as for ``augment_reference``."""
    n = int(geom.shape[0])
    data = data_u8.cpu()
    out = torch.empty(n, 3, out_hw, out_hw, dtype=torch.float32)
    ys, xs = torch.meshgrid(torch.arange(out_hw, dtype=torch.float32),
                            torch.arange(out_hw, dtype=torch.float32), indexing="ij")
    m = torch.tensor(mean, dtype=torch.float32).view(3, 1, 1)
    sd = torch.tensor(std, dtype=torch.float32).view(3, 1, 1)
    for i in range(n):
        off, H, W, RH, RW = [int(v) for v in geom[i]]
        p = params[i].to(torch.float32)
        top, left, ch, cw = [int(v) for v in p[:4]]
        img = data[off:off + H * W * 3].view(H, W, 3)[top:top + ch, left:left + cw]
        res = pil_resize_reference(img.contiguous(), RH, RW)                       # uint8 [RH, RW, 3]
        # the coordinate chain of augment_reference, evaluated in the same float32 operations
        y0, x0, vflip = int(round((RH - out_hw) / 2.0)), int(round((RW - out_hw) / 2.0)), False
        if view is not None:
            y0, x0, vflip = view_origin(view, RH, RW, out_hw, out_hw)
        ay = ys + y0
        ax = xs + x0
        bx = (RW - 1) - ax if (float(p[6]) > 0.5) != vflip else ax
        dx, dy = bx + 0.5 - RW / 2.0, ay + 0.5 - RH / 2.0
        rx = torch.floor(p[4] * dx - p[5] * dy + RW / 2.0)
        ry = torch.floor(p[5] * dx + p[4] * dy + RH / 2.0)
        inside = (rx >= 0) & (rx < RW) & (ry >= 0) & (ry < RH)
        v = res[ry.long().clamp(0, RH - 1), rx.long().clamp(0, RW - 1)].permute(2, 0, 1).to(torch.float32)
        v = torch.where(inside.unsqueeze(0), v, torch.zeros_like(v))
        out[i] = (v / 255.0 - m) / sd
    return out


# ------------------------------------------------------------------------ MixUp / CutMix (per batch)
class MixDraw(NamedTuple):
    """One training batch's MixUp or CutMix draw.  Sample i is mixed with sample (i-1) mod b, where b
    is the batch's actual size (torchvision's ``roll(1, 0)``)."""
    kind: str                           # "mixup" | "cutmix"
    lam: float                          # weight of sample i: MixUp's lam, CutMix's lam_adjusted
    box: Tuple[int, int, int, int]      # CutMix: (x1, y1, x2, y2) in network-input pixels; MixUp: zeros


def mix_seed(seed: int, epoch: int, rank: int, index: int) -> int:
    """Seed of the draw of training batch ``index`` of ``epoch`` on ``rank``."""
    return ((((seed * 1_000_003 + epoch) * 1_000_003 + rank) * 1_000_003 + index) * 2_654_435_761) % (1 << 63)


def draw_mix(mixup_alpha: float, cutmix_alpha: float, seed: int, epoch: int, rank: int, index: int,
             hw: int = DATA.crop) -> Optional[MixDraw]:
    """The batch's draw with torchvision's own parameter code, as its classification reference script
    builds it: ``RandomChoice([MixUp, CutMix])`` when both alphas are > 0 (its multinomial picks one),
    else the one enabled.  Drawn under ``torch.random.fork_rng`` with ``mix_seed``: reproducible, and
    no other random stream moves.  None when both alphas are 0 (no draw is made)."""
    if mixup_alpha <= 0 and cutmix_alpha <= 0:
        return None
    from torchvision.transforms import v2

    choices = []
    if mixup_alpha > 0:
        choices.append(v2.MixUp(alpha=mixup_alpha, num_classes=1))
    if cutmix_alpha > 0:
        choices.append(v2.CutMix(alpha=cutmix_alpha, num_classes=1))
    with torch.random.fork_rng(devices=[]):
        torch.manual_seed(mix_seed(seed, epoch, rank, index))
        t = choices[0]
        if len(choices) > 1:
            rc = v2.RandomChoice(choices)
            t = rc.transforms[int(torch.multinomial(torch.tensor(rc.p), 1))]
        # make_params reads only the image size; a stride-0 view gives it one without a buffer
        params = t.make_params([torch.zeros(()).expand(1, 3, hw, hw)])
    if isinstance(t, v2.CutMix):
        return MixDraw("cutmix", float(params["lam_adjusted"]), tuple(int(v) for v in params["box"]))
    return MixDraw("mixup", float(params["lam"]), (0, 0, 0, 0))


def _mix_transform(mix: MixDraw, labels: torch.Tensor):
    from torchvision.transforms import v2

    if mix.kind == "mixup":
        return v2.MixUp(alpha=1.0, num_classes=1), dict(lam=mix.lam, labels=labels, batch_size=labels.shape[0])
    return v2.CutMix(alpha=1.0, num_classes=1), dict(box=mix.box, lam_adjusted=mix.lam, labels=labels,
                                                     batch_size=labels.shape[0])


def apply_mix(x: torch.Tensor, labels: torch.Tensor, mix: Optional[MixDraw]) -> torch.Tensor:
    """Mix a float batch [b, 3, H, W] as torchvision's ``MixUp.transform`` / ``CutMix.transform`` do
    with the drawn params (the PIL pipeline and the oracle engine)."""
    if mix is None:
        return x
    t, params = _mix_transform(mix, labels)
    return t.transform(x, params)


def mixed_targets(labels: torch.Tensor, num_classes: int, mix: Optional[MixDraw]) -> torch.Tensor:
    """The probability targets torchvision hands to the loss for this draw: float32 [b, C]."""
    t, params = _mix_transform(mix, labels)
    t.num_classes = num_classes
    return t.transform(labels, params)


def reference_transforms(train: bool, resize: int = DATA.resize, crop: int = DATA.crop, tta: str = "none"):
    """The literal torchvision pipeline of the reference (distributedVggf.py:88-95 / :103-108), with
    its 256 / 224 made ``resize`` / ``crop`` (--train-crop-size, --val-resize-size, --val-crop-size).
    ``tta`` (validation only): Resize, then the mode's views with PIL's FiveCrop / TenCrop (``flip``: the centre
    crop and its mirror image), each made a tensor and normalised: float32 [V, 3, crop, crop] per image."""
    from torchvision import transforms as T

    norm = T.Normalize(list(DATA.mean), list(DATA.std))
    if train:
        return T.Compose([
            T.RandomResizedCrop(size=resize, scale=DATA.crop_scale),
            T.RandomRotation(degrees=DATA.rotation_deg),
            T.RandomHorizontalFlip(),
            T.CenterCrop(size=crop),
            T.ToTensor(),
            norm,
        ])
    if tta == "none":
        return T.Compose([T.Resize(size=resize), T.CenterCrop(size=crop), T.ToTensor(), norm])
    tta_views(tta)
    if tta == "flip":
        from torchvision.transforms import functional as TF
        views = T.Compose([T.CenterCrop(size=crop), T.Lambda(lambda im: (im, TF.hflip(im)))])
    else:
        views = T.FiveCrop(size=crop) if tta == "five-crop" else T.TenCrop(size=crop)
    return T.Compose([T.Resize(size=resize), views,
                      T.Lambda(lambda ims: torch.stack([norm(T.functional.to_tensor(im)) for im in ims]))])


def torchvision_chain_fixed(img_hwc_u8, params_row, resize: int = DATA.resize, crop: int = DATA.crop) -> torch.Tensor:
    """The reference's TRAIN pipeline (distributedVggf.py:88-95) with its random draws pinned to one row
    of ``sample_train_params``: torchvision's own functional ops on a PIL image --
    resized_crop(bilinear) -> rotate(nearest, zero fill) -> hflip -> center_crop -> to_tensor -> normalize.
    Used by the parity tests of ``augment_reference`` and of the sm_90a augment kernel."""
    from PIL import Image
    from torchvision.transforms import InterpolationMode
    from torchvision.transforms import functional as TF

    top, left, ch, cw, c, s, flip = [float(v) for v in params_row[:7]]
    img = Image.fromarray(img_hwc_u8.numpy() if isinstance(img_hwc_u8, torch.Tensor) else img_hwc_u8)
    img = TF.resized_crop(img, int(top), int(left), int(ch), int(cw), [resize, resize], InterpolationMode.BILINEAR)
    img = TF.rotate(img, math.degrees(math.atan2(s, c)), InterpolationMode.NEAREST, fill=0)
    if flip > 0.5:
        img = TF.hflip(img)
    img = TF.center_crop(img, [crop, crop])
    return TF.normalize(TF.to_tensor(img), list(DATA.mean), list(DATA.std))
