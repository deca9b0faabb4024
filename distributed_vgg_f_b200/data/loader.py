"""DataManager: ImageFolder -> mini-batches, in two flavours.

Reference (distributedVggf.py:63-123): ``DataManager(root_folder, mini_batch, train)`` exposes
``class_names / number_classes / data_size / loader / get_loader()``; the loader is a synchronous
``DataLoader(num_workers=0, pin_memory=False)`` over PIL transforms, sharded by a
``DistributedSampler`` only for the training split (validation runs in full on every rank).

Same surface here, two pipelines:
  * ``pipeline="reference"`` -- PIL decode + the literal torchvision transforms per sample.  Yields
    ``(float32 [mb,3,224,224], int64 [mb])``.  Bit-level semantics of the reference; ~400 img/s.
  * ``pipeline="fused"`` (default) -- every image is decoded ONCE into a uint8 cache (thread pool),
    a background thread gathers each batch into a pinned staging ring together with the sampled
    transform parameters, and the consumer runs the fused augment op on the device.  A split whose
    images all share one size of at most 256 x 256 (COIL-100, the synthetic set) yields
    ``FusedBatch``; any other split yields ``RaggedBatch``: the images of a batch back to back, one
    geometry row each, resampled on the device exactly as Pillow does.  The split must fit in host
    memory.  ``pipeline="auto"`` (the CLI default) switches to the reference pipeline for mixed
    image sizes or a split too big for host memory.
  * ``pipeline="stream"`` -- nothing is cached: each batch's files are read when it is drawn.  Host
    threads entropy-decode the JPEGs to quantised coefficients (csrc/jpeg_decode.cpp) and decode PNGs
    to RGB; files neither decoder takes are decoded once by PIL at start-up.  Yields ``JpegBatch``,
    which the device decodes (csrc/jpeg.cu) into exactly the ``RaggedBatch`` a ragged cache of the
    split would yield: same indices, labels, parameters, geometry and MixUp / CutMix draws.
Ragged final batches are preserved (``drop_last=False`` in the reference).

With ``mixup_alpha`` / ``cutmix_alpha`` > 0 every training batch carries a MixUp or CutMix draw
(``transforms.draw_mix``, seeded by (seed, epoch, rank, batch index)): fused batches in their ``mix``
field, for the augment kernel to apply; the reference pipeline applies it on the host and yields
``(mixed float batch, labels, draw)``.  Validation batches are never mixed.
"""
from __future__ import annotations

import os
import queue
import threading
from concurrent.futures import ThreadPoolExecutor
from typing import Iterator, List, NamedTuple, Optional, Tuple

import numpy as np
import torch

from ..config import DATA
from . import transforms as T
from .folder import scan_image_folder
from .sampler import ShardedSampler


class FusedBatch(NamedTuple):
    images_u8: torch.Tensor     # uint8 [mb, H, W, 3] (pinned when CUDA is present)
    params: torch.Tensor        # float32 [mb, 8]     (same)
    labels: torch.Tensor        # int64 [mb]          (same)
    resized_hw: Tuple[int, int]
    state: Optional[dict] = None    # consumer may set state["event"]: slot is reusable after it fires
    mix: Optional[T.MixDraw] = None     # MixUp / CutMix of this training batch

    def to_float(self, device="cpu", out_hw: int = DATA.crop, view: Optional[int] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """Evaluate the fused transform with torch ops (CPU / oracle path), cut to ``out_hw`` (at TTA view ``view``)."""
        x = T.augment_reference(self.images_u8.to(device), self.params, self.resized_hw, out_hw=out_hw, view=view)
        return x, self.labels.to(device)


class RaggedBatch(NamedTuple):
    """A batch of images of any sizes: ``data_u8`` holds them back to back, row i of ``geom`` is
    image i's (byte offset, H, W, RH, RW) with (RH, RW) the size it is resized to."""
    data_u8: torch.Tensor       # uint8 [bytes]        (pinned when CUDA is present)
    geom: torch.Tensor          # int64 [mb, 5]        (same)
    params: torch.Tensor        # float32 [mb, 8]      (same)
    labels: torch.Tensor        # int64 [mb]           (same)
    state: Optional[dict] = None    # consumer may set state["event"]: slot is reusable after it fires
    mix: Optional[T.MixDraw] = None     # MixUp / CutMix of this training batch

    @property
    def nbytes(self) -> int:
        """Bytes of the images."""
        return int(self.data_u8.numel())

    def to_float(self, device="cpu", out_hw: int = DATA.crop, view: Optional[int] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """Evaluate the transform with Pillow's resampling on the CPU (CPU / oracle path), cut to ``out_hw`` (at
        TTA view ``view``)."""
        x = T.ragged_reference(self.data_u8, self.geom, self.params, out_hw=out_hw, view=view)
        return x.to(device), self.labels.to(device)


class JpegBatch(NamedTuple):
    """A stream batch before decoding: the JPEGs' quantised coefficients and tables, the other images' RGB, one
    descriptor row per image (data/jpeg.py, csrc/include/jpeg.h), and ``geom`` rows of the decoded images back to
    back, exactly as ``RaggedBatch``'s."""
    coef: torch.Tensor          # int16 [blocks * 64]       (pinned when CUDA is present)
    quant: torch.Tensor         # int32 [mb * 3, 64]        (same)
    raw: torch.Tensor           # uint8 [bytes]             (same)
    desc: torch.Tensor          # int32 [mb, 16]            (same)
    geom: torch.Tensor          # int64 [mb, 5]             (same)
    params: torch.Tensor        # float32 [mb, 8]           (same)
    labels: torch.Tensor        # int64 [mb]                (same)
    state: Optional[dict] = None    # consumer may set state["event"]: slot is reusable after it fires
    mix: Optional[T.MixDraw] = None     # MixUp / CutMix of this training batch

    @property
    def nbytes(self) -> int:
        """Bytes of the decoded images."""
        g = self.geom[-1]
        return int(g[0] + g[1] * g[2] * 3)

    def decode(self) -> torch.Tensor:
        """The decoded images back to back (uint8, a ``RaggedBatch``'s ``data_u8``), by the CPU reference."""
        from .jpeg import decode_batch
        return torch.from_numpy(decode_batch(self.coef.numpy(), self.quant.numpy(), self.raw.numpy(),
                                             self.desc.numpy(), self.geom.numpy()))

    def to_float(self, device="cpu", out_hw: int = DATA.crop, view: Optional[int] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """Decode on the CPU, then evaluate the transform as ``RaggedBatch.to_float`` does."""
        x = T.ragged_reference(self.decode(), self.geom, self.params, out_hw=out_hw, view=view)
        return x.to(device), self.labels.to(device)


DEVICE_BATCHES = (FusedBatch, RaggedBatch, JpegBatch)     # batches whose transform runs on the consumer's side


def _decode(path: str) -> np.ndarray:
    from PIL import Image

    with open(path, "rb") as f:
        return np.asarray(Image.open(f).convert("RGB"), dtype=np.uint8)


class CacheUnavailable(ValueError):
    """The split cannot be cached (too big for host RAM, or mixed image sizes where they are refused)."""


def _cache_budget_bytes() -> int:
    """B200_MAX_CACHE_GB, else half of the memory the OS reports as available (at most 64 GB)."""
    env = os.environ.get("B200_MAX_CACHE_GB")
    if env:
        return int(float(env) * (1 << 30))
    try:
        with open("/proc/meminfo") as f:
            for line in f:
                if line.startswith("MemAvailable:"):
                    return min(int(line.split()[1]) * 1024 // 2, 64 << 30)
    except OSError:
        pass
    return 16 << 30


def _header_hw(path: str) -> Tuple[int, int]:
    from PIL import Image

    with Image.open(path) as im:
        w, h = im.size
    return h, w


class DecodedCache:
    """All images of a split, decoded once to uint8 HWC (PNGs by the native decoder where it can).

    One image size of at most ``resize`` (the split's resize size) on both sides: ``images`` is [N,H,W,3].  Otherwise
    (``ragged``): ``flat`` holds the images back to back, image i at ``offsets[i]`` with size
    ``hw[i]``.  ``allow_mixed=False`` refuses a split of mixed sizes.  The budget is checked from
    the file headers before anything is decoded."""

    def __init__(self, samples: List[Tuple[str, int]], threads: int = 8, max_bytes: Optional[int] = None,
                 allow_mixed: bool = True, resize: int = DATA.resize) -> None:
        paths = [p for p, _ in samples]
        with ThreadPoolExecutor(max_workers=threads) as ex:
            hw = list(ex.map(_header_hw, paths))
        sizes = set(hw)
        if len(sizes) > 1 and not allow_mixed:
            raise CacheUnavailable("mixed image sizes (%s ...)" % sorted(sizes)[:4])
        need = sum(h * w * 3 for h, w in hw)
        budget = _cache_budget_bytes() if max_bytes is None else max_bytes
        if need > budget:
            raise CacheUnavailable("decoded cache needs %.1f GB for %d images, budget %.1f GB "
                                   "(B200_MAX_CACHE_GB)" % (need / 2**30, len(paths), budget / 2**30))
        self.labels = torch.tensor([l for _, l in samples], dtype=torch.int64)
        self.ragged = bool(paths) and (len(sizes) > 1 or max(hw[0]) > resize)
        if self.ragged:
            self._decode_ragged(paths, hw, threads)
            return
        images = None
        try:   # native multi-threaded PNG decode (csrc/png_decode.cpp), falls back to PIL
            from ..ops import native_decode_pngs
            images = native_decode_pngs(paths, threads)
        except Exception:
            images = None
        self.native_decode = images is not None
        if images is None:
            with ThreadPoolExecutor(max_workers=threads) as ex:
                arrays = list(ex.map(_decode, paths))
            images = torch.from_numpy(np.stack(arrays))
        self.images = images                                          # [N,H,W,3] uint8
        self.src_hw = (int(self.images.shape[1]), int(self.images.shape[2]))

    def _decode_ragged(self, paths: List[str], hw: List[Tuple[int, int]], threads: int) -> None:
        self.images, self.src_hw = None, None
        self.hw = torch.tensor(hw, dtype=torch.int64).view(-1, 2)
        nbytes = self.hw[:, 0] * self.hw[:, 1] * 3
        self.offsets = torch.cumsum(nbytes, 0) - nbytes
        self.flat = torch.empty(int(nbytes.sum()), dtype=torch.uint8)
        done = torch.zeros(len(paths), dtype=torch.bool)
        png = [i for i, p in enumerate(paths) if p.lower().endswith(".png")]
        from .. import ops
        if png and ops.available():
            sel = torch.tensor(png, dtype=torch.int64)
            ok = ops.require().decode_pngs_into([paths[i] for i in png], self.flat, self.offsets[sel].contiguous(),
                                                self.hw[sel].contiguous(), threads)
            done[sel] = ok
        self.native_decode = int(done.sum())          # images the native decoder wrote

        def pil(i: int) -> None:
            a = _decode(paths[i])
            h, w = int(self.hw[i, 0]), int(self.hw[i, 1])
            if a.shape != (h, w, 3):
                raise ValueError("%s decodes to %s, its header says %dx%d" % (paths[i], a.shape, h, w))
            off = int(self.offsets[i])
            self.flat[off:off + h * w * 3].numpy().reshape(h, w, 3)[...] = a

        rest = [i for i in range(len(paths)) if not bool(done[i])]
        with ThreadPoolExecutor(max_workers=threads) as ex:
            list(ex.map(pil, rest))


class _FusedLoader:
    """Batches for the fused GPU pipeline.  With the native extension present, a C++ worker thread
    (csrc/prefetch.cpp) gathers images from the decoded cache into a pinned ring and draws the
    transform parameters without ever taking the GIL; otherwise a Python thread does the same."""

    def __init__(self, cache: DecodedCache, mb: int, train: bool, sampler: Optional[ShardedSampler],
                 shuffle: bool, seed: int, prefetch: int = 3, pin: Optional[bool] = None,
                 native: Optional[bool] = None, mixup_alpha: float = 0.0, cutmix_alpha: float = 0.0,
                 resize: int = DATA.resize, crop: int = DATA.crop) -> None:
        self.cache, self.mb, self.train = cache, mb, train
        self.resize, self.crop = resize, crop          # the network input the batches are cut to
        self.mixup_alpha, self.cutmix_alpha = (mixup_alpha, cutmix_alpha) if train else (0.0, 0.0)
        self.sampler, self.shuffle, self.seed = sampler, shuffle, seed
        self.prefetch = prefetch
        self.pin = torch.cuda.is_available() if pin is None else pin
        self.epoch = 0
        self.ragged = cache.ragged
        slots = prefetch + 1
        self._par = self._buf((slots, mb, T.PARAM_DIM), torch.float32)
        self._lab = self._buf((slots, mb), torch.int64)
        if self.ragged:
            # a slot holds any batch: the mb largest images of the split
            sizes = (cache.hw[:, 0] * cache.hw[:, 1] * 3).sort(descending=True).values
            self.resized_hw = None
            self._img = self._buf((slots, max(int(sizes[:mb].sum()), 1)), torch.uint8)
            self._geom = self._buf((slots, mb, T.GEOM_DIM), torch.int64)
        else:
            H, W = cache.src_hw
            self.resized_hw = T.resized_dims(train, H, W, resize)
            self._img = self._buf((slots, mb, H, W, 3), torch.uint8)
            self._geom = None
        self._ring = [(self._img[s], self._par[s], self._lab[s]) for s in range(slots)]
        self._state = [{} for _ in range(slots)]
        self._pf = None
        if native is None or native:
            try:
                from .. import ops
                if ops.available() and hasattr(ops.require(), "Prefetcher"):
                    extra = {}
                    if self.ragged:
                        extra = dict(offsets=cache.offsets, hw=cache.hw, ring_geom=self._geom, resize=resize)
                    self._pf = ops.require().Prefetcher(
                        cache.flat if self.ragged else cache.images, cache.labels, self._img, self._par, self._lab,
                        train, DATA.crop_scale[0], DATA.crop_scale[1], DATA.crop_ratio[0], DATA.crop_ratio[1],
                        DATA.rotation_deg, **extra)
            except Exception:
                if native:
                    raise
                self._pf = None

    def _buf(self, shape, dtype):
        t = torch.empty(shape, dtype=dtype)
        return t.pin_memory() if self.pin else t

    def __len__(self) -> int:
        n = len(self.sampler) if self.sampler is not None else len(self.cache.labels)
        return (n + self.mb - 1) // self.mb

    def set_epoch(self, epoch: int) -> None:
        self.epoch = epoch
        if self.sampler is not None:
            self.sampler.set_epoch(epoch)

    def _indices(self) -> List[int]:
        if self.sampler is not None:
            return list(iter(self.sampler))
        n = len(self.cache.labels)
        if self.shuffle:
            g = torch.Generator().manual_seed(self.seed + self.epoch)
            return torch.randperm(n, generator=g).tolist()
        return list(range(n))

    def _epoch_seed(self) -> int:
        return 1_000_003 * (self.seed + 1) + self.epoch * 7919 + (self.sampler.rank if self.sampler else 0)

    def _draw(self, index: int) -> Optional[T.MixDraw]:
        return T.draw_mix(self.mixup_alpha, self.cutmix_alpha, self.seed, self.epoch,
                          self.sampler.rank if self.sampler else 0, index, hw=self.crop)

    def _batch(self, slot: int, k: int, index: int = 0):
        img, par, lab = self._ring[slot]
        mix = self._draw(index)
        if not self.ragged:
            return FusedBatch(img[:k], par[:k], lab[:k], self.resized_hw, self._state[slot], mix)
        geom = self._geom[slot][:k]
        used = int(geom[k - 1, 0] + geom[k - 1, 1] * geom[k - 1, 2] * 3)
        return RaggedBatch(img[:used], geom, par[:k], lab[:k], self._state[slot], mix)

    def __iter__(self) -> Iterator[FusedBatch]:
        if self._pf is not None:
            return self._iter_native()
        return self._iter_python()

    # -- native worker thread ---------------------------------------------------------------------
    def _iter_native(self) -> Iterator[FusedBatch]:
        self._pf.start(self._indices(), self._epoch_seed())
        prev = None
        index = 0
        try:
            while True:
                item = self._pf.next()           # blocks with the GIL released
                if prev is not None:             # consumer asked for more: previous slot may be refilled
                    ev = self._state[prev].pop("event", None)
                    self._state[prev]["held"] = ev          # keep the event alive until the worker used it
                    self._pf.release(prev, int(ev.cuda_event) if ev is not None else 0)
                    prev = None
                if item is None:
                    break
                slot, k = item
                prev = slot
                yield self._batch(slot, k, index)
                index += 1
        finally:
            self._pf.stop()

    # -- Python fallback ---------------------------------------------------------------------------
    def _iter_python(self) -> Iterator[FusedBatch]:
        idx = self._indices()
        gen = torch.Generator().manual_seed(self._epoch_seed())
        H, W = self.cache.src_hw or (0, 0)
        q: "queue.Queue" = queue.Queue(maxsize=self.prefetch)
        free: "queue.Queue" = queue.Queue()
        for slot in range(len(self._ring)):
            free.put(slot)

        def produce():
            for b0 in range(0, len(idx), self.mb):
                sel = torch.tensor(idx[b0:b0 + self.mb], dtype=torch.int64)
                k = len(sel)
                slot = free.get()
                ev = self._state[slot].pop("event", None)
                if ev is not None:
                    ev.synchronize()        # async H2D of the previous occupant has finished
                img, par, lab = self._ring[slot]
                torch.index_select(self.cache.labels, 0, sel, out=lab[:k])
                if self.ragged:
                    hw = self.cache.hw[sel]
                    geom = self._geom[slot][:k]
                    geom.copy_(T.ragged_geometry(hw.tolist(), self.train, self.resize))
                    for i, (h, w) in enumerate(hw.tolist()):
                        off, o, n = int(self.cache.offsets[sel[i]]), int(geom[i, 0]), h * w * 3
                        img[o:o + n].copy_(self.cache.flat[off:off + n])
                        par[i] = (T.sample_train_params(1, h, w, gen) if self.train else T.val_params(1, h, w))[0]
                else:
                    torch.index_select(self.cache.images, 0, sel, out=img[:k])
                    par[:k] = (T.sample_train_params(k, H, W, gen) if self.train
                               else T.val_params(k, H, W))
                q.put((slot, k))
            q.put(None)

        th = threading.Thread(target=produce, daemon=True)
        th.start()
        prev = None
        index = 0
        while True:
            item = q.get()
            if prev is not None:
                free.put(prev)      # consumer is done with the previous slot once it asks for more
            if item is None:
                break
            slot, k = item
            prev = slot
            yield self._batch(slot, k, index)
            index += 1
        th.join()


class _StreamSplit(NamedTuple):
    """What the stream loader knows of its split without decoding it: labels, sizes and header rows."""
    labels: torch.Tensor        # int64 [N]
    hw: torch.Tensor            # int64 [N, 2]
    headers: torch.Tensor       # int64 [N, 12]: ops jpeg_scan rows


class _StreamLoader(_FusedLoader):
    """Batches for ``pipeline="stream"``: the ragged fused loader's batches, decoded from the files per batch.

    A native worker (csrc/prefetch.cpp) draws each batch exactly as ``_FusedLoader`` does over a ragged cache and
    lays it out in a pinned slot; ``threads`` decode threads fill the slot's fixed positions.  The slot holds the
    coefficients of the ``mb`` largest JPEGs of the split and the RGB of its ``mb`` largest other images."""

    def __init__(self, samples: List[Tuple[str, int]], mb: int, train: bool, sampler: Optional[ShardedSampler],
                 shuffle: bool, seed: int, threads: int = 8, prefetch: int = 3, pin: Optional[bool] = None,
                 mixup_alpha: float = 0.0, cutmix_alpha: float = 0.0, resize: int = DATA.resize,
                 crop: int = DATA.crop, max_bytes: Optional[int] = None) -> None:
        from .. import ops
        C = ops.require()
        self.mb, self.train, self.resize, self.crop = mb, train, resize, crop
        self.mixup_alpha, self.cutmix_alpha = (mixup_alpha, cutmix_alpha) if train else (0.0, 0.0)
        self.sampler, self.shuffle, self.seed = sampler, shuffle, seed
        self.prefetch, self.epoch, self.ragged, self.resized_hw = prefetch, 0, True, None
        self.pin = torch.cuda.is_available() if pin is None else pin
        self.threads = threads
        paths = [p for p, _ in samples]
        headers = C.jpeg_scan(paths, threads)
        # a PNG goes to the native decoder per batch only if that decoder takes it (the scan reads its IHDR alone)
        png = (headers[:, 0] == 2).nonzero().flatten()
        if len(png):
            ok = C.png_decodable([paths[i] for i in png.tolist()], headers[png, 1:3].contiguous(), threads)
            headers[png[~ok], 0] = 0
        kind = headers[:, 0]
        hw = headers[:, 1:3].clone()
        # files neither native decoder takes: decoded once by PIL, kept as RGB.  Their size comes from the scan
        # (JPEG frame, PNG IHDR) or PIL's header, and the budget is checked before anything is decoded.
        other = (kind == 0).nonzero().flatten().tolist()
        unsized = [i for i in other if hw[i, 0] < 1 or hw[i, 1] < 1]
        with ThreadPoolExecutor(max_workers=threads) as ex:
            for i, (h, w) in zip(unsized, ex.map(lambda i: _header_hw(paths[i]), unsized)):
                hw[i, 0], hw[i, 1] = h, w
        nbytes = (hw[other, 0] * hw[other, 1] * 3) if other else torch.zeros(0, dtype=torch.int64)
        need = int(nbytes.sum())
        budget = _cache_budget_bytes() if max_bytes is None else max_bytes
        if need > budget:
            raise CacheUnavailable("the %d files the stream decoders do not take need %.1f MB decoded, budget %.1f MB "
                                   "(B200_MAX_CACHE_GB)" % (len(other), need / 2**20, budget / 2**20))
        self.other_count, self.other_bytes = len(other), need
        other_off = torch.full((len(paths),), -1, dtype=torch.int64)
        if other:
            other_off[other] = torch.cumsum(nbytes, 0) - nbytes
        flat = torch.empty(max(need, 1), dtype=torch.uint8)

        def pil(i: int) -> None:         # one decoded image per thread at a time
            a = _decode(paths[i])
            h, w = int(hw[i, 0]), int(hw[i, 1])
            if a.shape != (h, w, 3):
                raise ValueError("%s decodes to %s, its header says %dx%d" % (paths[i], a.shape, h, w))
            off = int(other_off[i])
            flat[off:off + h * w * 3].numpy()[...] = a.reshape(-1)

        with ThreadPoolExecutor(max_workers=threads) as ex:
            list(ex.map(pil, other))
        self.cache = _StreamSplit(torch.tensor([l for _, l in samples], dtype=torch.int64), hw, headers)
        jpeg = kind == 1
        coef = (headers[jpeg, 11] * 64).sort(descending=True).values
        rgb = (hw[~jpeg, 0] * hw[~jpeg, 1] * 3).sort(descending=True).values
        slots = prefetch + 1
        self._coef = self._buf((slots, max(int(coef[:mb].sum()), 64)), torch.int16)
        self._raw = self._buf((slots, max(int(rgb[:mb].sum()), 1)), torch.uint8)
        self._quant = self._buf((slots, mb * 3, 64), torch.int32)
        self._desc = self._buf((slots, mb, C.JPEG_DESC), torch.int32)
        self._geom = self._buf((slots, mb, T.GEOM_DIM), torch.int64)
        self._par = self._buf((slots, mb, T.PARAM_DIM), torch.float32)
        self._lab = self._buf((slots, mb), torch.int64)
        self._state = [{} for _ in range(slots)]
        self._pf = C.StreamPrefetcher(paths, headers, self.cache.labels, hw, flat, other_off, self._coef, self._quant,
                                      self._raw, self._desc, self._geom, self._par, self._lab, train,
                                      DATA.crop_scale[0], DATA.crop_scale[1], DATA.crop_ratio[0], DATA.crop_ratio[1],
                                      DATA.rotation_deg, resize, threads)

    def _batch(self, slot: int, k: int, index: int = 0) -> JpegBatch:
        desc = self._desc[slot][:k]
        d = desc.numpy()
        blocks = int(d[-1, 3] + (d[-1, 5:8] * d[-1, 8:11]).sum())
        raw = d[d[:, 0] == 0]
        g = self._geom[slot][:k]
        rows = g.numpy()[d[:, 0] == 0]
        used = int((raw[:, 4] + rows[:, 1] * rows[:, 2] * 3).max()) if len(raw) else 0
        return JpegBatch(self._coef[slot][:blocks * 64], self._quant[slot][:k * 3], self._raw[slot][:used], desc, g,
                         self._par[slot][:k], self._lab[slot][:k], self._state[slot], self._draw(index))

    def __iter__(self) -> Iterator[JpegBatch]:
        return self._iter_native()


class _ReferenceLoader:
    """Synchronous PIL + torchvision loader with the reference's exact semantics."""

    def __init__(self, samples, mb: int, train: bool, sampler: Optional[ShardedSampler],
                 shuffle: bool, seed: int, mixup_alpha: float = 0.0, cutmix_alpha: float = 0.0,
                 resize: int = DATA.resize, crop: int = DATA.crop, tta: str = "none") -> None:
        self.samples, self.mb, self.sampler = samples, mb, sampler
        self.crop = crop
        self.shuffle, self.seed, self.epoch = shuffle, seed, 0
        self.mixup_alpha, self.cutmix_alpha = (mixup_alpha, cutmix_alpha) if train else (0.0, 0.0)
        self.tf = T.reference_transforms(train, resize, crop) if tta == "none" else \
            T.reference_transforms(train, resize, crop, tta)

    def __len__(self) -> int:
        n = len(self.sampler) if self.sampler is not None else len(self.samples)
        return (n + self.mb - 1) // self.mb

    def set_epoch(self, epoch: int) -> None:
        self.epoch = epoch
        if self.sampler is not None:
            self.sampler.set_epoch(epoch)

    def __iter__(self):
        from PIL import Image

        if self.sampler is not None:
            idx = list(iter(self.sampler))
        elif self.shuffle:
            idx = torch.randperm(len(self.samples)).tolist()
        else:
            idx = list(range(len(self.samples)))
        for b0 in range(0, len(idx), self.mb):
            xs, ys = [], []
            for i in idx[b0:b0 + self.mb]:
                path, label = self.samples[i]
                with open(path, "rb") as f:
                    xs.append(self.tf(Image.open(f).convert("RGB")))
                ys.append(label)
            x, y = torch.stack(xs), torch.tensor(ys, dtype=torch.int64)
            mix = T.draw_mix(self.mixup_alpha, self.cutmix_alpha, self.seed, self.epoch,
                             self.sampler.rank if self.sampler else 0, b0 // self.mb, hw=self.crop)
            if mix is None:
                yield x, y
            else:       # mixed on the host by torchvision, the draw travels with the batch
                yield T.apply_mix(x, y, mix), y, mix


class DataManager:
    """Same constructor / attributes as the reference's class (distributedVggf.py:63-123)."""

    def __init__(self, root_folder: str, mini_batch: int, train: bool = True, *,
                 world_size: int = 1, rank: int = 0, pipeline: str = "fused", seed: int = 0,
                 reference_order: bool = False, decode_threads: int = 8, shard_eval: bool = False,
                 mixup_alpha: float = 0.0, cutmix_alpha: float = 0.0, resize_size: int = DATA.resize,
                 crop_size: int = DATA.crop, tta: str = "none") -> None:
        """``resize_size`` / ``crop_size``: the split's RandomResizedCrop (train) or Resize (val) size and
        the CenterCrop after it, the network's input (torchvision's --train-crop-size, --val-resize-size,
        --val-crop-size).  ``tta`` (validation, --val-tta): the reference pipeline yields every image's views,
        float32 [mb, V, 3, crop, crop]; fused batches are the same for every mode (their consumer takes the views)."""
        if root_folder is None:
            raise ValueError("-rd/--root_dir is required")
        T.tta_views(tta)
        if train and tta != "none":
            raise ValueError("test-time augmentation applies to validation splits only")
        self.root_folder, self.mb_size, self.train = root_folder, mini_batch, train
        self.resize_size, self.crop_size = int(resize_size), int(crop_size)
        self.path = os.path.join(root_folder, DATA.train_dir if train else DATA.val_dir)
        self.class_names, self.samples = scan_image_folder(self.path)
        self.number_classes = len(self.class_names)
        self.data_size = len(self.samples)
        sampler = None
        if train and world_size > 1:      # validation is NOT sharded (distributedVggf.py:115)
            sampler = ShardedSampler(self.data_size, world_size, rank, seed=seed,
                                     reference_order=reference_order)
        elif shard_eval and world_size > 1:   # extension: exact partition, metrics all-reduced
            sampler = ShardedSampler(self.data_size, world_size, rank, shuffle=False, pad=False)
        if pipeline == "stream":
            self.loader = _StreamLoader(self.samples, mini_batch, train, sampler, True, seed, threads=decode_threads,
                                        mixup_alpha=mixup_alpha, cutmix_alpha=cutmix_alpha,
                                        resize=self.resize_size, crop=self.crop_size)
            self.pipeline = pipeline
            if self.loader.other_count:
                print("[Info] stream pipeline: %d file(s) no stream decoder takes, decoded by PIL at start-up "
                      "(%.1f MB)" % (self.loader.other_count, self.loader.other_bytes / 2**20), flush=True)
            return
        if pipeline in ("fused", "auto"):
            try:
                self.cache = DecodedCache(self.samples, decode_threads, allow_mixed=pipeline == "fused",
                                          resize=self.resize_size)
            except CacheUnavailable as e:
                if pipeline == "fused":
                    raise
                # mixed sizes / larger than host memory: the reference's per-sample PIL pipeline
                # handles anything an ImageFolder can hold (every rank sees the same files, so
                # every rank takes the same branch)
                print("[Info] %s -> using the per-sample (reference) input pipeline" % e, flush=True)
                pipeline = "reference"
        self.pipeline = pipeline = "fused" if pipeline == "auto" else pipeline
        if pipeline == "fused":
            self.loader = _FusedLoader(self.cache, mini_batch, train, sampler, True, seed,
                                       mixup_alpha=mixup_alpha, cutmix_alpha=cutmix_alpha,
                                       resize=self.resize_size, crop=self.crop_size)
        elif pipeline == "reference":
            self.loader = _ReferenceLoader(self.samples, mini_batch, train, sampler, True, seed,
                                           mixup_alpha=mixup_alpha, cutmix_alpha=cutmix_alpha,
                                           resize=self.resize_size, crop=self.crop_size, tta=tta)
        else:
            raise ValueError("pipeline must be 'fused', 'stream', 'reference' or 'auto'")

    def get_loader(self):
        return self.loader
