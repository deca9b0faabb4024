"""The fused input pipeline on ImageFolders of any image size (``RaggedBatch``), without a GPU: the
Pillow-exact resize oracle, the ragged train / val chains against torchvision, the ragged decoded
cache and both prefetchers.  Every image is made here with PIL."""
import hashlib
import math
import os

import numpy as np
import pytest
import torch
from PIL import Image

from distributed_vgg_f_b200 import ops
from distributed_vgg_f_b200.data import transforms as T
from distributed_vgg_f_b200.data.loader import (CacheUnavailable, DataManager, DecodedCache, FusedBatch,
                                                RaggedBatch, _FusedLoader)


def _textured(h, w, seed):
    """Fine stripes plus noise: content that aliases when a resize does not filter its footprint."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    base = (127 + 100 * np.sin(xx * 1.3 + seed) * np.cos(yy * 0.9))[..., None].repeat(3, 2)
    return np.clip(base + rng.integers(-20, 20, (h, w, 3)), 0, 255).astype(np.uint8)


def _flat(images):
    """(flat uint8 buffer, [k, 2] sizes) of images laid back to back."""
    data = torch.from_numpy(np.concatenate([a.reshape(-1) for a in images]))
    return data, [a.shape[:2] for a in images]


# ------------------------------------------------------------------------------------- oracle
@pytest.mark.parametrize("src,dst", [
    ((115, 122), (256, 256)),      # enlarge
    ((300, 352), (256, 256)),      # shrink a little
    ((827, 732), (256, 256)),
    ((480, 640), (256, 341)),      # val of a landscape photo
    ((1000, 750), (341, 256)),     # val of a portrait photo
    ((2300, 2100), (256, 256)),    # shrink by more than 8x
    ((97, 161), (256, 256)),       # odd sizes
    ((1, 255), (256, 256)),        # 1 x N strip
    ((60, 400), (256, 1706)),      # aspect beyond 4:1
    ((256, 333), (256, 256)),      # vertical axis unchanged
    ((301, 256), (256, 256)),      # horizontal axis unchanged
    ((77, 77), (77, 77)),          # nothing to do
])
def test_pil_resize_reference_is_bit_exact(src, dst):
    img = np.random.default_rng(src[0] * 7 + src[1]).integers(0, 256, src + (3,), dtype=np.uint8)
    ref = np.asarray(Image.fromarray(img).resize((dst[1], dst[0]), Image.BILINEAR))
    got = T.pil_resize_reference(img, *dst)
    assert got.dtype == np.uint8 and np.array_equal(got, ref)
    assert torch.equal(T.pil_resize_reference(torch.from_numpy(img), *dst), torch.from_numpy(ref.copy()))


SIZES = [(128, 128), (300, 400), (480, 640), (1000, 750), (61, 333), (257, 256)]


def test_ragged_val_chain_equals_torchvision():
    """Resize(256) -> CenterCrop(224) -> ToTensor -> Normalize of torchvision, to float rounding."""
    images = [_textured(h, w, i) for i, (h, w) in enumerate(SIZES)]
    data, hw = _flat(images)
    geom = T.ragged_geometry(hw, train=False)
    params = torch.cat([T.val_params(1, h, w) for h, w in hw])
    got = T.ragged_reference(data, geom, params)
    tf = T.reference_transforms(False)
    for i, a in enumerate(images):
        ref = tf(Image.fromarray(a))
        assert float((got[i] - ref).abs().max()) < 1e-6, (SIZES[i], float((got[i] - ref).abs().max()))


def test_ragged_train_chain_matches_torchvision_on_fixed_draws():
    """The train chain against torchvision's own ops with the same draws: equal but for pixels where
    the nearest rotation lands within float rounding of a pixel edge (as in test_scaffold_cpu's check
    of the uniform transform)."""
    images = [_textured(h, w, 10 + i) for i, (h, w) in enumerate(SIZES)]
    data, hw = _flat(images)
    g = torch.Generator().manual_seed(5)
    params = torch.cat([T.sample_train_params(1, h, w, g) for h, w in hw])
    params[0, 6], params[1, 6] = 0.0, 1.0
    params[2, 4], params[2, 5] = math.cos(math.radians(9.5)), math.sin(math.radians(9.5))
    params[3, 4], params[3, 5] = math.cos(math.radians(-9.5)), math.sin(math.radians(-9.5))
    got = T.ragged_reference(data, T.ragged_geometry(hw, train=True), params)
    for i, a in enumerate(images):
        ref = T.torchvision_chain_fixed(a, params[i])
        exact = float(((got[i] - ref).abs() < 1e-6).float().mean())
        assert exact >= 0.995, (SIZES[i], exact)


def test_ragged_reference_on_uniform_small_images_is_close_to_the_uniform_oracle():
    """Where Pillow's filter is the 2-tap one (enlarging), the uint8 rounding of the resized image is
    all that separates the ragged oracle from augment_reference."""
    images = [_textured(128, 128, i) for i in range(3)]
    data, hw = _flat(images)
    params = T.sample_train_params(3, 128, 128, torch.Generator().manual_seed(2))
    a = T.ragged_reference(data, T.ragged_geometry(hw, True), params)
    b = T.augment_reference(torch.from_numpy(np.stack(images)), params, (256, 256))
    close = float(((a - b).abs() < 0.03).float().mean())
    assert close > 0.995, close


# ------------------------------------------------------------------------------------- loader
MIXED = [(96, 130, "png"), (300, 200, "jpg"), (480, 640, "gray"), (1, 77, "palette"), (257, 256, "png"),
         (64, 300, "rgba"), (200, 90, "jpg"), (130, 96, "png")]


def _write_mixed(root):
    """Two classes of the MIXED images in each split: PNG, JPEG, grayscale, palette and RGBA PNGs."""
    for split in ("TrainData", "ValidationData"):
        for c, cls in enumerate(("alpha", "beta")):
            d = os.path.join(root, split, cls)
            os.makedirs(d, exist_ok=True)
            for i, (h, w, kind) in enumerate(MIXED):
                img = Image.fromarray(_textured(h, w, 100 * c + i))
                name = os.path.join(d, "%d.%s" % (i, "jpg" if kind == "jpg" else "png"))
                if kind == "gray":
                    img = img.convert("L")
                elif kind == "palette":
                    img = img.convert("P")
                elif kind == "rgba":
                    img = img.convert("RGBA")
                img.save(name)
    return root


@pytest.fixture(scope="module")
def mixed_root(tmp_path_factory):
    return _write_mixed(str(tmp_path_factory.mktemp("mixed")))


def _pil_rgb(path):
    with open(path, "rb") as f:
        return np.asarray(Image.open(f).convert("RGB"))


def _digest(a):
    return hashlib.sha1(np.ascontiguousarray(a).tobytes()).hexdigest()


def _delivered(batches):
    """(digest of the image, H, W, label) of every sample of RaggedBatches."""
    out = []
    for b in batches:
        assert isinstance(b, RaggedBatch)
        for i, (off, h, w, _, _) in enumerate(b.geom.tolist()):
            out.append((_digest(b.data_u8[off:off + h * w * 3].numpy()), h, w, int(b.labels[i])))
    return out


def test_fused_pipeline_on_a_mixed_folder_delivers_every_sample_once(mixed_root):
    expect = []
    dm = DataManager(mixed_root, 3, train=True, pipeline="fused")
    assert dm.pipeline == "fused" and dm.cache.ragged
    for path, label in dm.samples:
        a = _pil_rgb(path)
        expect.append((_digest(a), a.shape[0], a.shape[1], label))
    got = _delivered(dm.get_loader())
    assert sorted(got) == sorted(expect)
    if ops.available():            # the PNGs are decoded natively; JPEGs by PIL
        assert dm.cache.native_decode == sum(1 for p, _ in dm.samples if p.endswith(".png"))
    # two ranks: disjoint shards that cover the split
    shards = [_delivered(DataManager(mixed_root, 3, train=True, pipeline="fused", world_size=2, rank=r).get_loader())
              for r in range(2)]
    assert len(shards[0]) == len(shards[1]) == len(expect) // 2
    assert sorted(shards[0] + shards[1]) == sorted(expect)
    # validation: resized to shorter side 256, the whole image as the box, no rotation or flip
    dv = DataManager(mixed_root, 5, train=False, pipeline="fused")
    for b in dv.get_loader():
        for (off, h, w, rh, rw), p in zip(b.geom.tolist(), b.params.tolist()):
            assert (rh, rw) == T.resized_dims(False, h, w)
            assert p[:7] == [0, 0, h, w, 1.0, 0.0, 0.0]
    x, y = b.to_float()
    assert x.shape == (len(y), 3, 224, 224) and bool(torch.isfinite(x).all())


def test_train_params_of_ragged_batches_fit_each_image(mixed_root):
    dm = DataManager(mixed_root, 4, train=True, pipeline="fused", seed=2)
    for b in dm.get_loader():
        for (off, h, w, rh, rw), p in zip(b.geom.tolist(), b.params.tolist()):
            top, left, ch, cw = p[:4]
            assert (rh, rw) == (256, 256) and 0 <= top and 0 <= left and top + ch <= h and left + cw <= w
            assert abs(math.degrees(math.atan2(p[5], p[4]))) <= 10.0 + 1e-4


def test_native_and_python_prefetch_agree_on_ragged_batches(mixed_root):
    if not ops.available():
        pytest.skip("native extension not built")
    for train in (True, False):
        dm = DataManager(mixed_root, 3, train=train, pipeline="fused", seed=4)
        ld = dm.get_loader()
        assert ld._pf is not None
        ld.set_epoch(1)
        nat = [(b.data_u8.clone(), b.geom.clone(), b.labels.clone(), b.params.clone()) for b in ld]
        ld._pf, keep = None, ld._pf
        ld.set_epoch(1)
        py = [(b.data_u8.clone(), b.geom.clone(), b.labels.clone(), b.params.clone()) for b in ld]
        ld._pf = keep
        assert len(nat) == len(py) == math.ceil(len(dm.samples) / 3)
        for a, b in zip(nat, py):
            assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and torch.equal(a[2], b[2])
            if not train:
                assert torch.equal(a[3], b[3])
        # an abandoned iteration does not dead-lock the worker
        it = iter(ld)
        next(it)
        del it
        assert sum(len(b.labels) for b in ld) == len(dm.samples)


def test_ragged_native_prefetcher_draws_todays_parameters_on_a_uniform_split(synth_root):
    """On a uniform 128^2 split, the ragged mode of the native prefetcher draws exactly the
    parameters the uniform mode draws, sample for sample."""
    if not ops.available():
        pytest.skip("native extension not built")
    dm = DataManager(synth_root, 5, train=True, seed=3)
    cache = dm.cache
    assert not cache.ragged
    uniform = _FusedLoader(cache, 5, True, None, True, 3, pin=False)
    uniform.set_epoch(2)
    want = [(b.images_u8.clone(), b.params.clone(), b.labels.clone()) for b in uniform]
    # the same images as a ragged cache
    n = cache.images.shape[0]
    cache.ragged, cache.flat = True, cache.images.reshape(-1)
    cache.hw = torch.tensor([[128, 128]] * n, dtype=torch.int64)
    cache.offsets = torch.arange(n, dtype=torch.int64) * 128 * 128 * 3
    ragged = _FusedLoader(cache, 5, True, None, True, 3, pin=False)
    ragged.set_epoch(2)
    got = [(b.data_u8.clone(), b.params.clone(), b.labels.clone(), b.geom.clone()) for b in ragged]
    assert len(got) == len(want)
    for (img, par, lab), (data, par2, lab2, geom) in zip(want, got):
        assert torch.equal(par, par2) and torch.equal(lab, lab2)
        assert torch.equal(img.reshape(-1), data)
        assert geom[:, 0].tolist() == [i * 128 * 128 * 3 for i in range(len(lab))]


def test_uniform_small_splits_keep_the_fused_batch(synth_root, tmp_path):
    dm = DataManager(synth_root, 4, train=True, pipeline="fused")
    assert not dm.cache.ragged and isinstance(next(iter(dm.get_loader())), FusedBatch)
    # one size larger than 256: ragged under auto as well, resampled as Pillow does
    root = str(tmp_path / "big")
    for split in ("TrainData", "ValidationData"):
        for cls in ("a", "b"):
            d = os.path.join(root, split, cls)
            os.makedirs(d)
            for i in range(3):
                Image.fromarray(_textured(300, 400, i)).save(os.path.join(d, "%d.png" % i))
    dm = DataManager(root, 4, train=True, pipeline="auto")
    assert dm.pipeline == "fused" and isinstance(next(iter(dm.get_loader())), RaggedBatch)


def test_ragged_cache_refuses_mixed_sizes_when_asked_and_checks_the_budget(mixed_root):
    samples = DataManager(mixed_root, 4, pipeline="reference").samples
    with pytest.raises(CacheUnavailable, match="mixed"):
        DecodedCache(samples, allow_mixed=False)
    need = sum(_pil_rgb(p).size for p, _ in samples)
    with pytest.raises(CacheUnavailable, match="budget"):
        DecodedCache(samples, max_bytes=need - 1)
    c = DecodedCache(samples, max_bytes=need)
    assert c.ragged and c.flat.numel() == need
    for i, (p, _) in enumerate(samples):
        h, w = c.hw[i].tolist()
        off = int(c.offsets[i])
        assert np.array_equal(c.flat[off:off + h * w * 3].numpy().reshape(h, w, 3), _pil_rgb(p))
