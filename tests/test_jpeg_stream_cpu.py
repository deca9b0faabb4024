"""The streaming input pipeline (--pipeline stream) without a GPU: the native header scan against PIL, the entropy
decoder + CPU reference (data/jpeg.py) against Pillow's decode bit for bit, errors that name the file, the stream
loader against the fused loader over a ragged cache batch for batch, and CLI runs with a cache budget below the
split's size.  Every fixture is generated from a seed with PIL."""
import contextlib
import io
import itertools
import json
import os

import numpy as np
import pytest
import torch
from PIL import Image

from distributed_vgg_f_b200 import ops
from distributed_vgg_f_b200.config import DATA
from distributed_vgg_f_b200.data import jpeg as J
from distributed_vgg_f_b200.data.loader import DecodedCache, JpegBatch, _FusedLoader, _StreamLoader
from distributed_vgg_f_b200.data.sampler import ShardedSampler

pytestmark = pytest.mark.skipif(not ops.available(), reason="needs the native extension")

# (H, W).  Widths 1-6 and 64 x 3 / 1 x 64 cover chroma at most two samples wide (replicated, not fancy-upsampled)
# and the first widths that are fancy-upsampled; heights 1-6 the vertical edges of 4:2:0.
SIZES = [(1, 1), (3, 4), (2, 5), (5, 6), (6, 2), (4, 3), (1, 64), (64, 3), (7, 9), (8, 8), (16, 16), (17, 33),
         (255, 256), (500, 375), (1023, 769)]
KIND_OTHER, KIND_JPEG, KIND_PNG = 0, 1, 2


def textured(h, w, seed):
    """A photo-like RGB image: gradients, a product pattern and noise."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    a = np.stack([(x * 7 + y * 3) % 256, (x * y) % 256, (255 - x * 5) % 256], -1).astype(np.float64)
    a += rng.normal(0, 40, a.shape)
    return Image.fromarray(np.clip(a, 0, 255).astype(np.uint8))


def write_corpus(d):
    """Every variant the issue names: sizes x quality x subsampling, grey, optimised tables, restart intervals,
    and the fallback kinds (progressive, RGB-coded, CMYK, PNG).  Returns the paths."""
    os.makedirs(d, exist_ok=True)
    files = []

    def save(name, im, **kw):
        p = os.path.join(d, name)
        im.save(p, **kw)
        files.append(p)

    for n, ((h, w), q, ss) in enumerate(itertools.product(SIZES, [50, 75, 90, 95, 100], ["4:4:4", "4:2:2", "4:2:0"])):
        save("s%dx%d_q%d_%s.jpg" % (h, w, q, ss.replace(":", "")), textured(h, w, n), quality=q, subsampling=ss)
    for n, (h, w) in enumerate(SIZES):
        im = textured(h, w, 1000 + n)
        save("grey%dx%d.jpg" % (h, w), im.convert("L"), quality=85)
        save("opt%dx%d.jpg" % (h, w), im, quality=85, optimize=True, subsampling="4:2:2")
        save("rstb%dx%d.jpg" % (h, w), im, quality=85, restart_marker_blocks=3)
        save("rstr%dx%d.jpg" % (h, w), im, quality=85, restart_marker_rows=1, subsampling="4:2:0")
        save("prog%dx%d.jpg" % (h, w), im, quality=85, progressive=True)
        save("rgb%dx%d.jpg" % (h, w), im, quality=85, keep_rgb=True)
        save("cmyk%dx%d.jpg" % (h, w), im.convert("CMYK"), quality=85)
        save("png%dx%d.png" % (h, w), im)
    return files


@pytest.fixture(scope="module")
def corpus(tmp_path_factory):
    return write_corpus(str(tmp_path_factory.mktemp("jpeg_corpus")))


def pil_kind(path):
    """What the stream pipeline should do with a file, from what PIL reports about it."""
    with Image.open(path) as im:
        if im.format == "PNG":
            return KIND_PNG
        if im.format != "JPEG" or im.info.get("progressive") or im.mode not in ("L", "RGB"):
            return KIND_OTHER
        layer = im.layer
        if im.mode == "L":
            return KIND_JPEG
        ids = [l[0] for l in layer]
        if ids == [82, 71, 66] or im.info.get("adobe_transform", 1) == 0:
            return KIND_OTHER
        hv = [(l[1], l[2]) for l in layer]
        return KIND_JPEG if hv[0] in ((1, 1), (2, 1), (2, 2)) and hv[1] == hv[2] == (1, 1) else KIND_OTHER


def descriptor(row):
    """The batch descriptor of a lone image (its blocks from 0, its tables in rows 0..2)."""
    n, H, W = int(row[4]), int(row[1]), int(row[2])
    d = np.zeros(J.DESC_DIM, np.int32)
    d[0], d[1], d[2] = n, (row[5] if n == 3 else 1), (row[6] if n == 3 else 1)
    for c in range(n):
        if n == 1:
            bw, bh = -(-W // 8), -(-H // 8)
        else:
            bw, bh = -(-W // (8 * d[1])) * int(row[5 + 2 * c]), -(-H // (8 * d[2])) * int(row[6 + 2 * c])
        d[5 + c], d[8 + c], d[11 + c] = bw, bh, c
    return d


def reference_decode(path, row):
    coef, quant = ops.require().jpeg_entropy_decode(path, row)
    return J.decode_image(descriptor(row), int(row[1]), int(row[2]), coef.numpy(), quant.numpy(),
                          np.zeros(0, np.uint8))


# ------------------------------------------------------------------------------------------- header scan
def test_scan_gives_pil_size_and_kind(corpus):
    rows = ops.require().jpeg_scan(corpus, 8)
    assert {int(r[0]) for r in rows} == {KIND_OTHER, KIND_JPEG, KIND_PNG}
    for p, r in zip(corpus, rows):
        with Image.open(p) as im:
            w, h = im.size
            layer = getattr(im, "layer", None)
        assert (int(r[1]), int(r[2])) == (h, w), p
        assert int(r[0]) == pil_kind(p), p
        if int(r[0]) == KIND_JPEG:
            assert int(r[4]) == len(layer), p
            assert [(int(r[5 + 2 * c]), int(r[6 + 2 * c])) for c in range(len(layer))] == \
                [(l[1], l[2]) for l in layer], p


def test_scan_of_unreadable_and_foreign_files(tmp_path):
    gif = str(tmp_path / "a.gif")
    textured(5, 6, 0).save(gif)
    junk = str(tmp_path / "junk.jpg")
    open(junk, "wb").write(b"\xff\xd8\xff\xe0garbage")
    rows = ops.require().jpeg_scan([gif, junk, str(tmp_path / "missing.jpg")], 2)
    assert rows[:, 0].tolist() == [KIND_OTHER] * 3


# ---------------------------------------------------------------------------------------- exact decode
def test_entropy_decode_and_reference_equal_pillow(corpus):
    rows = ops.require().jpeg_scan(corpus, 8)
    n = 0
    for p, r in zip(corpus, rows):
        if int(r[0]) != KIND_JPEG:
            continue
        ref = np.asarray(Image.open(p).convert("RGB"))
        got = reference_decode(p, r)
        assert got.shape == ref.shape and np.array_equal(got, ref), p
        n += 1
    assert n == len(SIZES) * (15 + 4)


def test_reference_idct_range_limit_wraps_as_libjpeg():
    # a lone DC coefficient: (dc * q + 4) >> 3 after both passes, then libjpeg's range-limit table
    q = np.ones((1, 64), np.int32)
    for dc, want in ((0, 128), (8 * 127, 255), (8 * 128, 255), (-8 * 128, 0), (-8 * 129, 0), (8 * 600, 0),
                     (-8 * 600, 255)):
        c = np.zeros((1, 64), np.int16)
        c[0, 0] = dc
        assert (J.idct_islow(c, q) == want).all(), dc


# ----------------------------------------------------------------------------------------------- errors
def _sos_data_start(b):
    i = b.index(b"\xff\xda")
    return i + 2 + int.from_bytes(b[i + 2:i + 4], "big")


def _dht_tables(b):
    """(offset of the BITS counts, class, value count) of every Huffman table of a JPEG's DHT segments."""
    out, i = [], 0
    while True:
        i = b.find(b"\xff\xc4", i)
        if i < 0 or i >= _sos_data_start(b):
            return out
        end, q = i + 2 + int.from_bytes(b[i + 2:i + 4], "big"), i + 4
        while q < end:
            n = sum(b[q + 1:q + 17])
            out.append((q + 1, b[q] >> 4, n))
            q += 17 + n
        i = end


def broken_files(d):
    """(path, what) of a truncated file; of tables that over-subscribe a code length (three codes of length 1, and
    an AC table's 162 codes all declared at length 1, which a lookahead filled before the check would write far
    past); of a table with an all-ones code; and of entropy data that starts with a code no table holds."""
    src = io.BytesIO()
    textured(64, 80, 3).save(src, format="JPEG", quality=90)
    b = src.getvalue()
    out = []

    def write(name, data, what):
        p = os.path.join(d, name)
        open(p, "wb").write(bytes(data))
        out.append((p, what))

    write("truncated.jpg", b[:_sos_data_start(b) + (len(b) - _sos_data_start(b)) // 2], "truncated")
    tables = _dht_tables(b)
    dc = next(t for t in tables if t[1] == 0 and t[2] == 12)
    ac = next(t for t in tables if t[1] == 1 and t[2] == 162)
    bad = bytearray(b)
    bad[dc[0]:dc[0] + 16] = bytes([3] + [0] * 8 + [9] + [0] * 6)          # three codes of length 1
    write("corrupt.jpg", bad, "Huffman table")
    bad = bytearray(b)
    bad[ac[0]:ac[0] + 16] = bytes([162] + [0] * 15)                       # 162 codes of length 1
    write("corrupt_ac.jpg", bad, "Huffman table")
    bad = bytearray(b)
    bad[dc[0]:dc[0] + 16] = bytes([1] * 10 + [2] + [0] * 5)               # 11111111111 is a code
    write("all_ones.jpg", bad, "Huffman table")
    s = _sos_data_start(b)
    write("badcode.jpg", b[:s] + b"\xff\x00" * 32 + b[s + 64:], "bad Huffman code")
    return out


def test_malformed_files_raise_with_their_path(tmp_path):
    C = ops.require()
    for p, what in broken_files(str(tmp_path)):
        row = C.jpeg_scan([p], 1)[0]
        assert int(row[0]) == KIND_JPEG, p            # the headers are fine: the data is not
        with pytest.raises(RuntimeError, match=what) as e:
            C.jpeg_entropy_decode(p, row)
        assert p in str(e.value)
        if what != "bad Huffman code":                # libjpeg only warns about a bad code and decodes on
            with pytest.raises(OSError):
                Image.open(p).convert("RGB")


def test_stream_loader_raises_a_worker_error_in_next(tmp_path):
    files = []
    for i in range(6):
        p = str(tmp_path / ("%d.jpg" % i))
        textured(40 + i, 50, i).save(p, quality=90)
        files.append(p)
    (bad, _), = broken_files(str(tmp_path))[:1]
    samples = [(p, 0) for p in files[:4]] + [(bad, 0)] + [(p, 0) for p in files[4:]]
    ld = _StreamLoader(samples, 2, False, None, False, 0, threads=3)
    got = []
    with pytest.raises(RuntimeError, match="truncated") as e:
        for batch in ld:
            got.append(batch.labels.numel())
    assert bad in str(e.value)
    assert got == [2, 2]                              # the batches before the bad one arrive first


def short_palette_png(path):
    """An 8-bit palette PNG whose PLTE is shorter than its largest index: PIL reads the missing entries as black,
    csrc/png_decode.cpp refuses the file."""
    import struct
    import zlib

    im = Image.fromarray((np.arange(20 * 30).reshape(20, 30) % 21).astype(np.uint8), mode="P")
    im.putpalette(list(range(63)))
    buf = io.BytesIO()
    im.save(buf, format="PNG")
    b = buf.getvalue()
    i = b.index(b"PLTE") - 4
    n = int.from_bytes(b[i:i + 4], "big")
    data = b[i + 8:i + 8 + n][:30]
    chunk = struct.pack(">I", len(data)) + b"PLTE" + data + struct.pack(">I", zlib.crc32(b"PLTE" + data))
    open(path, "wb").write(b[:i] + chunk + b[i + 12 + n:])


def test_pngs_the_native_decoder_refuses_go_to_pil(tmp_path):
    bad = str(tmp_path / "short_plte.png")
    short_palette_png(bad)
    assert int(ops.require().jpeg_scan([bad], 1)[0, 0]) == KIND_PNG          # its IHDR looks fine
    samples = [(bad, 0)]
    for i in range(5):
        p = str(tmp_path / ("%d.%s" % (i, "png" if i % 2 else "jpg")))
        textured(30 + 7 * i, 40, i).save(p)
        samples.append((p, i % 2))
    a = _FusedLoader(DecodedCache(samples, 2), 4, True, None, True, 0)
    b = _StreamLoader(samples, 4, True, None, True, 0, threads=2)
    assert b.other_count == 1 and int(b.cache.headers[0, 0]) == KIND_OTHER
    _same_batches(a, b)


def test_start_up_budget_is_checked_before_anything_is_decoded(tmp_path, monkeypatch):
    from distributed_vgg_f_b200.data import loader

    samples = []
    for i, kw in enumerate([dict(progressive=True), dict(keep_rgb=True)]):
        p = str(tmp_path / ("%d.jpg" % i))
        textured(50, 60, i).save(p, quality=90, **kw)
        samples.append((p, 0))
    gif = str(tmp_path / "g.gif")
    textured(20, 30, 5).save(gif)
    samples.append((gif, 0))
    need = (2 * 50 * 60 + 20 * 30) * 3

    def no_decode(path):
        raise AssertionError("decoded %s before the budget check" % path)

    monkeypatch.setattr(loader, "_decode", no_decode)
    with pytest.raises(loader.CacheUnavailable, match="3 files"):
        _StreamLoader(samples, 2, False, None, False, 0, threads=2, max_bytes=need - 1)
    monkeypatch.undo()
    ld = _StreamLoader(samples, 2, False, None, False, 0, threads=2, max_bytes=need)
    assert (ld.other_count, ld.other_bytes) == (3, need)
    got = torch.cat([b.decode() for b in ld])
    want = torch.cat([torch.from_numpy(np.asarray(Image.open(p).convert("RGB")).copy()).view(-1) for p, _ in samples])
    assert torch.equal(got, want)


def test_files_pil_cannot_read_are_refused_at_start_up(tmp_path):
    p = str(tmp_path / "junk.jpg")
    open(p, "wb").write(b"not an image at all")
    with pytest.raises(Exception, match="junk.jpg"):
        _StreamLoader([(p, 0)], 1, False, None, False, 0, threads=1)


# --------------------------------------------------------------------------- loader: same batches as fused
def write_mixed_folder(root, seed=0, per_class=7):
    """A two-split ImageFolder of mixed sizes and kinds: baseline JPEGs of every sampling, grey, restart
    intervals, PNGs and progressive JPEGs (decoded by PIL at start-up)."""
    rng = np.random.default_rng(seed)
    n = 0
    for split in (DATA.train_dir, DATA.val_dir):
        for c in range(3):
            os.makedirs(os.path.join(root, split, "c%d" % c), exist_ok=True)
            for i in range(per_class):
                h, w = (int(v) for v in rng.integers(20, 300, 2))
                im, base = textured(h, w, n), os.path.join(root, split, "c%d" % c, "%d" % i)
                n += 1
                k = n % 6
                if k == 0:
                    im.save(base + ".jpg", quality=90, subsampling="4:2:0")
                elif k == 1:
                    im.save(base + ".png")
                elif k == 2:
                    im.save(base + ".jpg", quality=85, progressive=True)
                elif k == 3:
                    im.convert("L").save(base + ".jpg", quality=75)
                elif k == 4:
                    im.save(base + ".jpg", quality=95, subsampling="4:2:2", restart_marker_blocks=2)
                else:
                    im.save(base + ".jpg", quality=100, subsampling="4:4:4")
    return root


@pytest.fixture(scope="module")
def mixed_folder(tmp_path_factory):
    return write_mixed_folder(str(tmp_path_factory.mktemp("stream_folder")))


def _same_batches(a, b, epochs=2):
    for ep in range(epochs):
        a.set_epoch(ep)
        b.set_epoch(ep)
        n = 0
        for x, y in zip(a, b):
            assert isinstance(y, JpegBatch)
            assert torch.equal(x.geom, y.geom) and torch.equal(x.params, y.params), (ep, n)
            assert torch.equal(x.labels, y.labels) and x.mix == y.mix, (ep, n)
            assert torch.equal(x.data_u8, y.decode()), (ep, n)
            n += 1
        assert n == len(a) == len(b)
    return n


@pytest.mark.parametrize("train", [True, False])
@pytest.mark.parametrize("world", [1, 2])
@pytest.mark.parametrize("threads", [1, 8])
def test_stream_loader_yields_the_fused_loaders_batches(mixed_folder, train, world, threads):
    from distributed_vgg_f_b200.data.folder import scan_image_folder

    _, samples = scan_image_folder(os.path.join(mixed_folder, DATA.train_dir if train else DATA.val_dir))
    cache = DecodedCache(samples, 4)
    assert cache.ragged
    mb = 4                                  # 21 images: a ragged final batch at world 1 and 2
    for rank in range(world):
        def sampler():
            return ShardedSampler(len(samples), world, rank, seed=0) if world > 1 else None
        mix = dict(mixup_alpha=0.2, cutmix_alpha=1.0) if train else {}
        a = _FusedLoader(cache, mb, train, sampler(), True, 0, resize=72, crop=64, **mix)
        b = _StreamLoader(samples, mb, train, sampler(), True, 0, threads=threads, resize=72, crop=64, **mix)
        assert b.other_count == sum(1 for p, _ in samples if pil_kind(p) == KIND_OTHER) > 0
        _same_batches(a, b)


def test_jpeg_batch_to_float_equals_the_ragged_batch(mixed_folder):
    from distributed_vgg_f_b200.data.folder import scan_image_folder

    _, samples = scan_image_folder(os.path.join(mixed_folder, DATA.train_dir))
    a = _FusedLoader(DecodedCache(samples, 4), 5, True, None, True, 3, resize=72, crop=64)
    b = _StreamLoader(samples, 5, True, None, True, 3, threads=4, resize=72, crop=64)
    for x, y in itertools.islice(zip(a, b), 2):
        assert torch.equal(x.to_float(out_hw=64)[0], y.to_float(out_hw=64)[0])


def test_stream_slot_is_sized_from_the_headers(mixed_folder):
    from distributed_vgg_f_b200.data.folder import scan_image_folder

    _, samples = scan_image_folder(os.path.join(mixed_folder, DATA.train_dir))
    ld = _StreamLoader(samples, 4, True, None, True, 0, threads=2)
    h = ld.cache.headers
    jpeg = h[:, 0] == KIND_JPEG
    assert ld._coef.shape[1] == int((h[jpeg, 11] * 64).sort(descending=True).values[:4].sum())
    rgb = ld.cache.hw[~jpeg, 0] * ld.cache.hw[~jpeg, 1] * 3
    assert ld._raw.shape[1] == int(rgb.sort(descending=True).values[:4].sum())


# --------------------------------------------------------------------------------------------- CLI runs
BASE = ["-iu", "tcp://127.0.0.1:29998", "-rn", "0", "-ws", "1", "-nc", "-mb", "4", "--model", "vggf-tiny",
        "--engine", "oracle", "-ep", "1", "--train-crop-size", "64", "--val-crop-size", "64",
        "--train-resize-size", "72", "--val-resize-size", "72"]


def _main(argv):
    from distributed_vgg_f_b200 import cli

    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        assert cli.main(argv) == 0
    return buf.getvalue()


def test_flags_parse():
    from distributed_vgg_f_b200 import cli

    a = cli.parse_command_line(["-iu", "x", "-rn", "0", "-ws", "1", "-rd", "/r"], init=False)
    assert a.pipeline == "auto" and a.decode_threads == 8
    a = cli.parse_command_line(["-iu", "x", "-rn", "0", "-ws", "1", "-rd", "/r", "--pipeline", "stream",
                                "--decode-threads", "3"], init=False)
    assert a.pipeline == "stream" and a.decode_threads == 3


def _decoded_bytes(folder, split, kinds):
    d = os.path.join(folder, split)
    return sum(h * w * 3 for p in (os.path.join(r, f) for r, _, fs in os.walk(d) for f in fs) if pil_kind(p) in kinds
               for w, h in [Image.open(p).size])


def test_cli_streams_a_split_larger_than_the_cache_budget(mixed_folder, tmp_path, monkeypatch):
    splits = (DATA.train_dir, DATA.val_dir)
    fallback_bytes = max(_decoded_bytes(mixed_folder, s, (KIND_OTHER,)) for s in splits)
    budget = fallback_bytes + 1              # room for the start-up decodes, not for either split
    assert all(_decoded_bytes(mixed_folder, s, (KIND_OTHER, KIND_JPEG, KIND_PNG)) > budget for s in splits)
    monkeypatch.setenv("B200_MAX_CACHE_GB", repr(budget / 2**30))
    log = str(tmp_path / "log.jsonl")
    text = _main(BASE + ["-rd", mixed_folder, "--pipeline", "stream", "--decode-threads", "3", "--log-jsonl", log])
    fallback = sum(pil_kind(os.path.join(d, f)) == KIND_OTHER for d, _, fs in os.walk(mixed_folder) for f in fs)
    assert "[Info] input pipeline: stream (3 decode threads, %d file(s) decoded by PIL at start-up)" % fallback in text
    assert "reference) input pipeline" not in text
    assert "[Info] Epoch: 1/1" in text
    rec = json.loads(open(log).read().splitlines()[-1])
    assert rec["pipeline"] == "stream" and rec["decode_threads"] == 3 and rec["stream_fallback"] == fallback
    auto = _main(BASE + ["-rd", mixed_folder])
    assert "-> using the per-sample (reference) input pipeline" in auto
    assert "input pipeline: stream" not in auto


def test_stream_refuses_start_up_decodes_over_the_budget(mixed_folder, monkeypatch):
    from distributed_vgg_f_b200.data.loader import CacheUnavailable, DataManager

    budget = _decoded_bytes(mixed_folder, DATA.train_dir, (KIND_OTHER,)) - 1
    monkeypatch.setenv("B200_MAX_CACHE_GB", repr(budget / 2**30))
    with pytest.raises(CacheUnavailable, match="stream decoders do not take"):
        DataManager(mixed_folder, 4, train=True, pipeline="stream")
