"""The streaming input pipeline on the GPU: the decode kernels (csrc/jpeg.cu) against Pillow bit for bit in mixed
batches and on guarded operands, the host entry's refusals, the engine's staged input through --pipeline stream
against --pipeline fused (plain, MixUp, CutMix, ten-crop views), and deterministic VGG-F training through both."""
import itertools
import os

import numpy as np
import pytest
import torch
from PIL import Image

from distributed_vgg_f_b200 import ops
from distributed_vgg_f_b200.config import DATA
from distributed_vgg_f_b200.data import transforms as T
from distributed_vgg_f_b200.data.folder import scan_image_folder
from distributed_vgg_f_b200.data.loader import DecodedCache, _FusedLoader, _StreamLoader
from guarded import guarded
from test_jpeg_stream_cpu import textured, write_corpus, write_mixed_folder

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(scope="module")
def corpus(tmp_path_factory):
    return write_corpus(str(tmp_path_factory.mktemp("jpeg_corpus_gpu")))


def _pillow_flat(paths, batch):
    """Pillow's decode of the batch's files at the batch's geometry offsets."""
    g = batch.geom
    out = torch.empty(batch.nbytes, dtype=torch.uint8)
    for i, p in enumerate(paths):
        off, h, w = (int(v) for v in g[i, :3])
        a = np.asarray(Image.open(p).convert("RGB"))
        assert a.shape == (h, w, 3), p
        out[off:off + h * w * 3] = torch.from_numpy(a.copy()).view(-1)
    return out


def _device_decode(batch):
    C = ops.require()
    planes = torch.empty(max(batch.coef.numel(), 1), dtype=torch.uint8, device=DEV)
    out = torch.full((batch.nbytes,), 7, dtype=torch.uint8, device=DEV)
    raw = batch.raw.to(DEV) if batch.raw.numel() else torch.zeros(1, dtype=torch.uint8, device=DEV)
    C.jpeg_decode(batch.coef.to(DEV), batch.quant.to(DEV), batch.desc.to(DEV), batch.geom.to(DEV), raw, planes, out,
                  batch.desc, batch.geom)
    return out.cpu()


def _stream(paths, mb, threads=4):
    return _StreamLoader([(p, 0) for p in paths], mb, False, None, False, 0, threads=threads)


def test_decode_kernels_equal_pillow_in_mixed_batches(corpus):
    """Every corpus file (every JPEG variant, PNGs, fallbacks) in batches of 16 with a ragged final batch."""
    mb = 16
    assert len(corpus) % mb
    ld = _stream(corpus, mb)
    n = 0
    for k, batch in enumerate(ld):
        paths = corpus[k * mb:(k + 1) * mb]
        want = _pillow_flat(paths, batch)
        got = _device_decode(batch)
        bad = (got != want).nonzero()
        assert bad.numel() == 0, "batch %d: %d bytes differ, first at %d" % (k, bad.numel(), int(bad[0]))
        assert torch.equal(got, batch.decode()), k              # the CPU reference agrees
        n += len(paths)
    assert n == len(corpus)


def _guarded_decode(batch):
    C = ops.require()
    blocks = batch.coef.numel() // 64
    coef = guarded((batch.coef.numel(),), (1,), torch.int16, 0, 0x7fff, DEV, batch.coef)
    quant = guarded(tuple(batch.quant.shape), (64, 1), torch.int32, 0, 0x7fffffff, DEV, batch.quant)
    raw = guarded((max(batch.raw.numel(), 1),), (1,), torch.uint8, 0, 255, DEV,
                  batch.raw if batch.raw.numel() else torch.zeros(1, dtype=torch.uint8))
    desc = guarded(tuple(batch.desc.shape), (batch.desc.shape[1], 1), torch.int32, 0, 0, DEV, batch.desc)
    geom = guarded(tuple(batch.geom.shape), (5, 1), torch.int64, 0, 0, DEV, batch.geom)
    planes = guarded((blocks * 64,), (1,), torch.uint8, 0, 255, DEV)
    out = guarded((batch.nbytes,), (1,), torch.uint8, 0, 7, DEV)
    ops_ = (coef, quant, raw, desc, geom, planes, out)
    for g in ops_:
        g.seal()
    C.jpeg_decode(coef.t, quant.t, desc.t, geom.t, raw.t, planes.t, out.t, batch.desc, batch.geom)
    torch.cuda.synchronize()
    for g, w, name in ((coef, (), "coef"), (quant, (), "quant"), (raw, (), "raw"), (desc, (), "desc"),
                       (geom, (), "geom"), (planes, (planes.t,), "planes"), (out, (out.t,), "out")):
        g.check(w, name)
    return out.t.cpu()


def test_decode_kernels_stay_inside_their_operands(corpus):
    pick = [p for p in corpus if any(s in os.path.basename(p) for s in ("17x33", "255x256", "1x1_", "1x1."))]
    ld = _stream(pick, len(pick))
    batch = next(iter(ld))
    assert {int(v) for v in batch.desc[:, 0]} == {0, 1, 3}
    assert torch.equal(_guarded_decode(batch), _pillow_flat(pick, batch))


def test_decode_refuses_inconsistent_descriptors(corpus):
    pick = [p for p in corpus if "17x33" in p][:6] + [p for p in corpus if p.endswith("png17x33.png")]
    batch = next(iter(_stream(pick, len(pick))))
    C = ops.require()
    coef, quant, desc, geom = (t.to(DEV) for t in (batch.coef, batch.quant, batch.desc, batch.geom))
    raw = batch.raw.to(DEV)
    planes = torch.empty(batch.coef.numel(), dtype=torch.uint8, device=DEV)
    out = torch.empty(batch.nbytes, dtype=torch.uint8, device=DEV)

    def call(coef=coef, quant=quant, desc=desc, geom=geom, raw=raw, planes=planes, out=out, dh=batch.desc,
             gh=batch.geom):
        C.jpeg_decode(coef, quant, desc, geom, raw, planes, out, dh, gh)

    call()
    torch.cuda.synchronize()

    def edit(t, i, j, v):
        t = t.clone()
        t[i, j] = v
        return t

    jp = int((batch.desc[:, 0] > 0).nonzero()[1])           # a JPEG after the first image
    rw = int((batch.desc[:, 0] == 0).nonzero()[0])
    cases = {
        "block start": dict(dh=edit(batch.desc, jp, 3, int(batch.desc[jp, 3]) + 1)),
        "block grid": dict(dh=edit(batch.desc, jp, 5, int(batch.desc[jp, 5]) + 1)),
        "quant row": dict(dh=edit(batch.desc, jp, 11, batch.quant.shape[0])),
        "components": dict(dh=edit(batch.desc, jp, 0, 2)),
        "sampling": dict(dh=edit(batch.desc, jp, 2, 3)),
        "raw offset": dict(dh=edit(batch.desc, rw, 4, batch.raw.numel())),
        "geometry past out": dict(gh=edit(batch.geom, len(pick) - 1, 0, int(batch.geom[-1, 0]) + 1)),
        "size vs grid": dict(gh=edit(batch.geom, jp, 1, int(batch.geom[jp, 1]) + 8)),
        "short coef": dict(coef=coef[:-64]),
        "short planes": dict(planes=planes[:-1]),
        "short out": dict(out=out[:-1]),
        "desc shape": dict(desc=desc[:1]),
        "host desc on device": dict(dh=desc),
        "host geom shape": dict(gh=batch.geom[:1]),
    }
    for name, kw in cases.items():
        with pytest.raises(RuntimeError, match="jpeg_decode: "):     # refused on the host, nothing launched
            call(**kw)
    torch.cuda.synchronize()


# ----------------------------------------------------------------------------------------- engine staging
@pytest.fixture(scope="module")
def mixed_folder(tmp_path_factory):
    return write_mixed_folder(str(tmp_path_factory.mktemp("stream_folder_gpu")), per_class=8)


def _engine(batch, hw, spec=None, **kw):
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine
    from distributed_vgg_f_b200.models.vggf import vggf_mini_spec

    return NativeEngine(spec or vggf_mini_spec(3), device=torch.device(DEV), batch=batch, lr=1e-3, seed=0,
                        input_hw=hw, eval_hw=hw, **kw)


def _loaders(folder, train, mb, mix, resize, crop):
    _, samples = scan_image_folder(os.path.join(folder, DATA.train_dir if train else DATA.val_dir))
    kw = dict(resize=resize, crop=crop, **mix)
    return (_FusedLoader(DecodedCache(samples, 4), mb, train, None, True, 1, **kw),
            _StreamLoader(samples, mb, train, None, True, 1, threads=4, **kw))


@pytest.mark.parametrize("mix", [{}, dict(mixup_alpha=0.4), dict(cutmix_alpha=1.0)], ids=["plain", "mixup", "cutmix"])
def test_staged_input_is_bit_identical_to_the_fused_pipeline(mixed_folder, mix):
    mb, hw = 5, 64
    fused, stream = _loaders(mixed_folder, True, mb, mix, 72, hw)
    ea, eb = _engine(mb, hw), _engine(mb, hw)
    n = 0
    for x, y in zip(fused, stream):
        b = ea._stage_input(x)
        assert eb._stage_input(y) == b
        torch.cuda.synchronize()
        assert torch.equal(ea.x_nhwc[:b].view(torch.int16), eb.x_nhwc[:b].view(torch.int16)), n
        assert torch.equal(ea.labels_dev[:b], eb.labels_dev[:b])
        assert (ea._mix is None) == (eb._mix is None) and ea._mix == eb._mix
        ea._release_input()
        eb._release_input()
        n += 1
    assert n == len(fused) and n * mb > len(fused.cache.labels)      # a ragged final batch


def test_ten_crop_views_are_bit_identical_to_the_fused_pipeline(mixed_folder):
    mb, hw = 5, 64
    fused, stream = _loaders(mixed_folder, False, mb, {}, 72, hw)
    views = T.tta_views("ten-crop")
    ea, eb = _engine(mb, hw), _engine(mb, hw)
    for x, y in itertools.islice(zip(fused, stream), 3):
        b = ea._stage_input(x, views)
        eb._stage_input(y, views)
        for i in range(len(views)):
            if i:
                ea._view_input(x, b, i, views)
                eb._view_input(y, b, i, views)
            torch.cuda.synchronize()
            assert torch.equal(ea.x_nhwc[:b].view(torch.int16), eb.x_nhwc[:b].view(torch.int16)), i
        ea._release_input()
        eb._release_input()


def test_deterministic_vggf_trains_identically_through_both_pipelines(tmp_path):
    """Ten --deterministic VGG-F steps at batch 32, 224^2: identical losses and weights from either pipeline."""
    from distributed_vgg_f_b200.models.vggf import vggf_spec

    rng = np.random.default_rng(4)
    root = str(tmp_path)
    for c in range(3):
        d = os.path.join(root, DATA.train_dir, "c%d" % c)
        os.makedirs(d)
        for i in range(107):
            h, w = (int(v) for v in rng.integers(120, 420, 2))
            im = textured(h, w, c * 1000 + i)
            if i % 4 == 3:
                im.save(os.path.join(d, "%d.png" % i))
            else:
                im.save(os.path.join(d, "%d.jpg" % i), quality=90, subsampling=["4:2:0", "4:2:2", "4:4:4"][i % 3])
    fused, stream = _loaders(root, True, 32, dict(mixup_alpha=0.2), 256, 224)
    results = []
    for ld in (fused, stream):
        eng = _engine(32, 224, spec=vggf_spec(3), deterministic=True)
        losses = [eng.train_step(b).clone() for b in itertools.islice(ld, 10)]
        eng.sync()
        results.append((torch.stack(losses), eng.p32.clone()))
        del eng
    assert len(results[0][0]) == 10 and bool(torch.isfinite(results[0][0]).all())
    assert torch.equal(results[0][0], results[1][0])
    assert torch.equal(results[0][1], results[1][1])
