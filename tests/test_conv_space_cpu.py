"""The reachable convolution launch space without a GPU: conv_plan's classes at 132 SMs (H100 SXM) and 114 (H100
PCIe), their representatives, and the launchers' other host-side choices that the engine relies on."""
import pytest

import conv_space as S
from distributed_vgg_f_b200 import ops

pytestmark = pytest.mark.skipif(not ops.available(), reason="needs the built extension (host code only)")
SMS = (132, 114)


@pytest.fixture(scope="module", params=SMS)
def space(request):
    return ops.require(), request.param, S.classes(request.param), S.representatives(request.param)


def test_enumeration_is_deterministic(space):
    C, sms, cls, reps = space
    fresh = S.classes.__wrapped__(sms)
    assert fresh == cls
    assert S.pick_representatives(C, sms, fresh) == reps


def test_every_class_has_a_representative_with_its_signature(space, capsys):
    C, sms, cls, reps = space
    cheapest = {r.sig: r for r in reps if r.role == "cheapest"}
    assert set(cheapest) == set(cls)
    for r in reps:
        assert r.launch in cls[r.sig]
        assert S.signature(C, r.launch, sms) == r.sig, r.name
    for sig, ls in cls.items():
        assert cheapest[sig].launch == min(ls, key=lambda L: (L.macs, L.N, L.H, L.W, L))
    # every (kind, path) has a representative at batch 64 whose CTAs take the most tiles (or RING_TILES)
    for key in {s[:2] for s in cls if s[0] in S.CONV_KINDS}:
        most = max(S.tiles_per_cta(C, L, sms) for s, ls in cls.items() if s[:2] == key for L in ls if L.N == 64)
        assert any(r.sig[:2] == key and r.launch.N == 64 and
                   S.tiles_per_cta(C, r.launch, sms) >= min(most, S.RING_TILES) for r in reps), key
    with capsys.disabled():
        print("\n[conv space, %d SMs] %d launches, %d classes, %d representatives\n%s" %
              (sms, sum(len(v) for v in cls.values()), len(cls), len(reps), S.table(cls, reps)))


def test_partial_fill_boxes_are_reached_at_every_width(space):
    """FILL boxes that straddle the bottom edge or the last image, at every tile width, in fprop and dgrad."""
    _, _, cls, _ = space
    for kind in ("fprop", "dgrad"):
        fill = [s for s in cls if s[:2] == (kind, "fill")]
        for bn in (64, 128, 256):
            assert any(s[2] == bn and s[6] for s in fill), (kind, bn, "H edge")
            assert any(s[2] == bn and s[7] for s in fill), (kind, bn, "N edge")
            assert any(s[2] == bn and s[5] for s in fill), (kind, bn, "W edge")


@pytest.mark.parametrize("kind,N,H,Cin,Cout,want", [
    ("fprop", 64, 9, 512, 512, ("fill", 256, (2, 1, 64))),       # crop 144: W edge at width 256
    ("fprop", 64, 23, 256, 256, ("fill", 128, (8, 1, 16))),      # crop 184: W edge
    ("fprop", 64, 5, 512, 512, ("fill", 128, (5, 5, 5))),        # crop 80 / 88: the last box holds 4 images
    ("fprop", 1, 18, 128, 256, ("fill", 128, (18, 7, 1))),       # crop 72, batch 1: H edge
    ("dgrad", 17, 20, 64, 64, ("fill", 64, (7, 2, 9))),          # ragged batch 17: W and N edges
    ("fprop", 64, 11, 512, 512, ("fill", 256, (11, 11, 1))),
    ("fprop", 64, 25, 512, 512, ("fill", 256, (25, 5, 1))),
    ("fprop", 64, 56, 256, 256, ("pow2", 256, (8, 8, 2))),
    ("fprop", 64, 14, 512, 512, ("pow2", 128, (2, 2, 32))),
    ("fprop", 64, 224, 64, 64, ("halo", 64, (8, 16, 1))),
    ("fprop_pool", 64, 56, 128, 256, ("pow2", 256, (8, 8, 2))),
    ("wgrad", 64, 112, 64, 128, ("wgrad_halo64", 64, (8, 8, 1))),
    ("wgrad", 64, 28, 512, 512, ("wgrad", 256, (4, 4, 4))),
])
def test_conv_plan_at_known_shapes(kind, N, H, Cin, Cout, want):
    p = ops.require().conv_plan(kind, N, H, H, Cin, Cout, 132)
    assert (p["path"], p["bn"], tuple(p["box"])) == want


def test_halo_plan_reports_the_halo_tile_and_residency():
    C = ops.require()
    p = C.conv_plan("fprop", 64, 224, 224, 64, 64, 132)
    assert p["tiles"] == 64 * (224 // 8) * (224 // 16) and p["resident"]
    assert not C.conv_plan("fprop", 64, 224, 224, 64, 128, 132)["resident"]


def test_conv_plan_rejects_what_it_cannot_plan():
    C = ops.require()
    with pytest.raises(RuntimeError, match="kind"):
        C.conv_plan("fprop_relu", 1, 8, 8, 64, 64, 132)
    with pytest.raises(RuntimeError, match="positive"):
        C.conv_plan("fprop", 1, 8, 8, 64, 64, 0)
    with pytest.raises(RuntimeError, match="bn must be"):
        C.conv_plan("fprop", 1, 8, 8, 64, 64, 132, bn=96)


def test_an_explicit_width_is_planned_as_the_launcher_takes_it():
    """An explicit width keeps the pixel box, and any width takes a 64-channel wgrad off the halo64 kernel."""
    C = ops.require()
    auto = C.conv_plan("wgrad", 64, 28, 28, 256, 512, 132)
    wide = C.conv_plan("wgrad", 64, 28, 28, 256, 512, 132, bn=256)
    assert wide["bn"] == 256 and wide["box"] == auto["box"] == (4, 4, 4)
    assert C.conv_plan("wgrad", 64, 112, 112, 64, 128, 132, bn=64)["path"] == "wgrad"
    assert C.conv_plan("fprop", 64, 56, 56, 256, 256, 132, bn=128)["bn"] == 128


@pytest.mark.parametrize("sms", SMS)
def test_wgrad_splits_match_the_deterministic_plan(sms):
    """deterministic_plan (which sizes the --deterministic workspace through conv_wgrad_splits, a view of
    conv_plan) passes its batch and SM count through and walks the map sizes layer by layer as the engine does,
    so its split counts are the ones conv_plan gives each layer's wgrad_partial launch."""
    from distributed_vgg_f_b200.engine.native_engine import deterministic_plan

    C = ops.require()
    for spec in S.specs().values():
        for hw in S.crops()[::4] + (S.crops()[-1],):
            for b in (1, 17, 64):
                rows = {(name, what): splits for name, what, splits, _ in
                        deterministic_plan(spec, b, hw, sms, fused_head=False)}
                h = hw
                for i, c in enumerate(spec.convs):
                    if i > 0:
                        p = C.conv_plan("wgrad_partial", b, h, h, c.cin, c.cout, sms)
                        assert rows[(c.name, "wgrad")] == p["ksplit"], (hw, b, c.name)
                        assert p["ksplit"] == -(-p["tiles"] // p["tiles_per_split"])
                    if c.pool_after:
                        h //= 2


def test_pool_fusability_does_not_depend_on_the_batch():
    """The engine decides the fused pool once at its full batch B and launches it at every b <= B."""
    C = ops.require()
    layers, _ = S.layer_shapes()
    for h in sorted({h for first, h, _, _, pool in layers if pool and not first}):
        want = bool(C.conv_pool_fusable(64, h, h))
        for b in S.BATCHES:
            assert bool(C.conv_pool_fusable(b, h, h)) == want, (b, h)
