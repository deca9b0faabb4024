"""Every size-dependent convolution and pooling launch the native engine can make, and one representative of
each class of them, read from the launchers' own choices (the extension's ``conv_plan``: host code, so the
enumeration runs without a GPU).

The domain is what ``NativeEngine`` accepts: the specs VGG-F (= VGG-16's convolutions), VGG-11, -13, -19 and
vggf-mini; every crop ``check_native_hw`` takes; every batch 1 ... 64 (each ragged final batch of the default
per-GPU batch of 64) and 128.  The layers are walked as the engine lays out its buffers: a floor-mode 2 x 2
max-pool after each ``pool_after`` convolution, the fused conv + pool wherever ``conv_pool_fusable`` allows it
(and the plain forward and the separate pool kernels too, which run when fusion is switched off), the adaptive
average pool on a final map other than 7 x 7.

A convolution launch's signature is what its kernel branches on: the kind, path and tile width, whether the
halo kernel keeps every weight tile resident, whether the pixel box spans several images, whether it fails to
divide W, H or N (partial boxes at the right, bottom or last image), whether it holds fewer pixels than the
tile has rows (stale shared-memory rows), and for wgrad whether the last split is short.  The conv0 and pooling
kernels have no tile choice; their signature is the map size, so every reachable map is one class.

Representatives: per signature the cheapest launch (fewest MACs; ties to the smallest N, H, W), and per (kind,
path) a launch at batch 64 on which every CTA takes at least RING_TILES tiles, so that every ring of shared-memory
slots wraps several times (the cheapest such; the one with the most tiles per CTA where none reaches it).  Not
the deepest launch of all: at 512^2 and batch 64 the float64 reference might not fit next to the operands.
The unit is the one each ring advances by.  In fprop and dgrad it is the output tile: the epilogue hand-off
and the halo kernel's A ring (2-3 slots) advance once per tile and channel chunk, while the k-block operand
ring (at most 8 stages) and the halo weight ring (at most 18 slots, one per tap and chunk) turn over within
every tile of 9 x Ca / 64 >= 9 k-blocks or stay resident.  In wgrad it is the 64-pixel tile, one k-block of
the <= 8-stage operand ring, so tiles_per_cta counts the k-blocks a CTA takes over all its work items.

The enumeration costs about 1.5 s per SM count; ``classes`` and ``representatives`` keep it per SM count for
the process.
"""
from __future__ import annotations

import collections
import functools
from typing import Dict, List, NamedTuple, Tuple

BATCHES = tuple(range(1, 65)) + (128,)
CONV_KINDS = ("fprop", "fprop_pool", "dgrad", "wgrad", "wgrad_partial")
OTHER_KINDS = ("conv0_fprop", "conv0_wgrad", "maxpool_fwd", "maxpool_relu_bwd", "unpool", "avgpool_fwd",
               "avgpool_bwd")
# Tiles per CTA that wrap every per-tile ring several times (see the module docstring for the unit).
RING_TILES = 32


class Launch(NamedTuple):
    kind: str
    N: int
    H: int
    W: int
    Cin: int      # pooling kinds: the channels, Cin == Cout
    Cout: int

    @property
    def macs(self) -> int:
        if self.kind in CONV_KINDS:
            return self.N * self.H * self.W * self.Cin * self.Cout * 9
        if self.kind.startswith("conv0"):
            return self.N * self.H * self.W * 27 * 64
        return self.N * self.H * self.W * self.Cout

    @property
    def name(self) -> str:
        return "%s-N%d-%dx%d-%dx%d" % (self.kind, self.N, self.H, self.W, self.Cin, self.Cout)


class Rep(NamedTuple):
    launch: Launch
    sig: tuple
    role: str     # "cheapest" or "ring"

    @property
    def name(self) -> str:
        return "%s-%s" % (self.role, self.launch.name)


def specs() -> Dict[str, object]:
    from distributed_vgg_f_b200.models import vggf as V

    return {"vggf": V.vggf_spec(3), "vgg11": V.vgg_spec(11), "vgg13": V.vgg_spec(13), "vgg19": V.vgg_spec(19),
            "vggf-mini": V.vggf_mini_spec(3)}


def crops() -> Tuple[int, ...]:
    from distributed_vgg_f_b200.engine.native_engine import NATIVE_HW_MAX, NATIVE_HW_MIN, NATIVE_HW_STEP

    return tuple(range(NATIVE_HW_MIN, NATIVE_HW_MAX + 1, NATIVE_HW_STEP))


def layer_shapes():
    """{(first, h, cin, cout, pool_after)} of every spec's layers at every crop, and {(h, channels)} of the
    final maps that go through the adaptive average pool."""
    layers, finals = set(), set()
    for spec in specs().values():
        for hw in crops():
            h = hw
            for i, c in enumerate(spec.convs):
                layers.add((i == 0, h, c.cin, c.cout, c.pool_after))
                if c.pool_after:
                    h //= 2
            if h != spec.pooled_hw:
                finals.add((h, spec.convs[-1].cout))
    return layers, finals


def launches(C) -> List[Launch]:
    """Every launch of the domain, once, in a fixed order."""
    layers, finals = layer_shapes()
    out = set()
    for N in BATCHES:
        for first, h, cin, cout, pool in layers:
            if first:
                out.add(Launch("conv0_fprop", N, h, h, 3, cout))
                out.add(Launch("conv0_wgrad", N, h, h, 3, cout))
            else:
                for kind in ("fprop", "dgrad", "wgrad", "wgrad_partial"):
                    out.add(Launch(kind, N, h, h, cin, cout))
                if pool and C.conv_pool_fusable(N, h, h):
                    out.add(Launch("fprop_pool", N, h, h, cin, cout))
                    out.add(Launch("unpool", N, h, h, cout, cout))
            if pool:
                out.add(Launch("maxpool_fwd", N, h, h, cout, cout))
                out.add(Launch("maxpool_relu_bwd", N, h, h, cout, cout))
        for h, c in finals:
            out.add(Launch("avgpool_fwd", N, h, h, c, c))
            out.add(Launch("avgpool_bwd", N, h, h, c, c))
    return sorted(out)


def signature(C, L: Launch, sms: int) -> tuple:
    if L.kind not in CONV_KINDS:
        return (L.kind, L.H, L.W)
    p = C.conv_plan(L.kind, L.N, L.H, L.W, L.Cin, L.Cout, sms)
    wb, hb, nb = p["box"]
    rows = 64 if L.kind.startswith("wgrad") else 128
    return (L.kind, p["path"], p["bn"], p["resident"], nb > 1, L.W % wb != 0, L.H % hb != 0, L.N % nb != 0,
            wb * hb * nb < rows, p["tiles"] % p["tiles_per_split"] != 0)


SIG_FIELDS = ("kind", "path", "bn", "resident", "Nb>1", "W edge", "H edge", "N edge", "short box", "short split")


def tiles_per_cta(C, L: Launch, sms: int) -> int:
    """The most tiles (fprop / dgrad: output tiles; wgrad: pixel tiles of its work items) one CTA takes."""
    p = C.conv_plan(L.kind, L.N, L.H, L.W, L.Cin, L.Cout, sms)
    if L.kind in ("fprop", "fprop_pool", "dgrad"):
        cn = L.Cin if L.kind == "dgrad" else L.Cout
        work, depth = p["tiles"] * -(-cn // p["bn"]), 1
    elif p["path"] == "wgrad_halo64":
        work, depth = -(-L.Cout // 64) * p["ksplit"], p["tiles_per_split"]
    else:
        work, depth = -(-L.Cout // 128) * -(-L.Cin // p["bn"]) * 9 * p["ksplit"], p["tiles_per_split"]
    return -(-work // min(work, sms)) * depth


def _cost(L: Launch):
    return (L.macs, L.N, L.H, L.W, L)


def _ext():
    from distributed_vgg_f_b200 import ops

    return ops.require()


@functools.lru_cache(maxsize=None)
def classes(sms: int) -> Dict[tuple, Tuple[Launch, ...]]:
    """signature -> its launches, for ``sms`` SMs (computed once per process; do not modify)."""
    C = _ext()
    out = collections.defaultdict(list)
    for L in launches(C):
        out[signature(C, L, sms)].append(L)
    return {sig: tuple(ls) for sig, ls in out.items()}


@functools.lru_cache(maxsize=None)
def representatives(sms: int) -> Tuple[Rep, ...]:
    return pick_representatives(_ext(), sms, classes(sms))


def pick_representatives(C, sms: int, cls: Dict[tuple, Tuple[Launch, ...]]) -> Tuple[Rep, ...]:
    reps = [Rep(min(ls, key=_cost), sig, "cheapest") for sig, ls in sorted(cls.items(), key=lambda kv: repr(kv[0]))]
    by_path = collections.defaultdict(list)
    for sig, ls in cls.items():
        if sig[0] in CONV_KINDS:
            by_path[sig[:2]].extend((L, sig) for L in ls if L.N == 64)
    taken = {r.launch for r in reps}
    for key in sorted(by_path):
        cands = [(tiles_per_cta(C, L, sms), L, sig) for L, sig in by_path[key]]
        deep = [c for c in cands if c[0] >= RING_TILES]
        _, L, sig = min(deep, key=lambda c: _cost(c[1])) if deep else \
            max(cands, key=lambda c: (c[0], tuple(-v for v in _cost(c[1])[:4])))
        if L not in taken:
            reps.append(Rep(L, sig, "ring"))
            taken.add(L)
    return tuple(reps)


def table(cls: Dict[tuple, Tuple[Launch, ...]], reps: Tuple[Rep, ...]) -> str:
    """One row per convolution class (kind, path, width, flags: its launch count and representative), then the
    map classes of the other kinds per kind."""
    cheapest = {r.sig: r.launch for r in reps if r.role == "cheapest"}
    rows = ["%-13s %-12s %4s %5s %5s %6s %6s %6s %5s %5s %8s  %s" %
            (SIG_FIELDS + ("launches", "representative"))]
    flag = lambda v: "x" if v else "."
    for sig in sorted((s for s in cls if s[0] in CONV_KINDS), key=repr):
        rows.append("%-13s %-12s %4d %5s %5s %6s %6s %6s %5s %5s %8d  %s" %
                    ((sig[0], sig[1], sig[2]) + tuple(flag(v) for v in sig[3:]) + (len(cls[sig]), cheapest[sig].name)))
    per_kind = collections.Counter(s[0] for s in cls if s[0] not in CONV_KINDS)
    for kind in OTHER_KINDS:
        maps = sorted(s[1] for s in cls if s[0] == kind)
        rows.append("%-16s %3d maps: %s" % (kind, per_kind[kind], " ".join(str(m) for m in maps)))
    return "\n".join(rows)
