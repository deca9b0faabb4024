"""What the network input size costs: VGG-F, batch 64, Adam, synthetic data, on one GPU.

Training: one engine per crop C in {128, 160, 176, 192, 224} (--train-crop-size), each fed uint8 batches whose
RandomResizedCrop size is C * 256 / 224 rounded to a multiple of 8.  Evaluation: one engine per evaluation crop
C' in {224, 256, 288} (--val-crop-size; trained at 224).  The engines of each table alternate in one process
(device-timed blocks of steps, median of five), so that every size sees the same clocks and neighbours.  Also
printed per size: the convolution FLOPs per image relative to 224^2 (computed from the shapes, not measured)
and which layers run the 2x2 max-pool as a separate kernel (odd maps, or tiles the epilogue cannot pool).
Also printed: the pixel box and channel-tile width (conv_bn) the fprop / dgrad launchers pick for the odd maps
of crops 176, 200 and 232 (11^2, 25^2, 29^2), and with ``--layers`` only the kernel times of one 512 -> 512
layer at 11^2 (fprop, masked dgrad with its column sum): run it from a build with the power-of-two boxes and
from this one to compare the two.  Prints one JSON line; the card's name and power limit are read in the same run.

    python bench/resolution_bench.py [--batch 64] [--steps 10] [--repeats 5] [--layers]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

TRAIN_CROPS = (128, 160, 176, 192, 224)
EVAL_CROPS = (224, 256, 288)


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out or torch.cuda.get_device_name(0) + ", power limit unknown"


def _timed(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def _conv_flops(spec, hw):
    total, h = 0.0, hw
    for c in spec.convs:
        total += 2.0 * h * h * c.cout * 9 * c.cin
        if c.pool_after:
            h //= 2
    return total


def _alternate(fns, steps, repeats):
    for fn in fns.values():
        _timed(fn, 3)                                       # warm-up: every kernel of the pass
    times = {k: [] for k in fns}
    for _ in range(repeats):
        for k, fn in fns.items():                           # alternating
            times[k].append(_timed(fn, steps))
    return times


def _layer_times(ops, B, a, dev):
    """Median kernel time (ms, CUDA events over blocks of launches) of fprop and masked dgrad + column sum of a
    512 -> 512 convolution on 11 x 11 maps: the last block of VGG-F at crop 176."""
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(B, 11, 11, 512, device=dev, generator=g).to(torch.bfloat16)
    w = (torch.randn(512, 3, 3, 512, device=dev, generator=g) * 0.02).to(torch.bfloat16)
    bias = torch.zeros(512, device=dev)
    y = torch.empty_like(x)
    cs = torch.zeros(512, device=dev)
    C = ops.require()
    fns = {"fprop": lambda: C.conv_fprop(x, w, bias, y, True, 0),
           "dgrad_masked_colsum": lambda: C.conv_dgrad(x, w, x, y, cs, 0)}
    times = _alternate(fns, 50 * a.steps, a.repeats)
    box = list(C.conv_pixel_box(B, 11, 11)) if hasattr(C, "conv_pixel_box") else "make_tile (1, 1, 128)"
    return dict(batch=B, map="11x11", channels=512, box=box,
                kernel_ms={k: round(statistics.median(v), 4) for k, v in times.items()},
                blocks_ms={k: [round(t, 4) for t in v] for k, v in times.items()})


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=10, help="steps per timed block")
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--layers", action="store_true", help="only the kernel times of a 512-channel 11^2 layer")
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("resolution_bench measures on a GPU: none found")
    from distributed_vgg_f_b200 import ops
    from distributed_vgg_f_b200.data import transforms as T
    from distributed_vgg_f_b200.data.loader import FusedBatch
    from distributed_vgg_f_b200.data.synthetic import synthetic_uint8_batch
    from distributed_vgg_f_b200.engine.native_engine import NativeEngine
    from distributed_vgg_f_b200.models.vggf import vggf_spec

    ops.require()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    B, spec = a.batch, vggf_spec(3)
    if a.layers:
        print(json.dumps(dict(bench="resolution_bench layers", card=_card(), **_layer_times(ops, B, a, dev))))
        return 0
    C = ops.require()
    boxes = {"%dx%d" % (h, h): dict(box=list(C.conv_pixel_box(B, h, h)), conv_bn=C.conv_bn_choice(B, h, h, 512))
             for h in (11, 25, 29)} if hasattr(C, "conv_pixel_box") else None
    imgs, labels = synthetic_uint8_batch(B, 256, 3, seed=0)
    src, lab = torch.from_numpy(imgs).pin_memory(), torch.from_numpy(labels).pin_memory()
    init = NativeEngine(spec, device=dev, batch=B, lr=1e-4, seed=0).export_state()     # one set of weights for all

    def batch(train, resize):
        params = T.sample_train_params(B, 256, 256) if train else T.val_params(B, 256, 256)
        return FusedBatch(src, params.pin_memory(), lab, (resize, resize), None)

    base = _conv_flops(spec, 224)
    engines, fns, info = {}, {}, {}
    for c in TRAIN_CROPS:
        r = (c * 256 // 224 + 7) // 8 * 8
        eng = NativeEngine(spec, device=dev, batch=B, lr=1e-4, seed=0, init_state=init, input_hw=c)
        bt = batch(True, r)
        engines[c] = eng
        fns[c] = (lambda e=eng, b=bt: e.train_step(b))
        info[c] = dict(train_resize=r, conv_flops_vs_224=round(_conv_flops(spec, c) / base, 3),
                       separate_pool_layers=[spec.convs[i].name for i, m in enumerate(eng.pool_masks)
                                             if spec.convs[i].pool_after and m is None])
    times = _alternate(fns, a.steps, a.repeats)
    train_rows = [dict(crop=c, step_ms=round(statistics.median(times[c]), 3),
                       images_per_s=round(B / (statistics.median(times[c]) * 1e-3), 1),
                       blocks_ms=[round(v, 3) for v in times[c]], **info[c]) for c in TRAIN_CROPS]
    del engines, fns
    torch.cuda.empty_cache()
    engines, fns = {}, {}
    for c in EVAL_CROPS:
        eng = NativeEngine(spec, device=dev, batch=B, lr=1e-4, seed=0, init_state=init, input_hw=224, eval_hw=c)
        bt = batch(False, c * 256 // 224 // 8 * 8)
        engines[c] = eng
        fns[c] = (lambda e=eng, b=bt: e.eval_step(b))
    times = _alternate(fns, a.steps, a.repeats)
    eval_rows = [dict(crop=c, pass_ms=round(statistics.median(times[c]), 3),
                      images_per_s=round(B / (statistics.median(times[c]) * 1e-3), 1),
                      blocks_ms=[round(v, 3) for v in times[c]],
                      conv_flops_vs_224=round(_conv_flops(spec, c) / base, 3)) for c in EVAL_CROPS]
    res = dict(bench="resolution_bench", card=_card(), model="vggf", batch=B, optimizer="adam",
               steps_per_block=a.steps, repeats=a.repeats, train=train_rows, eval=eval_rows,
               odd_map_tiles_512ch=boxes)
    print(json.dumps(res))
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
