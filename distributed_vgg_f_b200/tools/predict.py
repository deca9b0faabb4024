"""Classify images with a checkpoint written by ``--save``.

The reference stops at the per-epoch validation line; this is the missing last step for a user who
trained a model: load the checkpoint (its ``args`` record the architecture and the input sizes), apply
the reference's validation transform (Resize 256 -> CenterCrop 224 -> Normalize, distributedVggf.py:103-108,
or the run's --val-resize-size / --val-crop-size; ``--resize`` / ``--crop`` override them) and print one
line per image::

    python -m distributed_vgg_f_b200.tools.predict ck.pt --classes edible,other,toy img1.png img2.png
    python -m distributed_vgg_f_b200.tools.predict ck.pt --data-root /data/coil3 /data/coil3/ValidationData/toy
    python -m distributed_vgg_f_b200.tools.predict ck.pt --ema img1.png      # the weights' moving average
    python -m distributed_vgg_f_b200.tools.predict ck.pt --tta ten-crop img1.png   # mean softmax of ten views

``--classes`` (or ``--data-root``, whose TrainData sub-folders define them) only names the outputs;
directories are expanded to the image files inside.  Runs on the GPU through the native engine when
one is present (``--engine auto``), else on the CPU oracle.
"""
from __future__ import annotations

import argparse
import os
from typing import List, Optional, Sequence

import torch

from ..config import DATA
from ..data.folder import IMG_EXTENSIONS, find_classes
from ..data.transforms import TTA_MODES, reference_transforms, tta_views
from ..models.vggf import build_oracle, get_spec
from ..utils.checkpoint import strip_module_prefix


def expand(paths: Sequence[str]) -> List[str]:
    out: List[str] = []
    for p in paths:
        if os.path.isdir(p):
            for dp, _, files in sorted(os.walk(p)):
                out += [os.path.join(dp, f) for f in sorted(files) if f.lower().endswith(IMG_EXTENSIONS)]
        else:
            out.append(p)
    return out


def eval_sizes(saved: dict):
    """(resize, crop) of the validation transform a run used, from the checkpoint's ``"args"`` (the reference's
    256 / 224 for a checkpoint that records none)."""
    return int(saved.get("val_resize_size") or DATA.resize), int(saved.get("val_crop_size") or DATA.crop)


def load_model(checkpoint: str, model: Optional[str] = None, num_classes: Optional[int] = None, ema: bool = False,
               with_args: bool = False):
    """(spec, torch-layout state) of a checkpoint; ``ema``: its moving average of the weights (--model-ema);
    ``with_args``: also the ``"args"`` the checkpoint's run recorded."""
    payload = torch.load(checkpoint, map_location="cpu", weights_only=True)
    if ema:
        if not isinstance(payload, dict) or "model_ema" not in payload:
            raise ValueError("%s holds no model EMA (it was not saved with --model-ema)" % checkpoint)
        state = strip_module_prefix({k: v for k, v in payload["model_ema"].items() if k != "n_averaged"})
    else:
        state = strip_module_prefix(payload["model"] if "model" in payload else payload)
    saved = payload.get("args", {}) if isinstance(payload, dict) else {}
    last = [k for k in state if k.endswith(".weight")][-1]
    classes = num_classes or int(state[last].shape[0])
    spec = get_spec(model or saved.get("model") or "vggf", classes)
    return (spec, state, saved) if with_args else (spec, state)


@torch.no_grad()
def predict(checkpoint: str, images: Sequence[str], model: Optional[str] = None, engine: str = "auto",
            batch: int = 32, ema: bool = False, resize: Optional[int] = None, crop: Optional[int] = None,
            tta: str = "none"):
    """Returns (logits [n, C] fp32 on the CPU, files).  ``resize`` / ``crop``: the validation transform's
    sizes (default: the ones recorded in the checkpoint).  ``tta`` (a --val-tta mode): every view's logits,
    [n, V, C]."""
    from PIL import Image

    spec, state, saved = load_model(checkpoint, model, ema=ema, with_args=True)
    files = expand(images)
    saved_resize, saved_crop = eval_sizes(saved)
    resize, crop = resize or saved_resize, crop or saved_crop
    if crop > resize:
        raise ValueError("crop %d exceeds resize %d: the crop must lie inside the resized image" % (crop, resize))
    tf = reference_transforms(False, resize, crop) if tta == "none" else reference_transforms(False, resize, crop, tta)
    from ..engine.native_engine import check_native_hw

    def native_runs(hw):
        try:
            check_native_hw(hw)
            return True
        except ValueError:
            return False

    # auto: the native engine on an H100 at a crop it runs, else the oracle (which takes any crop >= 32);
    # --engine native at a crop it does not run is refused by the engine
    use_native = engine == "native" or (engine == "auto" and torch.cuda.is_available()
                                        and torch.cuda.get_device_capability() == (9, 0) and native_runs(crop))
    if use_native:
        from ..engine.native_engine import NativeEngine
        net = NativeEngine(spec, device=torch.device("cuda", 0), batch=batch, init_state=state, distributed=False,
                           input_hw=crop)
        if tta != "none":
            net.set_val_tta(tta)
    else:
        net = build_oracle(spec, seed=0).eval()
        net.load_state_dict(state)
    out = []
    for i in range(0, len(files), batch):
        x = torch.stack([tf(Image.open(f).convert("RGB")) for f in files[i:i + batch]])
        if use_native:
            out.append(net.forward_logits((x, torch.zeros(x.shape[0], dtype=torch.int64))).float().cpu())
        elif tta != "none":                  # x: [b][V][3][crop][crop]
            out.append(torch.stack([net(x[:, v]).float() for v in range(x.shape[1])], 1))
        else:
            out.append(net(x).float())
    empty = (0, spec.num_classes) if tta == "none" else (0, len(tta_views(tta)), spec.num_classes)
    return (torch.cat(out) if out else torch.zeros(empty)), files


def mean_probabilities(logits: torch.Tensor) -> torch.Tensor:
    """Class probabilities of ``predict``'s logits: softmax, or with views ([n, V, C]) the mean of the views'
    softmaxes added in view order, as --val-tta scores them."""
    if logits.dim() == 2:
        return torch.softmax(logits, dim=1)
    acc = None
    for v in range(logits.shape[1]):
        p = torch.softmax(logits[:, v], dim=1)
        acc = p if acc is None else acc + p
    return acc / logits.shape[1]


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("checkpoint")
    ap.add_argument("images", nargs="+", help="image files and/or directories")
    ap.add_argument("--classes", default=None, help="comma-separated class names in label order")
    ap.add_argument("--data-root", default=None, help="take the class names from <root>/%s" % DATA.train_dir)
    ap.add_argument("--model", default=None, help="architecture (default: the one recorded in the checkpoint)")
    ap.add_argument("--engine", default="auto", choices=["auto", "native", "oracle"])
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--ema", action="store_true", help="classify with the checkpoint's EMA weights (--model-ema)")
    ap.add_argument("--resize", type=int, default=None,
                    help="Resize of the shorter side (default: the checkpoint's --val-resize-size, else %d)" % DATA.resize)
    ap.add_argument("--crop", type=int, default=None,
                    help="CenterCrop, the network's input (default: the checkpoint's --val-crop-size, else %d)" % DATA.crop)
    ap.add_argument("--tta", default="none", choices=list(TTA_MODES),
                    help="test-time augmentation: classify by the mean softmax of the mode's views, as --val-tta "
                         "(default: none, the centre crop)")
    a = ap.parse_args(argv)
    logits, files = predict(a.checkpoint, a.images, a.model, a.engine, a.batch, ema=a.ema, resize=a.resize,
                            crop=a.crop, tta=a.tta)
    names = a.classes.split(",") if a.classes else None
    if names is None and a.data_root:
        names = find_classes(os.path.join(a.data_root, DATA.train_dir))[0]
    prob = mean_probabilities(logits)
    for f, p in zip(files, prob):
        k = int(p.argmax())
        print("%s\t%s\t%.4f" % (f, names[k] if names and k < len(names) else k, float(p[k])))
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
