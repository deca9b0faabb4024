"""VGG-F ("VGG funnel") and plain VGG-16 as a *layer table*.

What the reference builds (distributedVggf.py:35-59): torchvision VGG-16 whose ``classifier[6]`` is
replaced by ``Linear(4096,512) -> ReLU -> Dropout(0.6) -> Linear(512,C)``; all layers trainable.
torchvision's VGG-16 topology (``D`` config): 13 conv3x3(pad 1)+ReLU in five blocks, each block
closed by a 2x2 max-pool, then AdaptiveAvgPool(7,7), flatten(25088) and
Linear(25088,4096)+ReLU+Dropout(.5), Linear(4096,4096)+ReLU+Dropout(.5).

Here the network is described once, as data (``VGGSpec``: a list of ``ConvSpec`` / ``FCSpec``),
and consumed twice:
  * ``build_oracle`` -> a plain ``nn.Module`` with *torchvision-identical state-dict keys*
    (``features.N.weight`` ... ``classifier.6.3.bias``) -- the CPU/gloo path and the numerical
    oracle for the kernels;
  * ``engine.native_engine`` -> flat parameter / gradient / optimizer arenas and a launch plan of
    hand-written sm_90a kernels.
Initialisation follows torchvision for the VGG part (kaiming_normal fan_out for conv, N(0, .01) for
Linear, zero bias) and ``nn.Linear``'s default for the funnel, which the reference creates after
the fact (SURVEY D5).  ``pretrained=True`` in the reference needs the network; we take an optional
local torchvision ``vgg16`` state dict instead.
"""
from __future__ import annotations

import dataclasses
import math
from typing import List, Optional, Sequence

import torch
from torch import nn

VGG16_CFG = (64, 64, "M", 128, 128, "M", 256, 256, 256, "M", 512, 512, 512, "M", 512, 512, 512, "M")


@dataclasses.dataclass(frozen=True)
class ConvSpec:
    name: str          # state-dict prefix, e.g. "features.0"
    cin: int
    cout: int
    pool_after: bool   # a 2x2/2 max-pool follows this conv's ReLU


@dataclasses.dataclass(frozen=True)
class FCSpec:
    name: str          # e.g. "classifier.0", "classifier.6.3"
    fin: int
    fout: int
    relu: bool
    dropout: float     # 0.0 -> no dropout layer after it
    torch_default_init: bool = False   # funnel layers use nn.Linear's default init


@dataclasses.dataclass(frozen=True)
class VGGSpec:
    convs: tuple
    fcs: tuple
    num_classes: int
    pooled_hw: int = 7     # AdaptiveAvgPool2d((7, 7))

    @property
    def param_names(self) -> List[str]:
        out = []
        for l in list(self.convs) + list(self.fcs):
            out += [l.name + ".weight", l.name + ".bias"]
        return out

    @property
    def num_layers(self) -> int:
        """Entries of the layer table, convs then fcs: what --freeze-layers counts."""
        return len(self.convs) + len(self.fcs)

    def check_freeze_layers(self, n: int) -> int:
        """``n`` leading layers frozen: 0 <= n < num_layers (the last Linear always trains)."""
        if not 0 <= int(n) < self.num_layers:
            raise ValueError("--freeze-layers must lie in [0, %d) for this model (got %d)" % (self.num_layers, n))
        return int(n)

    def frozen_param_names(self, n: int) -> List[str]:
        """The weights and biases of the first ``n`` layers."""
        return self.param_names[:2 * self.check_freeze_layers(n)]

    def param_shape(self, name: str):
        """Shape in the torch/torchvision layout (what a checkpoint stores)."""
        base, kind = name.rsplit(".", 1)
        for c in self.convs:
            if c.name == base:
                return (c.cout, c.cin, 3, 3) if kind == "weight" else (c.cout,)
        for f in self.fcs:
            if f.name == base:
                return (f.fout, f.fin) if kind == "weight" else (f.fout,)
        raise KeyError(name)

    @property
    def num_params(self) -> int:
        return sum(math.prod(self.param_shape(n)) for n in self.param_names)

    def flops_per_image(self, hw: int) -> float:
        """Forward multiply-add FLOPs (2*MAC) for a square ``hw`` input."""
        total, h = 0.0, hw
        for c in self.convs:
            total += 2.0 * h * h * c.cout * 9 * c.cin
            if c.pool_after:
                h //= 2
        for f in self.fcs:
            total += 2.0 * f.fin * f.fout
        return total


# torchvision's other plain VGG depths (configurations A, B, E of the paper; VGG16_CFG is D).  The
# reference only ever builds VGG-16; these come for free from the layer table: same kernels, same
# state-dict keys as torchvision.models.vgg11 / vgg13 / vgg19, with or without the funnel head.
VGG_CFGS = {
    11: [64, "M", 128, "M", 256, 256, "M", 512, 512, "M", 512, 512, "M"],
    13: [64, 64, "M", 128, 128, "M", 256, 256, "M", 512, 512, "M", 512, 512, "M"],
    19: [64, 64, "M", 128, 128, "M", 256, 256, 256, 256, "M", 512, 512, 512, 512, "M", 512, 512, 512, 512, "M"],
}


def _conv_specs(width_div: int = 1, cfg_list=None) -> tuple:
    convs, cin, idx = [], 3, 0
    cfg = [v if v == "M" else max(int(v) // width_div, 8) for v in (cfg_list or VGG16_CFG)]
    for i, v in enumerate(cfg):
        if v == "M":
            idx += 1
            continue
        pool = i + 1 < len(cfg) and cfg[i + 1] == "M"
        convs.append(ConvSpec("features.%d" % idx, cin, int(v), pool))
        cin = int(v)
        idx += 2     # conv + ReLU
    return tuple(convs)


def vggf_spec(num_classes: int) -> VGGSpec:
    """VGG-F: VGG-16 + funnel head (reference: distributedVggf.py:46-57)."""
    feat = 512 * 7 * 7
    fcs = (
        FCSpec("classifier.0", feat, 4096, True, 0.5),
        FCSpec("classifier.3", 4096, 4096, True, 0.5),
        FCSpec("classifier.6.0", 4096, 512, True, 0.6, torch_default_init=True),
        FCSpec("classifier.6.3", 512, num_classes, False, 0.0, torch_default_init=True),
    )
    return VGGSpec(_conv_specs(), fcs, num_classes)


def vgg16_spec(num_classes: int = 1000) -> VGGSpec:
    """Plain torchvision VGG-16 (BASELINE config #3: 1000 classes, 224x224)."""
    feat = 512 * 7 * 7
    fcs = (
        FCSpec("classifier.0", feat, 4096, True, 0.5),
        FCSpec("classifier.3", 4096, 4096, True, 0.5),
        FCSpec("classifier.6", 4096, num_classes, False, 0.0),
    )
    return VGGSpec(_conv_specs(), fcs, num_classes)


def vgg_spec(depth: int, num_classes: int = 1000, funnel: bool = False) -> VGGSpec:
    """torchvision VGG-11 / 13 / 16 / 19 (no batch norm), optionally with the reference's funnel head."""
    if depth == 16:
        return vggf_spec(num_classes) if funnel else vgg16_spec(num_classes)
    if depth not in VGG_CFGS:
        raise ValueError("VGG depth must be 11, 13, 16 or 19")
    head = vggf_spec(num_classes).fcs if funnel else vgg16_spec(num_classes).fcs
    return VGGSpec(_conv_specs(1, VGG_CFGS[depth]), head, num_classes)


def vggf_tiny_spec(num_classes: int) -> VGGSpec:
    """Same topology as VGG-F at 1/8 width (test / CI model: exercises every code path in seconds)."""
    convs = _conv_specs(8)
    feat = convs[-1].cout * 7 * 7
    fcs = (
        FCSpec("classifier.0", feat, 128, True, 0.5),
        FCSpec("classifier.3", 128, 128, True, 0.5),
        FCSpec("classifier.6.0", 128, 32, True, 0.6, torch_default_init=True),
        FCSpec("classifier.6.3", 32, num_classes, False, 0.0, torch_default_init=True),
    )
    return VGGSpec(convs, fcs, num_classes)


def vggf_mini_spec(num_classes: int) -> VGGSpec:
    """VGG-F topology with every conv at 64 channels and a narrow head: the smallest network the
    native wgmma kernels accept (channel counts must be multiples of 64); GPU test model."""
    convs = tuple(ConvSpec(c.name, 3 if i == 0 else 64, 64, c.pool_after) for i, c in enumerate(_conv_specs()))
    fcs = (
        FCSpec("classifier.0", 64 * 7 * 7, 256, True, 0.5),
        FCSpec("classifier.3", 256, 256, True, 0.5),
        FCSpec("classifier.6.0", 256, 64, True, 0.6, torch_default_init=True),
        FCSpec("classifier.6.3", 64, num_classes, False, 0.0, torch_default_init=True),
    )
    return VGGSpec(convs, fcs, num_classes)


def get_spec(model: str, num_classes: int) -> VGGSpec:
    if model in ("vggf-tiny", "tiny"):
        return vggf_tiny_spec(num_classes)
    if model in ("vggf-mini", "mini"):
        return vggf_mini_spec(num_classes)
    if model in ("vggf", "vgg-f", "vgg_funnel"):
        return vggf_spec(num_classes)
    if model in ("vgg16", "vgg-16"):
        return vgg16_spec(num_classes)
    for depth in (11, 13, 19):
        if model in ("vgg%d" % depth, "vgg-%d" % depth):
            return vgg_spec(depth, num_classes)
        if model in ("vggf%d" % depth, "vgg%d-funnel" % depth):
            return vgg_spec(depth, num_classes, funnel=True)
    raise ValueError("unknown model %r (vggf, vgg16, vgg11/13/19, vggf11/13/19, vggf-mini, vggf-tiny)" % model)


# ----------------------------------------------------------------------------------------------
# Oracle nn.Module (torch ops only).  Key-compatible with torchvision VGG + the reference funnel.
# ----------------------------------------------------------------------------------------------
class VGGOracle(nn.Module):
    def __init__(self, spec: VGGSpec):
        super().__init__()
        self.spec = spec
        feats: List[nn.Module] = []
        for c in spec.convs:
            feats += [nn.Conv2d(c.cin, c.cout, kernel_size=3, padding=1), nn.ReLU(inplace=True)]
            if c.pool_after:
                feats.append(nn.MaxPool2d(kernel_size=2, stride=2))
        self.features = nn.Sequential(*feats)
        self.avgpool = nn.AdaptiveAvgPool2d((spec.pooled_hw, spec.pooled_hw))
        self.classifier = _build_classifier(spec.fcs)
        init_oracle_(self)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        x = self.features(x)
        x = self.avgpool(x)
        x = torch.flatten(x, 1)
        return self.classifier(x)


def _fc_modules(f: FCSpec) -> List[nn.Module]:
    mods: List[nn.Module] = [nn.Linear(f.fin, f.fout)]
    if f.relu:
        mods.append(nn.ReLU(inplace=True))
    if f.dropout > 0:
        mods.append(nn.Dropout(f.dropout))
    return mods


def _build_classifier(fcs: Sequence[FCSpec]) -> nn.Sequential:
    """Reproduce the module indices behind names like ``classifier.3`` / ``classifier.6.0``."""
    top: List[nn.Module] = []
    nested: List[nn.Module] = []
    for f in fcs:
        parts = f.name.split(".")
        if len(parts) == 2:
            assert int(parts[1]) == len(top), f.name
            top += _fc_modules(f)
        else:   # classifier.6.K -> lives in a nested Sequential placed at index 6
            assert int(parts[2]) == len(nested), f.name
            nested += _fc_modules(f)
    if nested:
        top.append(nn.Sequential(*nested))
    return nn.Sequential(*top)


def init_oracle_(model: VGGOracle, generator: Optional[torch.Generator] = None) -> None:
    """torchvision VGG init for VGG layers, nn.Linear default for funnel layers."""
    mods = dict(model.named_modules())
    for c in model.spec.convs:
        m = mods[c.name]
        fan_out = c.cout * 9
        with torch.no_grad():
            m.weight.normal_(0.0, math.sqrt(2.0 / fan_out), generator=generator)
            m.bias.zero_()
    for f in model.spec.fcs:
        m = mods[f.name]
        with torch.no_grad():
            if f.torch_default_init:
                bound = 1.0 / math.sqrt(f.fin)     # kaiming_uniform(a=sqrt(5)) == U(+-1/sqrt(fan_in))
                m.weight.uniform_(-bound, bound, generator=generator)
                m.bias.uniform_(-bound, bound, generator=generator)
            else:
                m.weight.normal_(0.0, 0.01, generator=generator)
                m.bias.zero_()


def build_oracle(spec: VGGSpec, seed: Optional[int] = None,
                 pretrained_state: Optional[dict] = None) -> VGGOracle:
    gen = None
    if seed is not None:
        gen = torch.Generator().manual_seed(seed)
    model = VGGOracle(spec)
    if gen is not None:
        init_oracle_(model, gen)
    if pretrained_state is not None:
        load_pretrained_vgg16_(model, pretrained_state)
    return model


def freeze_leading_layers_(model: nn.Module, n: int) -> List[str]:
    """``requires_grad_(False)`` on both tensors of the first ``n`` layers of ``model.spec`` (--freeze-layers).
    Returns their names."""
    names = model.spec.frozen_param_names(n)
    params = dict(model.named_parameters())
    for name in names:
        params[name].requires_grad_(False)
    return names


def count_frozen_layers(model: nn.Module) -> int:
    """How many leading layers of ``model.spec`` have both tensors frozen."""
    params = dict(model.named_parameters())
    n = 0
    for layer in list(model.spec.convs) + list(model.spec.fcs):
        if params[layer.name + ".weight"].requires_grad or params[layer.name + ".bias"].requires_grad:
            break
        n += 1
    return n


def load_pretrained_vgg16_(model: nn.Module, state: dict) -> List[str]:
    """Copy every tensor of a torchvision ``vgg16`` state dict whose name and shape match.

    This is the offline counterpart of ``models.vgg16(pretrained=True)`` (distributedVggf.py:46):
    features.* and classifier.0/.3 are taken, the funnel keeps its fresh init.  A checkpoint of this
    project (``{"model": {"module.<name>": ...}, ...}``, e.g. the first stage of a fine-tune run with
    --freeze-layers) loads the same way, funnel included.
    """
    if isinstance(state.get("model"), dict):
        state = {(k[len("module."):] if k.startswith("module.") else k): v for k, v in state["model"].items()}
    own = model.state_dict()
    loaded = []
    for k, v in state.items():
        if k in own and tuple(own[k].shape) == tuple(v.shape):
            own[k].copy_(v)
            loaded.append(k)
    return loaded


def vgg_funnel_model(number_classes: int, pretrained_path: Optional[str] = None,
                     seed: Optional[int] = None) -> VGGOracle:
    """Drop-in for the reference's factory (distributedVggf.py:35)."""
    state = torch.load(pretrained_path, map_location="cpu") if pretrained_path else None
    return build_oracle(vggf_spec(number_classes), seed=seed, pretrained_state=state)
