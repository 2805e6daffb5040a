"""TEST ORACLE — the reference's ``NoHeadDenseNet`` (DenseNet-121, ``reproducibility/embedders/mudipath.py:125-130``)
restated with ``torch.nn.functional`` only, so that it needs no torchvision, plus the seeded synthetic weights the
tests use.

``features(sd, x)`` is torchvision's ``DenseNet.features`` in eval mode and ``forward`` ends in
``adaptive_avg_pool2d`` with no ReLU.  ``emulate=True`` follows the numerics of ``plip_b200/csrc/densenet.cu`` instead:
bf16 operands at exactly the points the kernels round (the normalised input, every convolution weight, every stored
activation), fp32 accumulation, BN as the folded ``x * scale + shift`` (two fp32 roundings), the transition's 2x2
average pool taken before its 1x1 convolution and the tail's BN after the average.
"""
from __future__ import annotations

import hashlib
from typing import Dict

import numpy as np
import torch
import torch.nn.functional as F

GROWTH, BOTTLENECK, STEM = 32, 128, 64
BLOCKS = (6, 12, 24, 16)
EPS = 1e-5
MEAN = (0.485, 0.456, 0.406)
STD = (0.229, 0.224, 0.225)


def layer_names():
    """``(kind, prefix, in_channels)`` of every BN + conv of DenseNet-121, in forward order."""
    out, c = [], STEM
    for b, n in enumerate(BLOCKS):
        for j in range(n):
            out.append(("layer", f"features.denseblock{b + 1}.denselayer{j + 1}", c + GROWTH * j))
        c += GROWTH * n
        if b < 3:
            out.append(("transition", f"features.transition{b + 1}", c))
            c //= 2
    return out


def normalize_u8(tiles: torch.Tensor) -> torch.Tensor:
    """uint8 ``[n,224,224,3]`` -> float32 ``[n,3,224,224]``: ``ToTensor`` + ImageNet ``Normalize``."""
    x = tiles.permute(0, 3, 1, 2).float().div(255)
    mean = torch.tensor(MEAN, dtype=torch.float32, device=x.device).view(1, 3, 1, 1)
    std = torch.tensor(STD, dtype=torch.float32, device=x.device).view(1, 3, 1, 1)
    return (x - mean) / std


def fold(sd, name):
    """Eval BN of ``name`` as float32 ``(scale, shift)``, folded in float64."""
    g, b, m, v = (sd[f"{name}.{k}"].double() for k in ("weight", "bias", "running_mean", "running_var"))
    s = g / torch.sqrt(v + EPS)
    return s.float(), (b - m * s).float()


def _bn(sd, name, x):
    return F.batch_norm(x, sd[f"{name}.running_mean"], sd[f"{name}.running_var"], sd[f"{name}.weight"],
                        sd[f"{name}.bias"], training=False, eps=EPS)


def _bf(t):
    return t.to(torch.bfloat16).float()


def _affine(sd, name, x):
    s, b = fold(sd, name)
    return x * s.view(1, -1, 1, 1) + b.view(1, -1, 1, 1)


def features(sd: Dict[str, torch.Tensor], x: torch.Tensor, emulate: bool = False, stats=None) -> torch.Tensor:
    """``DenseNet.features`` (eval) of normalised float32 NCHW ``x``.  ``stats`` (a dict): train-mode batch statistics
    are used and recorded there instead of the running ones (the calibration pass of :func:`make_state_dict`)."""
    def bn(name, t):
        if stats is not None:
            mean, var = t.mean((0, 2, 3)), t.var((0, 2, 3), unbiased=False)
            stats[name] = (mean, t.var((0, 2, 3), unbiased=True))
            g, b = sd[f"{name}.weight"], sd[f"{name}.bias"]
            return (t - mean.view(1, -1, 1, 1)) / torch.sqrt(var.view(1, -1, 1, 1) + EPS) * g.view(1, -1, 1, 1) \
                + b.view(1, -1, 1, 1)
        return _affine(sd, name, t) if emulate else _bn(sd, name, t)

    W = (lambda k: _bf(sd[k])) if emulate else (lambda k: sd[k])
    r = _bf if emulate else (lambda t: t)
    x = r(x)
    x = r(F.relu(bn("features.norm0", F.conv2d(x, W("features.conv0.weight"), stride=2, padding=3))))
    x = F.max_pool2d(x, 3, 2, 1)
    for kind, pre, c in layer_names():
        if kind == "layer":
            h = r(F.relu(bn(f"{pre}.norm1", x)))
            h = r(F.relu(bn(f"{pre}.norm2", F.conv2d(h, W(f"{pre}.conv1.weight")))))
            h = r(F.conv2d(h, W(f"{pre}.conv2.weight"), padding=1))
            x = torch.cat([x, h], 1)
        elif emulate:   # pool first, in the kernel's summation order
            h = F.relu(bn(f"{pre}.norm", x))
            h = ((h[:, :, 0::2, 0::2] + h[:, :, 0::2, 1::2]) + h[:, :, 1::2, 0::2]) + h[:, :, 1::2, 1::2]
            x = r(F.conv2d(r(h * 0.25), W(f"{pre}.conv.weight")))
        else:
            x = F.avg_pool2d(F.conv2d(F.relu(bn(f"{pre}.norm", x)), W(f"{pre}.conv.weight")), 2, 2)
    if emulate:
        return x   # norm5 is applied after the average pool (forward)
    return bn("features.norm5", x)


@torch.no_grad()
def forward(sd, x: torch.Tensor, emulate: bool = False) -> torch.Tensor:
    """``NoHeadDenseNet.forward(x)`` flattened to ``[n,1024]`` float32."""
    f = features(sd, x, emulate)
    if emulate:
        s, b = fold(sd, "features.norm5")
        return f.mean((2, 3)) * s + b
    return F.adaptive_avg_pool2d(f, (1, 1)).flatten(1)


@torch.no_grad()
def forward_u8(sd, tiles: torch.Tensor, emulate: bool = False) -> torch.Tensor:
    return forward(sd, normalize_u8(tiles), emulate)


def param_shapes() -> Dict[str, tuple]:
    """torchvision ``densenet121()`` feature parameters (BN buffers included, ``num_batches_tracked`` excluded)."""
    shapes = {"features.conv0.weight": (STEM, 3, 7, 7)}

    def bn(name, c):
        for k in ("weight", "bias", "running_mean", "running_var"):
            shapes[f"{name}.{k}"] = (c,)
    bn("features.norm0", STEM)
    for kind, pre, c in layer_names():
        if kind == "layer":
            bn(f"{pre}.norm1", c)
            shapes[f"{pre}.conv1.weight"] = (BOTTLENECK, c, 1, 1)
            bn(f"{pre}.norm2", BOTTLENECK)
            shapes[f"{pre}.conv2.weight"] = (GROWTH, BOTTLENECK, 3, 3)
        else:
            bn(f"{pre}.norm", c)
            shapes[f"{pre}.conv.weight"] = (c // 2, c, 1, 1)
    bn("features.norm5", 1024)
    return shapes


@torch.no_grad()
def make_state_dict(seed: int = 0) -> Dict[str, torch.Tensor]:
    """Seeded synthetic DenseNet-121 weights with torchvision's names.

    Convolutions are initialised as torchvision does (``kaiming_normal_``: std ``sqrt(2 / fan_in)``), BN ``gamma`` /
    ``beta`` are randomised, and the running statistics come from one train-mode pass (PyTorch's ``momentum=None``:
    the batch's mean and unbiased variance) over a fixed synthetic batch — so eval BN is far from the identity and
    the folding is exercised.  Includes torchvision's ``classifier`` and ``num_batches_tracked`` entries so that
    ``densenet121().load_state_dict`` accepts it."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for name, shape in param_shapes().items():
        if name.endswith("conv0.weight") or name.endswith("conv1.weight") or name.endswith("conv2.weight") \
                or name.endswith("conv.weight"):
            fan_in = shape[1] * shape[2] * shape[3]
            sd[name] = torch.randn(shape, generator=g) * (2.0 / fan_in) ** 0.5
        elif name.endswith(".weight"):
            sd[name] = 0.6 + 0.8 * torch.rand(shape, generator=g)
        elif name.endswith(".bias"):
            sd[name] = 0.2 * torch.randn(shape, generator=g)
        elif name.endswith("running_mean"):
            sd[name] = torch.zeros(shape)
        else:
            sd[name] = torch.ones(shape)
    batch = torch.randint(0, 256, (4, 128, 128, 3), generator=g, dtype=torch.uint8)
    stats = {}
    features(sd, normalize_u8(batch), stats=stats)
    for name, (mean, var) in stats.items():
        sd[f"{name}.running_mean"] = mean.clone()
        sd[f"{name}.running_var"] = var.clone()
    for name in list(sd):
        if name.endswith("running_var"):
            sd[name.replace("running_var", "num_batches_tracked")] = torch.tensor(1, dtype=torch.long)
    sd["classifier.weight"] = torch.zeros(1000, 1024)
    sd["classifier.bias"] = torch.zeros(1000)
    return sd


def checksum(sd: Dict[str, torch.Tensor]) -> str:
    """sha256 over the float32 bytes of every floating-point tensor, in sorted name order."""
    h = hashlib.sha256()
    for k in sorted(sd):
        if sd[k].is_floating_point():
            h.update(k.encode())
            h.update(np.ascontiguousarray(sd[k].float().numpy()).tobytes())
    return h.hexdigest()


def cosine_gap(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """Per-row ``1 - cos(a, b)`` in float64."""
    a, b = a.double(), b.double()
    return 1 - (a * b).sum(1) / (a.norm(dim=1) * b.norm(dim=1))
