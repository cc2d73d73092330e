"""Seeded synthetic DISK weights and images (test infrastructure for the DISK extractor).

The published DISK checkpoints (``depth-save.pth`` / ``epipolar-save.pth``) cannot be downloaded here, so the extractor
is pinned on synthetic weights under kornia's state_dict key names.  Only uniform draws from a seeded CPU generator and
exact elementwise fp32 ops are used, so the tensors are bit-identical on every CPU.

Scales: convolution weights uniform in +-sqrt(3 / fan_in) (unit variance after each instance norm), biases in +-0.1,
PReLU slopes in [0.1, 0.4].  Images are smooth blobs on a gradient, clipped to [0, 1]: the clipped areas are exactly
flat, so the heatmap has exact plateaus there (the NMS tie rule matters), and the blobs give clear maxima elsewhere.
"""
from __future__ import annotations

import math
from typing import Dict, List, Tuple

import torch

DOWN = [16, 32, 64, 64, 64]
UP = [64, 64, 64, 129]
SIZE = 5


def layout() -> List[Tuple[str, Tuple[int, ...]]]:
    """(key, shape) of every tensor of kornia's ``DISK.state_dict()``, in state_dict order."""
    out: List[Tuple[str, Tuple[int, ...]]] = []
    cins = [3] + DOWN[:-1]
    for i, (ci, co) in enumerate(zip(cins, DOWN)):
        p = f"unet.path_down.{i}.1"
        out += [(f"{p}.1.weight", (ci,)), (f"{p}.3.weight", (co, ci, SIZE, SIZE)), (f"{p}.3.bias", (co,))]
    bots = [DOWN[-1]] + UP[:-1]
    hors = DOWN[-2::-1]
    for i, (cb, ch, co) in enumerate(zip(bots, hors, UP)):
        p = f"unet.path_up.{i}.conv"
        ci = cb + ch
        out += [(f"{p}.1.weight", (ci,)), (f"{p}.3.weight", (co, ci, SIZE, SIZE)), (f"{p}.3.bias", (co,))]
    return out


def make_disk_state_dict(seed: int = 0) -> Dict[str, torch.Tensor]:
    g = torch.Generator().manual_seed(seed)
    sd: Dict[str, torch.Tensor] = {}
    for key, shape in layout():
        u = torch.rand(shape, generator=g, dtype=torch.float32)
        if len(shape) == 4:
            bound = math.sqrt(3.0 / (shape[1] * shape[2] * shape[3]))
            sd[key] = (u * 2 - 1) * bound
        elif key.endswith(".1.weight"):  # PReLU slopes
            sd[key] = 0.1 + 0.3 * u
        else:
            sd[key] = (u * 2 - 1) * 0.1
    return sd


def make_image(h: int, w: int, b: int = 1, seed: int = 0) -> torch.Tensor:
    """[b, 3, h, w] fp32 in [0, 1]: Gaussian blobs of random colour on a gradient, clipped (flat areas at 0 and 1)."""
    g = torch.Generator().manual_seed(seed)
    ys = torch.arange(h, dtype=torch.float32)[:, None]
    xs = torch.arange(w, dtype=torch.float32)[None, :]
    out = torch.empty(b, 3, h, w)
    n_blobs = max(4, (h * w) // 600)
    for i in range(b):
        params = torch.rand(n_blobs, 7, generator=g)
        img = 0.3 + 0.4 * (xs / max(w, 1)) + 0.0 * ys + torch.zeros(3, h, w)
        for cy, cx, r, a0, a1, a2, sgn in params.tolist():
            sigma = 1.5 + 6.0 * r
            blob = torch.exp(-((ys - cy * h) ** 2 + (xs - cx * w) ** 2) / (2 * sigma * sigma))
            s = 1.6 if sgn > 0.5 else -1.6
            img = img + s * torch.stack([a0 * blob, a1 * blob, a2 * blob])
        out[i] = img.clamp(0.0, 1.0)
    return out
