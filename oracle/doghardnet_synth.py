"""Seeded HardNet weights for the DoG-HardNet tests (test infrastructure only): kornia's ``HardNet.features`` layout
with Kaiming-scaled convolutions and BatchNorm running statistics that are far from (0, 1), so that folding them into
the convolutions is exercised.  Images come from ``oracle/sift_synth.py``."""
from __future__ import annotations

import torch

LAYERS = [(1, 32, 3), (32, 32, 3), (32, 64, 3), (64, 64, 3), (64, 128, 3), (128, 128, 3), (128, 128, 8)]
CONVS = [0, 3, 6, 9, 12, 15, 19]


def layout() -> list:
    """(name, shape) of HardNet's state_dict, in order (``features.*``)."""
    out = []
    for (ci, co, k), i in zip(LAYERS, CONVS):
        out += [(f"features.{i}.weight", (co, ci, k, k)), (f"features.{i + 1}.running_mean", (co,)),
                (f"features.{i + 1}.running_var", (co,)), (f"features.{i + 1}.num_batches_tracked", ())]
    return out


def make_state_dict(seed: int = 0) -> dict:
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for (ci, co, k), i in zip(LAYERS, CONVS):
        w = torch.randn(co, ci, k, k, generator=g) * (2.0 / (ci * k * k)) ** 0.5
        sd[f"features.{i}.weight"] = w
        sd[f"features.{i + 1}.running_mean"] = 0.3 * torch.randn(co, generator=g)
        sd[f"features.{i + 1}.running_var"] = 0.4 + 1.6 * torch.rand(co, generator=g)
        sd[f"features.{i + 1}.num_batches_tracked"] = torch.tensor(1000, dtype=torch.long)
    return sd
