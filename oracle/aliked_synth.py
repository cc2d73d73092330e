"""Seeded synthetic ALIKED weights and images (test infrastructure for the ALIKED extractor).

The official ``{model_name}.pth`` checkpoints cannot be downloaded here, so the extractor is pinned on synthetic weights
under the reference's state_dict key names (lightglue/aliked.py, class ``ALIKED``).  Only uniform draws and exact
elementwise fp32 ops are used, so the tensors are bit-identical on every CPU (same rule as superpoint_synth.py).

Scale factors, and what each one is for:
  * convolution weights: uniform in +-sqrt(3 / fan_in) (LeCun-uniform: unit variance through the SELU stack, so the
    deep layers still depend on the image);
  * BatchNorm: gamma in [0.6, 1.4], beta in +-0.1, running_mean in +-0.3, running_var in [0.5, 2.0] -- far from the
    (0, 1) defaults, so folding BN into the convolutions is really exercised;
  * ``DCN_OFFSET_PX`` scales the deformable offset convolutions of block3 / block4 so that offsets reach several pixels
    (std ~ 3 px): some taps leave the map and hit torchvision's zero-outside rule, and some are clamped at
    +-max(h, w) / 4 (2.5 px at the 1/32 level of a 240 x 320 image);
  * ``SCORE_SHIFT`` moves the score head's last-layer weights up by 0.3: its SELU inputs are mostly negative, so the
    logits move down and the sigmoid score map spreads around ``detection_threshold = 0.2`` (median ~0.03, 90th
    percentile ~0.37 at 240 x 320): hundreds of NMS maxima pass it, not none and not all, and no score saturates at 1.0
    (saturated plateaus would make NMS ties).  ``SCORE_GAIN`` (1.0) is kept as the knob for that spread;
  * SDDH's offset MLP reads unit-norm 128-vectors (per channel ~1/sqrt(dim)): ``SDDH_IN_GAIN`` restores unit scale in
    its first layer and ``SDDH_OFFSET_PX`` scales its second, so descriptor samples move by more than a pixel;
  * biases (offset convolutions, 1x1 downsamples, SDDH offset MLP) in +-0.05 (plus the scalings above).
"""
from __future__ import annotations

import math
from typing import Dict, List, Tuple

import torch

# c1, c2, c3, c4, dim, K, M   (aliked.py, ALIKED.cfgs)
CFGS = {
    "aliked-t16": [8, 16, 32, 64, 64, 3, 16],
    "aliked-n16": [16, 32, 64, 128, 128, 3, 16],
    "aliked-n16rot": [16, 32, 64, 128, 128, 3, 16],
    "aliked-n32": [16, 32, 64, 128, 128, 3, 32],
}
DCN_OFFSET_PX = 3.0
SCORE_GAIN = 1.0
SCORE_SHIFT = 0.3
SDDH_IN_GAIN = 8.0
SDDH_OFFSET_PX = 2.5


def layout(model_name: str) -> List[Tuple[str, Tuple[int, ...]]]:
    """(key, shape) of every tensor of the reference state_dict except ``num_batches_tracked``, in state_dict order."""
    c1, c2, c3, c4, dim, K, M = CFGS[model_name]
    out: List[Tuple[str, Tuple[int, ...]]] = []

    def bn(p, c):
        out.extend([(f"{p}.weight", (c,)), (f"{p}.bias", (c,)), (f"{p}.running_mean", (c,)), (f"{p}.running_var", (c,))])

    def conv(p, ci, co, dcn):
        if dcn:
            out.extend([(f"{p}.offset_conv.weight", (18, ci, 3, 3)), (f"{p}.offset_conv.bias", (18,)),
                        (f"{p}.regular_conv.weight", (co, ci, 3, 3))])
        else:
            out.append((f"{p}.weight", (co, ci, 3, 3)))

    for blk, ci, co, dcn, res in (("block1", 3, c1, False, False), ("block2", c1, c2, False, True),
                                  ("block3", c2, c3, True, True), ("block4", c3, c4, True, True)):
        conv(f"{blk}.conv1", ci, co, dcn)
        bn(f"{blk}.bn1", co)
        conv(f"{blk}.conv2", co, co, dcn)
        bn(f"{blk}.bn2", co)
        if res:
            out.extend([(f"{blk}.downsample.weight", (co, ci, 1, 1)), (f"{blk}.downsample.bias", (co,))])
    for i, ci in enumerate((c1, c2, c3, dim), 1):
        out.append((f"conv{i}.weight", (dim // 4, ci, 1, 1)))
    out.extend([("score_head.0.weight", (8, dim, 1, 1)), ("score_head.2.weight", (4, 8, 3, 3)),
                ("score_head.4.weight", (4, 4, 3, 3)), ("score_head.6.weight", (1, 4, 3, 3))])
    out.extend([("desc_head.agg_weights", (M, dim, dim)), ("desc_head.offset_conv.0.weight", (2 * M, dim, K, K)),
                ("desc_head.offset_conv.0.bias", (2 * M,)), ("desc_head.offset_conv.2.weight", (2 * M, 2 * M, 1, 1)),
                ("desc_head.offset_conv.2.bias", (2 * M,)), ("desc_head.sf_conv.weight", (dim, dim, 1, 1))])
    return out


def _u(g, shape, lo, hi):
    return torch.rand(*shape, generator=g) * (hi - lo) + lo


def make_aliked_state_dict(model_name: str = "aliked-n16", seed: int = 0) -> Dict[str, torch.Tensor]:
    g = torch.Generator().manual_seed(seed)
    sd: Dict[str, torch.Tensor] = {}
    for key, shape in layout(model_name):
        leaf = key.rsplit(".", 1)[1]
        if ".bn" in key:
            lo, hi = {"weight": (0.6, 1.4), "bias": (-0.1, 0.1), "running_mean": (-0.3, 0.3), "running_var": (0.5, 2.0)}[leaf]
            t = _u(g, shape, lo, hi)
        elif leaf == "bias":
            t = _u(g, shape, -0.05, 0.05)
        elif key == "desc_head.agg_weights":
            b = math.sqrt(3.0 / (shape[0] * shape[1]))
            t = _u(g, shape, -b, b)
        else:
            fan_in = 1
            for s in shape[1:]:
                fan_in *= s
            b = math.sqrt(3.0 / fan_in)
            t = _u(g, shape, -b, b)
            if "offset_conv.weight" in key:  # block3 / block4 deformable offsets
                t = t * DCN_OFFSET_PX
            elif key == "score_head.6.weight":
                t = t * SCORE_GAIN + SCORE_SHIFT
            elif key == "desc_head.offset_conv.0.weight":
                t = t * SDDH_IN_GAIN
            elif key == "desc_head.offset_conv.2.weight":
                t = t * SDDH_OFFSET_PX
        sd[key] = t
    for key in list(sd):  # BatchNorm counters: part of the state_dict, not of the math
        if key.endswith(".running_var"):
            sd[key[: -len("running_var")] + "num_batches_tracked"] = torch.tensor(0, dtype=torch.long)
    return sd


def make_image(h: int, w: int, b: int = 1, seed: int = 0) -> torch.Tensor:
    """[b, 3, h, w] in [0, 1]: random 8x8 colour blocks plus per-pixel noise (exact fp32 arithmetic only)."""
    g = torch.Generator().manual_seed(seed)
    coarse = torch.rand(b, 3, (h + 7) // 8, (w + 7) // 8, generator=g)
    fine = torch.rand(b, 3, h, w, generator=g)
    return coarse.repeat_interleave(8, 2).repeat_interleave(8, 3)[:, :, :h, :w] * 0.7 + fine * 0.3
