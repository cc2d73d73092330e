"""Torch-only restatement of kornia's DISK as ``lightglue.DISK`` runs it (reference lightglue/disk.py ->
``kornia.feature.DISK``): the U-Net, the padding to multiples of 16, NMS, the threshold, the kthvalue top-k and the
descriptor lookup.  Kornia is not a dependency, so this module is the specification the CUDA path is tested against; it
runs in any dtype on any device.

``sd`` is a state dict under kornia's ``DISK`` names (``unet.path_down.{i}.1.{1,3}.*``, ``unet.path_up.{i}.conv.{1,3}.*``).
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

DEFAULT_CONF = {"max_num_keypoints": None, "nms_window_size": 5, "detection_threshold": 0.0, "pad_if_not_divisible": True}


LAYERS = 9  # down0 .. down4, up0 .. up3


def params(sd, l):
    """(PReLU slope, conv weight, conv bias) of layer l: down0 .. down4 (0 .. 4), up0 .. up3 (5 .. 8)."""
    p = f"unet.path_down.{l}.1" if l < 5 else f"unet.path_up.{l - 5}.conv"
    return sd[f"{p}.1.weight"], sd[f"{p}.3.weight"], sd[f"{p}.3.bias"]


def gather(l, inputs, align_corners: bool = False):
    """Layer l's input before its instance norm.  l = 0: ``inputs`` is the (padded, 3-channel) image; l >= 1:
    ``inputs[i]`` is layer i's raw output (only layers l - 1 and, for the up path, 8 - l are read).  down1 .. down4
    average-pool layer l - 1; up0 .. up3 upsample it x2 (bilinear) and concatenate down block 8 - l."""
    if l == 0:
        return inputs
    if l <= 4:
        return F.avg_pool2d(inputs[l - 1], 2)
    up = F.interpolate(inputs[l - 1], scale_factor=2, mode="bilinear", align_corners=align_corners)
    return torch.cat([up, inputs[8 - l]], 1)


def prepare(sd, l, inputs):
    """Layer l's convolution operand: its gathered input, InstanceNorm2d (no affine, eps 1e-5), PReLU.  For l = 8 this
    is x3, the input of up3."""
    return F.prelu(F.instance_norm(gather(l, inputs), eps=1e-5), params(sd, l)[0])


def layer(sd, l, inputs):
    """Layer l's raw output (kornia's ``Conv`` block on its gathered input): the 5x5 convolution of ``prepare``."""
    _, w, b = params(sd, l)
    return F.conv2d(prepare(sd, l, inputs), w, b, padding=w.shape[-1] // 2)


def unet(sd, x):
    raw = [layer(sd, 0, x)]
    for l in range(1, LAYERS):
        raw.append(layer(sd, l, raw))
    return raw[-1]


def network_input(image, pad_if_not_divisible: bool = True):
    """image [B, 1 or 3, H, W] -> the U-Net's input: three channels, zero-padded right / bottom to multiples of 16."""
    if image.shape[1] == 1:
        image = image.repeat(1, 3, 1, 1)
    h, w = image.shape[-2:]
    if pad_if_not_divisible:
        ph, pw = (16 - h % 16) % 16, (16 - w % 16) % 16
        image = F.pad(image, (0, pw, 0, ph))
    return image


def heads(sd, image, pad_if_not_divisible: bool = True):
    """image [B, 1 or 3, H, W] -> (heatmap [B, H, W], raw descriptors [B, 128, H, W]), in the image's dtype."""
    h, w = image.shape[-2:]
    image = network_input(image, pad_if_not_divisible)
    sd = {k: v.to(image) for k, v in sd.items()}
    out = unet(sd, image)[..., :h, :w]
    return out[:, 128], out[:, :128]


def nms_mask(heat, window: int):
    """[H, W] -> bool: the pixels that are the first maximum of their own window (max_pool2d's index rule)."""
    if window % 2 == 0:
        raise ValueError(f"window_size has to be odd, got {window}")
    _, ix = F.max_pool2d(heat[None, None], window, stride=1, padding=window // 2, return_indices=True)
    own = torch.arange(heat.numel(), device=heat.device).reshape(heat.shape)
    return ix[0, 0] == own


def detect(heat, window: int, threshold: float, n):
    """One image's heatmap [H, W] -> (keypoints [k, 2] (x, y) long, scores [k]) in row-major order."""
    keep = nms_mask(heat, window) & (heat > threshold)
    yx = keep.nonzero()
    logp = heat[keep]
    if n is not None:
        n_ = min(n + 1, logp.numel())
        thr = torch.kthvalue(-logp, n_).values  # raises on zero candidates, as the reference does
        sel = logp > -thr
        yx, logp = yx[sel][:n], logp[sel][:n]
    return yx.flip(1), logp


def forward(sd, image, conf=None):
    conf = {**DEFAULT_CONF, **(conf or {})}
    heat, desc = heads(sd, image, conf["pad_if_not_divisible"])
    kps, scs, dss = [], [], []
    for b in range(heat.shape[0]):
        xy, logp = detect(heat[b], conf["nms_window_size"], conf["detection_threshold"], conf["max_num_keypoints"])
        d = desc[b][:, xy[:, 1], xy[:, 0]].T
        kps.append(xy.to(heat.dtype))
        scs.append(logp)
        dss.append(F.normalize(d, dim=-1))
    return {"keypoints": torch.stack(kps), "keypoint_scores": torch.stack(scs), "descriptors": torch.stack(dss)}
