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


def _conv(x, a, w, b):
    """kornia's ``Conv`` block: InstanceNorm2d (no affine, eps 1e-5) -> PReLU -> Conv2d(5x5, padding 2)."""
    x = F.instance_norm(x, eps=1e-5)
    x = F.prelu(x, a)
    return F.conv2d(x, w, b, padding=w.shape[-1] // 2)


def unet(sd, x):
    feats = []
    for i in range(5):
        if i:
            x = F.avg_pool2d(x, 2)
        p = f"unet.path_down.{i}.1"
        x = _conv(x, sd[f"{p}.1.weight"], sd[f"{p}.3.weight"], sd[f"{p}.3.bias"])
        feats.append(x)
    bot = feats[4]
    for i in range(4):
        up = F.interpolate(bot, scale_factor=2, mode="bilinear", align_corners=False)
        p = f"unet.path_up.{i}.conv"
        bot = _conv(torch.cat([up, feats[3 - i]], 1), sd[f"{p}.1.weight"], sd[f"{p}.3.weight"], sd[f"{p}.3.bias"])
    return bot


def heads(sd, image, pad_if_not_divisible: bool = True):
    """image [B, 1 or 3, H, W] -> (heatmap [B, H, W], raw descriptors [B, 128, H, W]), in the image's dtype."""
    if image.shape[1] == 1:
        image = image.repeat(1, 3, 1, 1)
    h, w = image.shape[-2:]
    if pad_if_not_divisible:
        ph, pw = (16 - h % 16) % 16, (16 - w % 16) % 16
        image = F.pad(image, (0, pw, 0, ph))
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
