"""Torch restatement of what the reference's DoGHardNet computes after detection (test infrastructure only): kornia's
``laf_from_center_scale_ori``, ``extract_patches_from_pyramid`` (with ``pyrdown``) and ``HardNet``, as ``LAFDescriptor``
runs them.  Kornia is not a dependency here, so each rule below is restated from kornia 0.7's sources as recalled; the
ones that could not be checked offline are listed in INTEGRATION.md (DoG-HardNet).  Every function works in the dtype
and on the device of its inputs (the GPU tests run it in float64).

* LAF: A = s R, R = [[cos t, sin t], [-sin t, cos t]], t = deg2rad(ori_deg); centre column (x, y), no 0.5 shift.
* normalize_laf / denormalize_laf: the 2x2 part divided / multiplied by min(h - 1, w - 1), the centre by (w - 1, h - 1).
* extract_patches_from_pyramid(img, laf, 32): level = floor(clamp(log2(2 sqrt(|det A + 1e-10|) / 32), 0,
  max(0, min(H, W) // 32 - 1))); levels are visited in order, each sampling its own keypoints, and the loop stops after
  the first level whose shorter side is < 32 -- a keypoint whose level is never reached keeps an all-zero patch.
* pyrdown: 5x5 binomial / 256 with torch "reflect" borders, then bilinear F.interpolate to (int(h / 2), w // 2).
* patch grid: affine_grid(denormalize(nlaf, level), [N, 1, 32, 32], align_corners=False), then 2 g / (w - 1) - 1 (and
  likewise y), then grid_sample(bilinear, padding_mode="border", align_corners=False).
* HardNet: (x - mean) / (std + 1e-6) per patch (unbiased std over C, H, W); the seven bias-free convolutions, each
  followed by BatchNorm2d(affine=False, eps=1e-5) in eval mode and ReLU (except the last); flatten; F.normalize.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

PS = 32
CONVS = [0, 3, 6, 9, 12, 15, 19]  # features.{i}: the convolutions; their BatchNorms are features.{i + 1}
STRIDES = [1, 1, 2, 1, 2, 1, 1]


# ---------------------------------------------------------------------------------------------------------- LAFs
def laf_from_center_scale_ori(xy: torch.Tensor, scale: torch.Tensor, ori: torch.Tensor) -> torch.Tensor:
    """xy [B, N, 2], scale [B, N, 1, 1], ori [B, N, 1] (degrees) -> LAFs [B, N, 2, 3]."""
    t = torch.deg2rad(ori.squeeze(-1))
    c, s = torch.cos(t), torch.sin(t)
    rot = torch.stack([c, s, -s, c], dim=-1).view(*t.shape, 2, 2)
    return torch.cat([rot * scale, xy.unsqueeze(-1)], dim=-1)


def _coef(h: int, w: int, like: torch.Tensor) -> torch.Tensor:
    wf, hf = float(w - 1), float(h - 1)
    coef = torch.full((1, 1, 2, 3), min(wf, hf), dtype=like.dtype, device=like.device)
    coef[0, 0, 0, 2] = wf
    coef[0, 0, 1, 2] = hf
    return coef


def normalize_laf(laf: torch.Tensor, h: int, w: int) -> torch.Tensor:
    return laf / _coef(h, w, laf)


def denormalize_laf(laf: torch.Tensor, h: int, w: int) -> torch.Tensor:
    return laf * _coef(h, w, laf)


def get_laf_scale(laf: torch.Tensor) -> torch.Tensor:
    det = laf[..., 0:1, 0:1] * laf[..., 1:2, 1:2] - laf[..., 1:2, 0:1] * laf[..., 0:1, 1:2] + 1e-10
    return det.abs().sqrt()


# ---------------------------------------------------------------------------------------------------------- pyramid
def pyrdown(img: torch.Tensor) -> torch.Tensor:
    """img [B, C, h, w] -> [B, C, int(h / 2), w // 2]."""
    k1 = torch.tensor([1.0, 4.0, 6.0, 4.0, 1.0], dtype=img.dtype, device=img.device)
    k = (k1[:, None] * k1[None, :] / 256.0)[None, None].repeat(img.shape[1], 1, 1, 1)
    h, w = img.shape[-2:]
    blur = F.conv2d(F.pad(img, (2, 2, 2, 2), mode="reflect"), k, groups=img.shape[1])
    return F.interpolate(blur, size=(int(float(h) / 2.0), int(float(w) // 2.0)), mode="bilinear", align_corners=False)


def pyramid(img: torch.Tensor) -> list:
    """The levels extract_patches_from_pyramid visits: level 0, then pyrdown while the shorter side is >= 32."""
    levels = [img]
    while min(levels[-1].shape[-2:]) >= PS:
        levels.append(pyrdown(levels[-1]))
    return levels


def pyramid_levels(laf: torch.Tensor, h: int, w: int) -> torch.Tensor:
    """The pyramid level of each LAF [..., 2, 3] of an h x w image (before the loop decides which are reached)."""
    scale = 2.0 * get_laf_scale(denormalize_laf(normalize_laf(laf, h, w), h, w)) / float(PS)
    max_level = min(h, w) // PS
    return scale.log2().clamp(min=0.0, max=max(0, max_level - 1)).long().reshape(laf.shape[:-2])


def patch_grid(nlaf: torch.Tensor, h: int, w: int) -> torch.Tensor:
    """nlaf [N, 2, 3] normalised LAFs -> grid_sample grid [N, 32, 32, 2] on an h x w level."""
    laf = denormalize_laf(nlaf[None], h, w)[0]
    grid = F.affine_grid(laf, [laf.shape[0], 1, PS, PS], align_corners=False)
    gx = 2.0 * grid[..., 0] / float(w - 1) - 1.0
    gy = 2.0 * grid[..., 1] / float(h - 1) - 1.0
    return torch.stack([gx, gy], dim=-1)


def extract_patches(img: torch.Tensor, laf: torch.Tensor) -> torch.Tensor:
    """img [1, 1, h, w], laf [N, 2, 3] (pixels of img) -> patches [N, 1, 32, 32]."""
    h, w = img.shape[-2:]
    nlaf = normalize_laf(laf[None], h, w)[0]
    lv = pyramid_levels(laf, h, w)
    out = torch.zeros(laf.shape[0], img.shape[1], PS, PS, dtype=img.dtype, device=img.device)
    for i, cur in enumerate(pyramid(img)):
        m = lv == i
        if m.any():
            ch, cw = cur.shape[-2:]
            grid = patch_grid(nlaf[m], ch, cw)
            out[m] = F.grid_sample(cur.expand(grid.shape[0], -1, -1, -1), grid, mode="bilinear", padding_mode="border",
                                   align_corners=False)
    return out


# ---------------------------------------------------------------------------------------------------------- HardNet
def hardnet(sd: dict, patches: torch.Tensor) -> torch.Tensor:
    """sd: HardNet's state_dict (``features.*``); patches [N, 1, 32, 32] -> unit descriptors [N, 128]."""
    x = patches
    if x.shape[0] == 0:
        return x.new_zeros(0, 128)
    sp, mp = torch.std_mean(x, dim=(1, 2, 3), keepdim=True)
    x = (x - mp) / (sp + 1e-6)
    for li, (i, s) in enumerate(zip(CONVS, STRIDES)):
        wt = sd[f"features.{i}.weight"].to(x)
        x = F.conv2d(x, wt, stride=s, padding=1 if wt.shape[-1] == 3 else 0)
        x = F.batch_norm(x, sd[f"features.{i + 1}.running_mean"].to(x), sd[f"features.{i + 1}.running_var"].to(x),
                         training=False, eps=1e-5)
        if li < len(CONVS) - 1:
            x = F.relu(x)
    return F.normalize(x.reshape(x.shape[0], -1), dim=1)


def folded(sd: dict, li: int, like: torch.Tensor):
    """Convolution li's weight and bias with its eval BatchNorm folded in, in double as dhn_create folds them:
    w rs and -running_mean rs, rs = 1 / sqrt(running_var + 1e-5); returned in the dtype and on the device of `like`."""
    i = CONVS[li]
    rs = 1.0 / torch.sqrt(sd[f"features.{i + 1}.running_var"].double() + 1e-5)
    w = sd[f"features.{i}.weight"].double() * rs.view(-1, 1, 1, 1)
    b = -sd[f"features.{i + 1}.running_mean"].double() * rs
    return w.to(like), b.to(like)


def hardnet_layers(sd: dict, patches: torch.Tensor) -> list:
    """HardNet layer by layer on folded weights (`folded`): the post-ReLU outputs of convs 0 .. 5 [N, C, h, w] and conv
    6's output before F.normalize [N, 128].  Each layer l >= 1 is ``hardnet_conv(sd, l, outputs[l - 1])``."""
    sp, mp = torch.std_mean(patches, dim=(1, 2, 3), keepdim=True)
    x = (patches - mp) / (sp + 1e-6)
    out = []
    for li in range(len(CONVS)):
        x = hardnet_conv(sd, li, x)
        out.append(x)
    out[-1] = out[-1].reshape(out[-1].shape[0], -1)
    return out


def hardnet_conv(sd: dict, li: int, x: torch.Tensor) -> torch.Tensor:
    """Convolution li (folded BatchNorm), with its ReLU for li < 6, on the previous layer's output x [N, C, h, w]."""
    w, b = folded(sd, li, x)
    y = F.conv2d(x, w, b, stride=STRIDES[li], padding=1 if w.shape[-1] == 3 else 0)
    return F.relu(y) if li < len(CONVS) - 1 else y


# ---------------------------------------------------------------------------------------------------------- the extractor
def gray(image: torch.Tensor) -> torch.Tensor:
    """kornia's rgb_to_grayscale of [B, 3, H, W] (0.299 r + 0.587 g + 0.114 b); gray images pass through."""
    if image.shape[1] != 3:
        return image
    wts = torch.tensor([0.299, 0.587, 0.114], dtype=image.dtype, device=image.device)
    return wts[0] * image[:, 0:1] + wts[1] * image[:, 1:2] + wts[2] * image[:, 2:3]


def describe_one(sd: dict, img: torch.Tensor, kpts: torch.Tensor, scales: torch.Tensor, oris: torch.Tensor) -> torch.Tensor:
    """One gray crop img [1, h, w]; kpts [n, 2], scales [n] (cv2 sizes), oris [n] (radians) -> [n, 128]."""
    laf = laf_from_center_scale_ori(kpts.reshape(1, -1, 2), 6.0 * scales.reshape(1, -1, 1, 1),
                                    torch.rad2deg(oris).reshape(1, -1, 1))
    return hardnet(sd, extract_patches(img[None], laf[0]))


def describe(sd: dict, image: torch.Tensor, kpts: torch.Tensor, scales: torch.Tensor, oris: torch.Tensor,
             image_size=None) -> torch.Tensor:
    """LAFDescriptor(HardNet) as DoGHardNet.forward runs it: image [B, 1 or 3, H, W] -> gray, cropped to image_size
    [B, 2] (w, h) when given; kpts [B, n, 2], scales [B, n], oris [B, n] -> descriptors [B, n, 128]."""
    g = gray(image)
    out = []
    for k in range(g.shape[0]):
        img = g[k]
        if image_size is not None:
            w, h = (int(v) for v in image_size[k])
            img = img[:, :h, :w]
        out.append(describe_one(sd, img, kpts[k], scales[k], oris[k]))
    return torch.stack(out)


def forward(sd: dict, image: torch.Tensor, feats: list, image_size=None) -> dict:
    """DoGHardNet.forward given each image's SIFT output ``feats[k]`` (keypoints, scales, oris, keypoint_scores: a SIFT
    fixture's rows or the CUDA SIFT's): adds the descriptors and stacks over the batch (equal counts required)."""
    g = gray(image)
    pred = []
    for k, f in enumerate(feats):
        img = g[k]
        if image_size is not None:
            w, h = (int(v) for v in image_size[k])
            img = img[:, :h, :w]
        p = {key: f[key] for key in ("keypoints", "scales", "oris", "keypoint_scores")}
        p["descriptors"] = describe_one(sd, img, p["keypoints"].to(img), p["scales"].to(img), p["oris"].to(img))
        pred.append(p)
    return {key: torch.stack([p[key] for p in pred], 0) for key in pred[0]}


def level_is_ambiguous(scales: torch.Tensor, tol: float = 1e-5) -> torch.Tensor:
    """Keypoints whose float64 log2(pyramid scale) = log2(6 size / 16) lies within tol of an integer >= 1: float32 and
    float64 may pick different levels for them."""
    v = torch.log2(6.0 * scales.double() / 16.0)
    return ((v - v.round()).abs() < tol) & (v.round() >= 1)


# ---------------------------------------------------------------------------------------------------------- kornia stand-ins
class HardNet(torch.nn.Module):
    """Stand-in for kornia.feature.HardNet: ``HardNet(True)`` runs :func:`hardnet` with ``HardNet.state_dict_source``."""

    state_dict_source: dict = {}

    def __init__(self, pretrained: bool = False):
        super().__init__()
        self.sd = dict(self.state_dict_source)

    def forward(self, patches: torch.Tensor) -> torch.Tensor:
        return hardnet(self.sd, patches)


class LAFDescriptor(torch.nn.Module):
    """Stand-in for kornia.feature.LAFDescriptor(patch_descriptor_module, patch_size=32, grayscale_descriptor=True)."""

    def __init__(self, patch_descriptor_module=None, patch_size: int = 32, grayscale_descriptor: bool = True):
        super().__init__()
        self.descriptor = patch_descriptor_module
        self.grayscale_descriptor = grayscale_descriptor

    def forward(self, img: torch.Tensor, lafs: torch.Tensor) -> torch.Tensor:
        if self.grayscale_descriptor:
            img = gray(img)
        out = [self.descriptor(extract_patches(img[i:i + 1], lafs[i])) for i in range(img.shape[0])]
        return torch.stack(out)


def level_count(h: int, w: int) -> int:
    """Number of pyramid levels extract_patches_from_pyramid samples for an h x w image."""
    n = 1
    while min(h, w) >= PS:
        h, w = int(float(h) / 2.0), w // 2
        n += 1
    return n
