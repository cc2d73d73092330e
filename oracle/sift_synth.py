"""Seeded synthetic images for the SIFT extractor (torch only: the GPU tests regenerate them without cv2).

An image is a smooth random field plus discs, rectangles and straight edges at several scales, in [0, 1], which gives
a few hundred OpenCV SIFT keypoints at 240x320.  ``exact_levels=True`` snaps every value to k / 255 (as fp32) and
repeats channel 0 in every channel: the gray value of such an RGB pixel lands just below k / 255 at some pixels, where
the reference's ``(image * 255).astype(uint8)`` truncation gives k - 1."""
from __future__ import annotations

import math

import torch


def make_image(h: int, w: int, b: int = 1, seed: int = 0, channels: int = 1, exact_levels: bool = False) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    out = []
    ys = torch.arange(h, dtype=torch.float64)[:, None]
    xs = torch.arange(w, dtype=torch.float64)[None, :]
    for _ in range(b):
        chans = []
        for _c in range(channels):
            # smooth field: a few low-frequency cosines
            img = torch.full((h, w), 0.5, dtype=torch.float64)
            for _k in range(6):
                fy, fx, ph, a = torch.rand(4, generator=g, dtype=torch.float64).unbind()
                img += 0.08 * a * torch.cos(2 * math.pi * (fy * 3 * ys / h + fx * 3 * xs / w) + 6.283 * ph)
            n_shapes = max(8, h * w // 600)
            for _k in range(n_shapes):
                kind = int(torch.randint(0, 3, (1,), generator=g))
                cy, cx = float(torch.rand(1, generator=g)) * h, float(torch.rand(1, generator=g)) * w
                size = 2.0 + float(torch.rand(1, generator=g)) ** 2 * min(h, w) / 6
                val = float(torch.rand(1, generator=g)) * 0.8 - 0.4
                if kind == 0:  # disc
                    m = ((ys - cy) ** 2 + (xs - cx) ** 2) <= size * size
                elif kind == 1:  # rectangle
                    sy = size * (0.5 + float(torch.rand(1, generator=g)))
                    m = ((ys - cy).abs() <= sy) & ((xs - cx).abs() <= size)
                else:  # half-plane edge through (cy, cx), limited to a band
                    t = float(torch.rand(1, generator=g)) * math.pi
                    d = (ys - cy) * math.cos(t) + (xs - cx) * math.sin(t)
                    m = (d > 0) & (((ys - cy) ** 2 + (xs - cx) ** 2) <= (3 * size) ** 2)
                img = torch.where(m, img + val, img)
            chans.append(img.clamp(0.0, 1.0))
        out.append(torch.stack(chans))
    img = torch.stack(out).to(torch.float32)
    if exact_levels:
        img = torch.round(img * 255.0).to(torch.float32) / 255.0
        img = img[:, :1].expand(-1, channels, -1, -1)
    return img.contiguous()
