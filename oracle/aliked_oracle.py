"""Pure-torch restatement of the ALIKED forward (reference lightglue/aliked.py), CPU, fp32, no torchvision.

What the GPU tests compare against at image sizes that have no fixture; pinned to the reference itself by
tests/test_aliked_oracle_golden.py.  Written from the algorithm, not from the reference's code:
  * the deformable convolution is explicit bilinear sampling: tap (i, j) of output pixel (y, x) reads the input at
    (y - 1 + i + dy, x - 1 + j + dx) with the offset pair (dy, dx) stored as channels (2 t, 2 t + 1), t = 3 i + j, and
    torchvision's zero-outside rule (a sample whose position lies at or beyond one pixel outside the map is 0, and each
    bilinear corner outside the map contributes 0);
  * BatchNorm runs in eval mode (running statistics, eps 1e-5);
  * ``forward`` returns per-image lists (keypoints in pixels, scores, descriptors) plus the integer NMS positions.
Differences from the reference on purpose: with ``image_size`` each image's positions are decoded with the score map's
width (the reference decodes every image with the last image's ``image_size``), and in top-k mode an image with fewer
than k NMS maxima is filled with zero-score pixels in row-major order.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch
import torch.nn.functional as F

N_LIMIT_MAX = 20000
CFGS = {
    "aliked-t16": [8, 16, 32, 64, 64, 3, 16],
    "aliked-n16": [16, 32, 64, 128, 128, 3, 16],
    "aliked-n16rot": [16, 32, 64, 128, 128, 3, 16],
    "aliked-n32": [16, 32, 64, 128, 128, 3, 32],
}


def _bn(x, sd, p):
    return F.batch_norm(x, sd[f"{p}.running_mean"], sd[f"{p}.running_var"], sd[f"{p}.weight"], sd[f"{p}.bias"], False, 0.0, 1e-5)


def _bilinear_zero(x, py, px):
    """x [C, H, W]; py, px [...] float sample positions -> [C, ...]; torchvision deform_conv2d's outside rule."""
    c, h, w = x.shape
    inside = (py > -1) & (py < h) & (px > -1) & (px < w)
    y0, x0 = torch.floor(py), torch.floor(px)
    ly, lx = py - y0, px - x0
    y0, x0 = y0.long(), x0.long()
    out = torch.zeros((c,) + py.shape, dtype=x.dtype)
    for yy, xx, wt in ((y0, x0, (1 - ly) * (1 - lx)), (y0, x0 + 1, (1 - ly) * lx), (y0 + 1, x0, ly * (1 - lx)), (y0 + 1, x0 + 1, ly * lx)):
        ok = inside & (yy >= 0) & (yy < h) & (xx >= 0) & (xx < w)
        v = x[:, yy.clamp(0, h - 1), xx.clamp(0, w - 1)]
        out = out + torch.where(ok, wt, torch.zeros_like(wt)) * torch.where(ok, v, torch.zeros_like(v))
    return out


def deform_conv3x3(x, offset, weight):
    """x [B, Ci, H, W], offset [B, 18, H, W], weight [Co, Ci, 3, 3] -> [B, Co, H, W] (stride 1, padding 1, no bias)."""
    b, ci, h, w = x.shape
    ys = torch.arange(h, dtype=x.dtype)[:, None].expand(h, w)
    xs = torch.arange(w, dtype=x.dtype)[None, :].expand(h, w)
    outs = []
    for ib in range(b):
        cols = []
        for i in range(3):
            for j in range(3):
                t = 3 * i + j
                py = ys - 1 + i + offset[ib, 2 * t]
                px = xs - 1 + j + offset[ib, 2 * t + 1]
                cols.append(_bilinear_zero(x[ib], py, px))  # [Ci, H, W]
        col = torch.stack(cols, 1).reshape(ci * 9, h * w)  # im2col: row (ci, tap)
        outs.append((weight.reshape(weight.shape[0], ci * 9) @ col).reshape(-1, h, w))
    return torch.stack(outs)


def _selu(x):
    return F.selu(x)


def _conv(x, wt, bias=None, pad=1):
    return F.conv2d(x, wt, bias, padding=pad)


def _dcn(x, sd, p):
    h, w = x.shape[-2:]
    lim = max(h, w) / 4.0
    off = _conv(x, sd[f"{p}.offset_conv.weight"], sd[f"{p}.offset_conv.bias"]).clamp(-lim, lim)
    return deform_conv3x3(x, off, sd[f"{p}.regular_conv.weight"])


def _block(x, sd, p, dcn, res):
    conv = (lambda t, q: _dcn(t, sd, q)) if dcn else (lambda t, q: _conv(t, sd[f"{q}.weight"]))
    y = _selu(_bn(conv(x, f"{p}.conv1"), sd, f"{p}.bn1"))
    y = _bn(conv(y, f"{p}.conv2"), sd, f"{p}.bn2")
    if res:
        y = y + _conv(x, sd[f"{p}.downsample.weight"], sd[f"{p}.downsample.bias"], pad=0)
    return _selu(y)


def _pads(h, w, div=32):
    ph, pw = (-h) % div, (-w) % div
    return pw // 2, pw - pw // 2, ph // 2, ph - ph // 2


def dense_maps(sd, image):
    """(normalised feature map [B, dim, H, W], score map [B, 1, H, W]) of extract_dense_map."""
    h, w = image.shape[-2:]
    l, r, t, bt = _pads(h, w)
    x = F.pad(image, (l, r, t, bt), mode="replicate")
    x1 = _block(x, sd, "block1", False, False)
    x2 = _block(F.avg_pool2d(x1, 2), sd, "block2", False, True)
    x3 = _block(F.avg_pool2d(x2, 4), sd, "block3", True, True)
    x4 = _block(F.avg_pool2d(x3, 4), sd, "block4", True, True)
    a = [_selu(_conv(v, sd[f"conv{i}.weight"], pad=0)) for i, v in enumerate((x1, x2, x3, x4), 1)]
    size = x1.shape[-2:]
    up = [a[0]] + [F.interpolate(v, size=size, mode="bilinear", align_corners=True) for v in a[1:]]
    x1234 = torch.cat(up, 1)
    s = _selu(_conv(x1234, sd["score_head.0.weight"], pad=0))
    s = _selu(_conv(s, sd["score_head.2.weight"]))
    s = _selu(_conv(s, sd["score_head.4.weight"]))
    score = torch.sigmoid(_conv(s, sd["score_head.6.weight"]))
    feat = F.normalize(x1234, p=2, dim=1)
    hp, wp = x1234.shape[-2:]
    return feat[..., t:hp - bt, l:wp - r], score[..., t:hp - bt, l:wp - r]


def _simple_nms(s, r):
    mp = lambda t: F.max_pool2d(t, 2 * r + 1, stride=1, padding=r)  # noqa: E731
    zeros = torch.zeros_like(s)
    mask = s == mp(s)
    for _ in range(2):
        supp = mp(mask.float()) > 0
        ss = torch.where(supp, zeros, s)
        mask = mask | ((ss == mp(ss)) & ~supp)
    return torch.where(mask, s, zeros)


def _grid_sample_pts(x, pts):
    """x [C, H, W], pts [N, 2] in [-1, 1] (x, y) -> [C, N]: grid_sample bilinear, align_corners=True, zeros."""
    return F.grid_sample(x[None], pts.view(1, 1, -1, 2), mode="bilinear", align_corners=True)[0, :, 0, :]


def forward(sd, image, model_name="aliked-n16", max_num_keypoints=-1, detection_threshold=0.2, nms_radius=2,
            image_size: Optional[torch.Tensor] = None) -> Dict[str, list]:
    c1, c2, c3, c4, dim, K, M = CFGS[model_name]
    top_k = -1 if detection_threshold > 0 else max_num_keypoints
    n_limit = max_num_keypoints if max_num_keypoints > 0 else N_LIMIT_MAX
    feat, score = dense_maps(sd, image)
    b, _, h, w = score.shape
    r = nms_radius
    nms = _simple_nms(score, r)
    nms[:, :, :r, :] = 0
    nms[:, :, :, :r] = 0
    if image_size is not None:
        for i in range(b):
            wi, hi = (int(v) for v in image_size[i].long())
            nms[i, :, hi - r:, :] = 0
            nms[i, :, :, wi - r:] = 0
    else:
        nms[:, :, -r:, :] = 0
        nms[:, :, :, -r:] = 0
    flat = nms.reshape(b, -1)
    idx = []
    if top_k > 0:
        for i in range(b):  # score descending, lower index first among equals; zero-score filler in row-major order
            pos = torch.nonzero(flat[i] > 0)[:, 0]
            pos = pos[torch.argsort(-flat[i, pos], stable=True)]
            if len(pos) < top_k:
                pos = torch.cat([pos, torch.nonzero(flat[i] <= 0)[:, 0][: top_k - len(pos)]])
            idx.append(pos[:top_k])
    else:
        if detection_threshold > 0:
            masks = flat > detection_threshold
            if masks.sum() == 0:
                masks = flat > score.reshape(b, -1).mean(dim=1)[:, None]
        else:
            masks = flat > score.reshape(b, -1).mean(dim=1)[:, None]
        for i in range(b):
            pos = masks[i].nonzero()[:, 0]
            if len(pos) > n_limit:
                o = torch.argsort(-flat[i, pos], stable=True)
                pos = pos[o[:n_limit]]
            idx.append(pos)
    wh = torch.tensor([w - 1, h - 1], dtype=torch.float32)
    ks = 2 * r + 1
    lin = torch.linspace(-r, r, ks)
    grid = torch.stack([lin.repeat(ks), lin.repeat_interleave(ks)], 1)  # tap (ky, kx) -> (dx, dy)
    patches = F.unfold(score, kernel_size=ks, padding=r)  # [B, ks*ks, H*W]
    out = {"keypoints": [], "keypoint_scores": [], "descriptors": [], "nms_positions": []}
    lim = max(h, w) / 4.0
    for i in range(b):
        pos = idx[i]
        xy = torch.stack([pos % w, torch.div(pos, w, rounding_mode="trunc")], 1)
        p = patches[i].t()[pos]
        e = ((p - p.max(dim=1).values[:, None]) / 0.1).exp()
        res = e @ grid / e.sum(dim=1)[:, None]
        kp = (xy + res) / wh * 2 - 1
        kscore = _grid_sample_pts(score[i], kp)[0]
        # SDDH
        kwh = (kp / 2 + 0.5) * wh
        corner = (kwh.long() - K / 2 + 1).long()
        corner[:, 0] = corner[:, 0].clamp(min=0, max=w - 1 - K)
        corner[:, 1] = corner[:, 1].clamp(min=0, max=h - 1 - K)
        ar = torch.arange(K)
        py = corner[:, 1, None, None] + ar[None, :, None]
        px = corner[:, 0, None, None] + ar[None, None, :]
        patch = feat[i][:, py, px].permute(1, 0, 2, 3)  # [N, C, K, K]
        o = F.conv2d(patch, sd["desc_head.offset_conv.0.weight"], sd["desc_head.offset_conv.0.bias"])
        o = F.conv2d(_selu(o), sd["desc_head.offset_conv.2.weight"], sd["desc_head.offset_conv.2.bias"]).clamp(-lim, lim)
        off = o[:, :, 0, 0].view(-1, 2, M).permute(0, 2, 1)  # [N, M, (dx, dy)]
        spos = (kwh[:, None, :] + off) * 2.0 / wh - 1
        f = _grid_sample_pts(feat[i], spos.reshape(-1, 2)).reshape(dim, -1, M).permute(1, 0, 2)  # [N, C, M]
        f = _selu(torch.einsum("dc,ncm->ndm", sd["desc_head.sf_conv.weight"][:, :, 0, 0], f))
        d = F.normalize(torch.einsum("ncp,pcd->nd", f, sd["desc_head.agg_weights"]), p=2, dim=1)
        out["keypoints"].append(wh * (kp + 1) / 2.0)
        out["keypoint_scores"].append(kscore)
        out["descriptors"].append(d)
        out["nms_positions"].append(xy)
    return out

