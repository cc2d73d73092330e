"""Pure-torch restatement of the ALIKED forward (reference lightglue/aliked.py), no torchvision, in stages.

What the GPU tests compare against at image sizes that have no fixture; pinned to the reference itself by
tests/test_aliked_oracle_golden.py.  Every stage takes tensors of any floating dtype on any device, so the per-stage GPU
checks (tests/test_gpu_aliked_layers.py) apply them in float64 to the kernels' own inputs, and the calibration
(tests/test_aliked_layer_emulation.py) runs them in fp32 on the CPU with the defect switches some stages take.
``forward`` composes the stages.  Written from the algorithm, not from the reference's code:
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


def _bn(x, sd, p, nobias=False):
    if nobias:  # the folded bias beta - mean * gamma / sqrt(var + eps) lost: only the scale is applied
        z = torch.zeros_like(sd[f"{p}.bias"])
        return F.batch_norm(x, z, sd[f"{p}.running_var"], sd[f"{p}.weight"], z, False, 0.0, 1e-5)
    return F.batch_norm(x, sd[f"{p}.running_mean"], sd[f"{p}.running_var"], sd[f"{p}.weight"], sd[f"{p}.bias"], False, 0.0, 1e-5)


def _bilinear_zero(x, py, px, edge=False):
    """x [C, H, W]; py, px [...] float sample positions -> [C, ...]; torchvision deform_conv2d's outside rule
    (``edge``: clamp-to-edge instead, a defect)."""
    c, h, w = x.shape
    if edge:
        py, px = py.clamp(0, h - 1), px.clamp(0, w - 1)
    inside = (py > -1) & (py < h) & (px > -1) & (px < w)
    y0, x0 = torch.floor(py), torch.floor(px)
    ly, lx = py - y0, px - x0
    y0, x0 = y0.long(), x0.long()
    out = torch.zeros((c,) + py.shape, dtype=x.dtype, device=x.device)
    for yy, xx, wt in ((y0, x0, (1 - ly) * (1 - lx)), (y0, x0 + 1, (1 - ly) * lx), (y0 + 1, x0, ly * (1 - lx)), (y0 + 1, x0 + 1, ly * lx)):
        ok = inside & (yy >= 0) & (yy < h) & (xx >= 0) & (xx < w)
        v = x[:, yy.clamp(0, h - 1), xx.clamp(0, w - 1)]
        out = out + torch.where(ok, wt, torch.zeros_like(wt)) * torch.where(ok, v, torch.zeros_like(v))
    return out


def deform_conv3x3(x, offset, weight, swap=False, edge=False):
    """x [B, Ci, H, W], offset [B, 18, H, W], weight [Co, Ci, 3, 3] -> [B, Co, H, W] (stride 1, padding 1, no bias).
    Defects: ``swap`` reads (dx, dy) from channels (2 t, 2 t + 1); ``edge`` clamps taps to the map."""
    b, ci, h, w = x.shape
    ys = torch.arange(h, dtype=x.dtype, device=x.device)[:, None].expand(h, w)
    xs = torch.arange(w, dtype=x.dtype, device=x.device)[None, :].expand(h, w)
    outs = []
    for ib in range(b):
        cols = []
        for i in range(3):
            for j in range(3):
                t = 3 * i + j
                dy, dx = offset[ib, 2 * t], offset[ib, 2 * t + 1]
                if swap:
                    dy, dx = dx, dy
                cols.append(_bilinear_zero(x[ib], ys - 1 + i + dy, xs - 1 + j + dx, edge))  # [Ci, H, W]
        col = torch.stack(cols, 1).reshape(ci * 9, h * w)  # im2col: row (ci, tap)
        outs.append((weight.reshape(weight.shape[0], ci * 9) @ col).reshape(-1, h, w))
    return torch.stack(outs)


def _selu(x):
    return F.selu(x)


def _conv(x, wt, bias=None, pad=1):
    return F.conv2d(x, wt, bias, padding=pad)


def _drop_tail(y, drop_tail):
    """Defect: the outputs of the last partial 4-pixel group of each row left at zero."""
    if drop_tail and y.shape[-1] % 4:
        y = y.clone()
        y[..., y.shape[-1] // 4 * 4:] = 0
    return y


# ----------------------------------------------------------------------------------------------------------- encoder
def _pads(h, w, div=32):
    ph, pw = (-h) % div, (-w) % div
    return pw // 2, pw - pw // 2, ph // 2, ph - ph // 2


def pad(image):
    """InputPadder: replicate-pad [B, 3, H, W] to multiples of 32."""
    return F.pad(image, _pads(*image.shape[-2:]), mode="replicate")


def pool(x, k):
    return F.avg_pool2d(x, k)


def offsets(sd, p, x, lim_min=False, drop_group=False, drop_tail=False):
    """The offset convolution of the deformable layer ``p`` (``block3.conv1`` ...) + bias, clamped to
    +-max(h, w) / 4 -> [B, 18, h, w].  Defects: ``lim_min`` clamps at min(h, w) / 4; ``drop_group`` leaves channels 16,
    17 (the last group of 8) at zero; ``drop_tail`` see _drop_tail."""
    h, w = x.shape[-2:]
    lim = (min(h, w) if lim_min else max(h, w)) / 4.0
    off = _drop_tail(_conv(x, sd[f"{p}.offset_conv.weight"], sd[f"{p}.offset_conv.bias"]).clamp(-lim, lim), drop_tail)
    if drop_group:
        off = off.clone()
        off[:, 16:] = 0
    return off


def conv_bn(sd, blk, k, x, off=None, nobias=False, swap=False, edge=False, **off_defects):
    """BN(conv k of block ``blk``)(x), before the activation; block3 / block4: deformable, with the given offsets or, when
    ``off`` is None, ``offsets`` of x.  Defects: ``nobias`` loses the folded-BN bias; ``swap`` / ``edge`` see
    deform_conv3x3; the rest go to ``offsets``."""
    p = f"{blk}.conv{k}"
    if f"{p}.offset_conv.weight" in sd:
        if off is None:
            off = offsets(sd, p, x, **off_defects)
        y = deform_conv3x3(x, off, sd[f"{p}.regular_conv.weight"], swap, edge)
    else:
        y = _conv(x, sd[f"{p}.weight"])
    return _bn(y, sd, f"{blk}.bn{k}", nobias)


def downsample(sd, blk, x, nobias=False, drop_tail=False):
    """The ResBlock's 1x1 downsample + bias."""
    return _drop_tail(_conv(x, sd[f"{blk}.downsample.weight"], None if nobias else sd[f"{blk}.downsample.bias"], pad=0),
                      drop_tail)


def block_out(sd, blk, t, d, off=None, nores=False, **defects):
    """The ResBlock's output SELU(BN(conv2 t) + d) from t = SELU(BN(conv1 x)) and the downsample d (``nores``: a dropped
    residual, a defect)."""
    y = conv_bn(sd, blk, 2, t, off, **defects)
    return _selu(y if nores else y + d)


def block(sd, i, x):
    """block{i} (1 .. 4) of the encoder on its input (the padded image, or the pooled previous output)."""
    blk = f"block{i}"
    t = _selu(conv_bn(sd, blk, 1, x))
    if i == 1:
        return _selu(conv_bn(sd, blk, 2, t))
    return block_out(sd, blk, t, downsample(sd, blk, x))


def encoder(sd, xp):
    """x1 .. x4 from the padded image."""
    x1 = block(sd, 1, xp)
    x2 = block(sd, 2, pool(x1, 2))
    x3 = block(sd, 3, pool(x2, 4))
    x4 = block(sd, 4, pool(x3, 4))
    return x1, x2, x3, x4


# ----------------------------------------------------------------------------------------------------------- head
def aggregate(sd, i, x, drop_tail=False):
    """a_i = SELU(conv{i} x_i) (1x1, dim / 4 channels) at x_i's resolution."""
    return _drop_tail(_selu(_conv(x, sd[f"conv{i}.weight"], pad=0)), drop_tail)


def upsample(a, align_corners=True):
    """x1234 = cat(a1, up2(a2), up8(a3), up32(a4)) [B, dim, Hp, Wp] (bilinear; ``align_corners=False``: a defect)."""
    size = a[0].shape[-2:]
    return torch.cat([a[0]] + [F.interpolate(v, size=size, mode="bilinear", align_corners=align_corners) for v in a[1:]], 1)


def inv_norm(x1234):
    """1 / max(|x1234|, 1e-12) per pixel [B, Hp, Wp] (F.normalize's divisor)."""
    return 1.0 / x1234.norm(p=2, dim=1).clamp_min(1e-12)


def score_layer(sd, k, s):
    """score_head.{k}: 0 (1x1 dim -> 8, SELU), 2 (3x3 8 -> 4, SELU), 4 (3x3 4 -> 4, SELU), 6 (3x3 4 -> 1, sigmoid)."""
    if k == 0:
        return _selu(_conv(s, sd["score_head.0.weight"], pad=0))
    y = _conv(s, sd[f"score_head.{k}.weight"])
    return torch.sigmoid(y) if k == 6 else _selu(y)


def score_head(sd, x1234):
    s = x1234
    for k in (0, 2, 4, 6):
        s = score_layer(sd, k, s)
    return s


def crop(m, h, w):
    """The [h, w] image inside the padded frame of map m [..., Hp, Wp]."""
    l, r, t, bt = _pads(h, w)
    hp, wp = m.shape[-2:]
    return m[..., t:t + h, l:wp - r]


def dense_maps(sd, image, padded=False):
    """(normalised feature map [B, dim, H, W], score map [B, 1, H, W]) of extract_dense_map; ``padded``: both on the
    padded frame, before the crop."""
    h, w = image.shape[-2:]
    xs = encoder(sd, pad(image))
    x1234 = upsample([aggregate(sd, i, v) for i, v in enumerate(xs, 1)])
    score = score_head(sd, x1234)
    feat = F.normalize(x1234, p=2, dim=1)
    if padded:
        return feat, score
    return crop(feat, h, w), crop(score, h, w)


# ----------------------------------------------------------------------------------------------------------- DKD
def _simple_nms(s, r):
    mp = lambda t: F.max_pool2d(t, 2 * r + 1, stride=1, padding=r)  # noqa: E731
    zeros = torch.zeros_like(s)
    mask = s == mp(s)
    for _ in range(2):
        supp = mp(mask.float()) > 0
        ss = torch.where(supp, zeros, s)
        mask = mask | ((ss == mp(ss)) & ~supp)
    return torch.where(mask, s, zeros)


def nms_borders(score, r, image_size=None):
    """simple_nms of the score map [B, 1, H, W] with the borders zeroed: the first r rows / columns, and the last r, or
    with ``image_size`` (w, h per image) rows >= h - r and columns >= w - r (Python's slice rule: a negative start
    counts from the end)."""
    nms = _simple_nms(score, r)
    nms[:, :, :r, :] = 0
    nms[:, :, :, :r] = 0
    if image_size is not None:
        for i in range(score.shape[0]):
            wi, hi = (int(v) for v in image_size[i].long())
            nms[i, :, hi - r:, :] = 0
            nms[i, :, :, wi - r:] = 0
    else:
        nms[:, :, -r:, :] = 0
        nms[:, :, :, -r:] = 0
    return nms


def thresholds(nms, score, detection_threshold):
    """Per-image threshold of threshold mode: detection_threshold, or the image's mean score when it is <= 0 or no
    NMS value of the whole batch passes it -> [B, 1]."""
    b = nms.shape[0]
    flat = nms.reshape(b, -1)
    mean = score.reshape(b, -1).mean(dim=1)[:, None]
    if detection_threshold > 0 and bool((flat > detection_threshold).any()):
        return torch.full_like(mean, detection_threshold)
    return mean


def select(nms, score, detection_threshold, max_num_keypoints, thr=None):
    """Flat NMS positions per image, in output order: top-k mode (``detection_threshold <= 0`` and k > 0) by descending
    score, lower index first among equals, filled up with zero-score pixels in row-major order; threshold mode in
    row-major order, or by descending score when more than n_limit pass.  ``thr`` [B, 1] replaces ``thresholds``."""
    b = nms.shape[0]
    top_k = -1 if detection_threshold > 0 else max_num_keypoints
    n_limit = max_num_keypoints if max_num_keypoints > 0 else N_LIMIT_MAX
    flat = nms.reshape(b, -1)
    idx = []
    if top_k > 0:
        for i in range(b):
            pos = torch.nonzero(flat[i] > 0)[:, 0]
            pos = pos[torch.argsort(-flat[i, pos], stable=True)]
            if len(pos) < top_k:
                pos = torch.cat([pos, torch.nonzero(flat[i] <= 0)[:, 0][: top_k - len(pos)]])
            idx.append(pos[:top_k])
    else:
        masks = flat > (thresholds(nms, score, detection_threshold) if thr is None else thr)
        for i in range(b):
            pos = masks[i].nonzero()[:, 0]
            if len(pos) > n_limit:
                o = torch.argsort(-flat[i, pos], stable=True)
                pos = pos[o[:n_limit]]
            idx.append(pos)
    return idx


def _grid_sample_pts(x, pts):
    """x [C, H, W], pts [N, 2] in [-1, 1] (x, y) -> [C, N]: grid_sample bilinear, align_corners=True, zeros."""
    return F.grid_sample(x[None], pts.view(1, 1, -1, 2), mode="bilinear", align_corners=True)[0, :, 0, :]


def soft_argmax(score, pos, r, temperature=0.1):
    """score [1, H, W] of one image, flat positions pos [N] -> (normalised keypoints [N, 2] (x, y) in [-1, 1], scores
    [N] sampled there, integer positions [N, 2]): the (2r+1)^2 window's soft-argmax (zero padded)."""
    h, w = score.shape[-2:]
    wh = torch.tensor([w - 1, h - 1], dtype=score.dtype, device=score.device)
    ks = 2 * r + 1
    lin = torch.linspace(-r, r, ks, dtype=score.dtype, device=score.device)
    grid = torch.stack([lin.repeat(ks), lin.repeat_interleave(ks)], 1)  # tap (ky, kx) -> (dx, dy)
    patches = F.unfold(score[None], kernel_size=ks, padding=r)[0]  # [ks*ks, H*W]
    xy = torch.stack([pos % w, torch.div(pos, w, rounding_mode="trunc")], 1)
    p = patches.t()[pos]
    e = ((p - p.max(dim=1).values[:, None]) / temperature).exp()
    res = e @ grid / e.sum(dim=1)[:, None]
    kp = (xy + res) / wh * 2 - 1
    return kp, _grid_sample_pts(score, kp)[0], xy


def pixels(kp, h, w):
    """Normalised keypoints -> pixels."""
    wh = torch.tensor([w - 1, h - 1], dtype=kp.dtype, device=kp.device)
    return wh * (kp + 1) / 2.0


# ----------------------------------------------------------------------------------------------------------- SDDH
def sddh(sd, featp, box, kp, M, K=3, swap=False, padded=False, agg_t=False):
    """Descriptors [N, dim] of one image: featp [dim, Hp, Wp] the normalised feature map on the padded frame, box =
    (top, left, h, w) the image inside it, kp [N, 2] normalised keypoints.  The patch corner comes from the fp32
    rounding of (kp / 2 + 0.5) * (w - 1, h - 1), whatever kp's dtype.  Defects: ``swap`` reads the offsets as
    (dy, dx); ``padded`` samples the padded frame, zero only outside it; ``agg_t`` transposes agg_weights."""
    t, l, h, w = box
    feat = featp[:, t:t + h, l:l + w]
    wh = torch.tensor([w - 1, h - 1], dtype=kp.dtype, device=kp.device)
    kwh = (kp / 2 + 0.5) * wh
    kwh32 = kwh if kp.dtype == torch.float32 else (kp.float() / 2 + 0.5) * wh.float()
    corner = (kwh32.long() - K / 2 + 1).long()
    corner[:, 0] = corner[:, 0].clamp(min=0, max=w - 1 - K)
    corner[:, 1] = corner[:, 1].clamp(min=0, max=h - 1 - K)
    ar = torch.arange(K, device=kp.device)
    py = corner[:, 1, None, None] + ar[None, :, None]
    px = corner[:, 0, None, None] + ar[None, None, :]
    patch = feat[:, py, px].permute(1, 0, 2, 3)  # [N, C, K, K]
    lim = max(h, w) / 4.0
    o = F.conv2d(patch, sd["desc_head.offset_conv.0.weight"], sd["desc_head.offset_conv.0.bias"])
    o = F.conv2d(_selu(o), sd["desc_head.offset_conv.2.weight"], sd["desc_head.offset_conv.2.bias"]).clamp(-lim, lim)
    off = o[:, :, 0, 0].view(-1, 2, M).permute(0, 2, 1)  # [N, M, (dx, dy)]
    if swap:
        off = off.flip(-1)
    dim = featp.shape[0]
    if padded:
        hp, wp = featp.shape[-2:]
        fwh = torch.tensor([wp - 1, hp - 1], dtype=kp.dtype, device=kp.device)
        shift = torch.tensor([l, t], dtype=kp.dtype, device=kp.device)
        f = _grid_sample_pts(featp, ((kwh[:, None, :] + off + shift) * 2.0 / fwh - 1).reshape(-1, 2))
    else:
        spos = (kwh[:, None, :] + off) * 2.0 / wh - 1
        f = _grid_sample_pts(feat, spos.reshape(-1, 2))
    f = f.reshape(dim, -1, M).permute(1, 0, 2)  # [N, C, M]
    f = _selu(torch.einsum("dc,ncm->ndm", sd["desc_head.sf_conv.weight"][:, :, 0, 0], f))
    agg = sd["desc_head.agg_weights"]
    if agg_t:
        agg = agg.transpose(1, 2)
    return F.normalize(torch.einsum("ncp,pcd->nd", f, agg), p=2, dim=1)


def forward(sd, image, model_name="aliked-n16", max_num_keypoints=-1, detection_threshold=0.2, nms_radius=2,
            image_size: Optional[torch.Tensor] = None) -> Dict[str, list]:
    c1, c2, c3, c4, dim, K, M = CFGS[model_name]
    h, w = image.shape[-2:]
    featp, scorep = dense_maps(sd, image, padded=True)
    score = crop(scorep, h, w)
    l, _, t, _ = _pads(h, w)
    nms = nms_borders(score, nms_radius, image_size)
    idx = select(nms, score, detection_threshold, max_num_keypoints)
    out = {"keypoints": [], "keypoint_scores": [], "descriptors": [], "nms_positions": []}
    for i in range(score.shape[0]):
        kp, kscore, xy = soft_argmax(score[i], idx[i], nms_radius)
        out["keypoints"].append(pixels(kp, h, w))
        out["keypoint_scores"].append(kscore)
        out["descriptors"].append(sddh(sd, featp[i], (t, l, h, w), kp, M, K))
        out["nms_positions"].append(xy)
    return out
