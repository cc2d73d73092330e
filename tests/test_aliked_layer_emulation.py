"""Calibration of the per-stage tolerances of tests/test_gpu_aliked_layers.py and of the end-to-end gates of
tests/test_gpu_aliked.py (ALIKED, fp32 on CUDA cores).

Each GPU check applies a float64 stage of ``oracle/aliked_oracle.py`` to the kernels' own fp32 input and compares the
kernels' output with it.  The emulation is the same stage in fp32 on the CPU, applied to the fp32 chain's own values;
each tolerance must be at least 3x the emulated error and at most 1/3 of every defect listed for it, each defect being
a switch of the stage functions.  Measure: max|delta| / max|ref| per image; keypoints relative to the image's extent
max(w - 1, h - 1), keypoint scores and unit descriptors absolute.  The stages whose error grows with the image's
extent (the keypoint, its score and SDDH, all through the fp32 rounding of normalised coordinates) are also placed at
768 x 1024, the largest image of tests/test_gpu_aliked_layers.py.

The end-to-end gates of tests/test_gpu_aliked.py keep the values that file asserted before they were derived here (its
assertions are not loosened).  On the images of its reference fixtures one fp32 forward is within e of float64, and
every listed defect moves the outputs by at least 3x the gates; but the gates are only 1.5x (scores, t16 fixture) to
3.8x (keypoints) e, not 3x everywhere, because each side of that comparison rounds in fp32 on its own.  The per-stage
checks are the ones placed by the 3x / 1/3 rule.

Checks without a listed defect: the poolings (a 2x2 / 4x4 mean has no switch a kernel could get subtly wrong: a wrong
window is a wrong map), a2 and a3 (bias-free 1x1 convolutions; the partial-group defect is listed where a level is
narrower than the group, at 1/32) and the score head's 3x3 layers (bias-free; a wrong tap moves a layer by O(1)).  The
crop has no tolerance to place: the GPU test compares it bit for bit, which is what catches a crop one row off.  A
clamp at min(h, w) / 4 is invisible on a square level (33x47 pads to 64x64), and SDDH samples bounded by the padded
frame instead of the crop are invisible without padding (768 x 1024); the other shapes resolve both.
"""
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import aliked_oracle as alo
from oracle import aliked_synth as als

TOL = {
    "x1": 1e-5,      # block1 (two 3x3 convolutions) from the padded image
    "pool": 1e-6,    # p1, p2, p3 from x1, x2, x3
    "conv": 1e-5,    # d2, t2, d3, d4 from p; x2 .. x4 from t, d (and o); a2 .. a4 from x
    "dcn": 1e-5,     # t3, t4 from p, with the offsets in float64
    "offset": 1e-5,  # o3, o4 from t
    "head": 2e-5,    # s1 and invn from x1 and a2 .. a4 (x1234 evaluated at every padded pixel)
    "score": 1e-5,   # s2, s3 and the pre-crop score, each from its predecessor
    "kpt": 5e-7,     # keypoints from the float64 soft-argmax at the selected positions of the fp32 score, relative to
                     # max(w - 1, h - 1): the fp32 normalised keypoint's rounding grows with the image's extent
    "kscore": 3e-5,  # keypoint scores, idem (absolute; placed at 768 x 1024, where it is largest)
    "desc": 3e-5,    # descriptors from float64 SDDH on the captured maps and normalised keypoints (placed at 768 x 1024)
    "mean": 1e-6,    # threshold mode's mean score, relative to the float64 mean
    "mean_margin": 1e-5,  # NMS values this close to the float64 mean (relative) are not decided by the fp32 mean
}
# tests/test_gpu_aliked.py: keypoints in pixels, scores and descriptors absolute (see the module docstring)
E2E_KPT, E2E_SCORE, E2E_DESC = 1e-4, 1e-5, 1e-5
# (model, H, W): odd pads, a 1/32 level narrower than a 4-pixel group (W3 = 5, 2, 3) and H != W
SHAPES = [("aliked-n16", 50, 145), ("aliked-t16", 33, 47), ("aliked-n32", 60, 90)]


def rel(a, ref):
    return float((a.double() - ref).abs().max() / ref.abs().max())


def absd(a, ref):
    return float((a.double() - ref).abs().max())


def assert_between(tol, emulated, defects):
    assert 3 * emulated <= tol, (emulated, tol)
    for name, dev in defects.items():
        assert dev >= 3 * tol, (name, dev, tol)


def D(t):
    return t.double()


@pytest.fixture(scope="module", params=SHAPES, ids=[f"{m[7:]}-{h}x{w}" for m, h, w in SHAPES])
def chain(request):
    """The fp32 chain of one image (what the kernels store), and the weights in fp32 and float64."""
    torch.set_grad_enabled(False)
    model_name, h, w = request.param
    sd = als.make_aliked_state_dict(model_name, 0)
    sd64 = {k: D(v) for k, v in sd.items()}
    c = {"model": model_name, "sd": sd, "sd64": sd64, "h": h, "w": w, "M": alo.CFGS[model_name][6]}
    c["xp"] = alo.pad(als.make_image(h, w, 1, 7))
    c["x1"] = alo.block(sd, 1, c["xp"])
    c["p1"] = alo.pool(c["x1"], 2)
    for i, prev in ((2, "p1"), (3, "p2"), (4, "p3")):
        blk, p = f"block{i}", c[prev]
        c[f"d{i}"] = alo.downsample(sd, blk, p)
        c[f"t{i}"] = F.selu(alo.conv_bn(sd, blk, 1, p))
        if i > 2:
            c[f"o{i}"] = alo.offsets(sd, f"{blk}.conv2", c[f"t{i}"])
        c[f"x{i}"] = alo.block_out(sd, blk, c[f"t{i}"], c[f"d{i}"], c.get(f"o{i}"))
        if i < 4:
            c[f"p{i}"] = alo.pool(c[f"x{i}"], 4)
    c["a"] = [alo.aggregate(sd, i, c[f"x{i}"]) for i in range(1, 5)]
    c["x1234"] = alo.upsample(c["a"])
    c["x1234_64"] = alo.upsample([alo.aggregate(sd64, 1, D(c["x1"]))] + [D(v) for v in c["a"][1:]])
    s = [alo.score_layer(sd, 0, c["x1234"])]
    for k in (2, 4, 6):
        s.append(alo.score_layer(sd, k, s[-1]))
    c["s"] = s
    c["score"] = alo.crop(s[-1], h, w)
    c["pos"] = alo.select(alo.nms_borders(c["score"], 2), c["score"], 0.2, -1)[0]
    assert len(c["pos"]) >= 10
    return c


# ------------------------------------------------------------------------------------ the oracle before the split
# A private copy of oracle/aliked_oracle.py as it was before its split into stages: ``forward`` must still compute
# exactly what this did.
def _pre_bn(x, sd, p):
    return F.batch_norm(x, sd[f"{p}.running_mean"], sd[f"{p}.running_var"], sd[f"{p}.weight"], sd[f"{p}.bias"], False, 0.0, 1e-5)


def _pre_bilinear_zero(x, py, px):
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


def _pre_deform_conv3x3(x, offset, weight):
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
                cols.append(_pre_bilinear_zero(x[ib], py, px))  # [Ci, H, W]
        col = torch.stack(cols, 1).reshape(ci * 9, h * w)  # im2col: row (ci, tap)
        outs.append((weight.reshape(weight.shape[0], ci * 9) @ col).reshape(-1, h, w))
    return torch.stack(outs)


def _pre_selu(x):
    return F.selu(x)


def _pre_conv(x, wt, bias=None, pad=1):
    return F.conv2d(x, wt, bias, padding=pad)


def _pre_dcn(x, sd, p):
    h, w = x.shape[-2:]
    lim = max(h, w) / 4.0
    off = _pre_conv(x, sd[f"{p}.offset_conv.weight"], sd[f"{p}.offset_conv.bias"]).clamp(-lim, lim)
    return _pre_deform_conv3x3(x, off, sd[f"{p}.regular_conv.weight"])


def _pre_block(x, sd, p, dcn, res):
    conv = (lambda t, q: _pre_dcn(t, sd, q)) if dcn else (lambda t, q: _pre_conv(t, sd[f"{q}.weight"]))
    y = _pre_selu(_pre_bn(conv(x, f"{p}.conv1"), sd, f"{p}.bn1"))
    y = _pre_bn(conv(y, f"{p}.conv2"), sd, f"{p}.bn2")
    if res:
        y = y + _pre_conv(x, sd[f"{p}.downsample.weight"], sd[f"{p}.downsample.bias"], pad=0)
    return _pre_selu(y)


def _pre_pads(h, w, div=32):
    ph, pw = (-h) % div, (-w) % div
    return pw // 2, pw - pw // 2, ph // 2, ph - ph // 2


def _pre_dense_maps(sd, image):
    """(normalised feature map [B, dim, H, W], score map [B, 1, H, W]) of extract_dense_map."""
    h, w = image.shape[-2:]
    l, r, t, bt = _pre_pads(h, w)
    x = F.pad(image, (l, r, t, bt), mode="replicate")
    x1 = _pre_block(x, sd, "block1", False, False)
    x2 = _pre_block(F.avg_pool2d(x1, 2), sd, "block2", False, True)
    x3 = _pre_block(F.avg_pool2d(x2, 4), sd, "block3", True, True)
    x4 = _pre_block(F.avg_pool2d(x3, 4), sd, "block4", True, True)
    a = [_pre_selu(_pre_conv(v, sd[f"conv{i}.weight"], pad=0)) for i, v in enumerate((x1, x2, x3, x4), 1)]
    size = x1.shape[-2:]
    up = [a[0]] + [F.interpolate(v, size=size, mode="bilinear", align_corners=True) for v in a[1:]]
    x1234 = torch.cat(up, 1)
    s = _pre_selu(_pre_conv(x1234, sd["score_head.0.weight"], pad=0))
    s = _pre_selu(_pre_conv(s, sd["score_head.2.weight"]))
    s = _pre_selu(_pre_conv(s, sd["score_head.4.weight"]))
    score = torch.sigmoid(_pre_conv(s, sd["score_head.6.weight"]))
    feat = F.normalize(x1234, p=2, dim=1)
    hp, wp = x1234.shape[-2:]
    return feat[..., t:hp - bt, l:wp - r], score[..., t:hp - bt, l:wp - r]


def _pre_simple_nms(s, r):
    mp = lambda t: F.max_pool2d(t, 2 * r + 1, stride=1, padding=r)  # noqa: E731
    zeros = torch.zeros_like(s)
    mask = s == mp(s)
    for _ in range(2):
        supp = mp(mask.float()) > 0
        ss = torch.where(supp, zeros, s)
        mask = mask | ((ss == mp(ss)) & ~supp)
    return torch.where(mask, s, zeros)


def _pre_grid_sample_pts(x, pts):
    """x [C, H, W], pts [N, 2] in [-1, 1] (x, y) -> [C, N]: grid_sample bilinear, align_corners=True, zeros."""
    return F.grid_sample(x[None], pts.view(1, 1, -1, 2), mode="bilinear", align_corners=True)[0, :, 0, :]


def _pre_forward(sd, image, model_name="aliked-n16", max_num_keypoints=-1, detection_threshold=0.2, nms_radius=2,
            image_size=None) -> dict:
    c1, c2, c3, c4, dim, K, M = alo.CFGS[model_name]
    top_k = -1 if detection_threshold > 0 else max_num_keypoints
    n_limit = max_num_keypoints if max_num_keypoints > 0 else alo.N_LIMIT_MAX
    feat, score = _pre_dense_maps(sd, image)
    b, _, h, w = score.shape
    r = nms_radius
    nms = _pre_simple_nms(score, r)
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
        kscore = _pre_grid_sample_pts(score[i], kp)[0]
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
        o = F.conv2d(_pre_selu(o), sd["desc_head.offset_conv.2.weight"], sd["desc_head.offset_conv.2.bias"]).clamp(-lim, lim)
        off = o[:, :, 0, 0].view(-1, 2, M).permute(0, 2, 1)  # [N, M, (dx, dy)]
        spos = (kwh[:, None, :] + off) * 2.0 / wh - 1
        f = _pre_grid_sample_pts(feat[i], spos.reshape(-1, 2)).reshape(dim, -1, M).permute(1, 0, 2)  # [N, C, M]
        f = _pre_selu(torch.einsum("dc,ncm->ndm", sd["desc_head.sf_conv.weight"][:, :, 0, 0], f))
        d = F.normalize(torch.einsum("ncp,pcd->nd", f, sd["desc_head.agg_weights"]), p=2, dim=1)
        out["keypoints"].append(wh * (kp + 1) / 2.0)
        out["keypoint_scores"].append(kscore)
        out["descriptors"].append(d)
        out["nms_positions"].append(xy)
    return out


@pytest.mark.parametrize("model_name,h,w,b,conf", [
    ("aliked-n16", 50, 145, 1, {}),
    ("aliked-t16", 33, 47, 2, dict(max_num_keypoints=30, detection_threshold=-1)),
    ("aliked-n32", 60, 90, 1, dict(max_num_keypoints=12)),
    ("aliked-n16", 64, 96, 1, dict(detection_threshold=0.9999999, nms_radius=1)),
    ("aliked-n16", 48, 64, 3, dict(image_size=torch.tensor([[64.0, 48.0], [40.0, 30.0], [1.0, 48.0]]))),
])
def test_forward_is_bit_identical_to_the_pre_split_oracle(model_name, h, w, b, conf):
    torch.set_grad_enabled(False)
    sd = als.make_aliked_state_dict(model_name, 0)
    image = als.make_image(h, w, b, 11)
    new = alo.forward(sd, image, model_name=model_name, **conf)
    old = _pre_forward(sd, image, model_name=model_name, **conf)
    for k in old:
        for x, y in zip(new[k], old[k]):
            assert x.dtype == y.dtype and torch.equal(x, y), k
    feat, score = alo.dense_maps(sd, image)
    feat0, score0 = _pre_dense_maps(sd, image)
    assert torch.equal(feat, feat0) and torch.equal(score, score0)


def test_forward_runs_in_float64():
    sd = {k: v.double() if v.is_floating_point() else v for k, v in als.make_aliked_state_dict("aliked-t16", 0).items()}
    out = alo.forward(sd, als.make_image(33, 47, 1, 3).double(), model_name="aliked-t16")
    assert out["keypoints"][0].dtype == torch.float64 and len(out["keypoints"][0]) > 0


def test_layers_compose_to_forward(chain):
    c = chain
    out = alo.forward(c["sd"], alo.crop(c["xp"], c["h"], c["w"]), model_name=c["model"])
    assert torch.equal(out["nms_positions"][0][:, 1] * c["w"] + out["nms_positions"][0][:, 0], c["pos"])


def _block1(sd, x, k, **d):
    t = F.selu(alo.conv_bn(sd, "block1", 1, x, **(d if k == 1 else {})))
    return F.selu(alo.conv_bn(sd, "block1", 2, t, **(d if k == 2 else {})))


def test_x1(chain):
    c = chain
    ref = alo.block(c["sd64"], 1, D(c["xp"]))
    assert_between(TOL["x1"], rel(c["x1"], ref), {f"conv{k} lost BN bias": rel(_block1(c["sd"], c["xp"], k, nobias=True), ref)
                                                  for k in (1, 2)})


def test_pools(chain):
    c = chain
    for x, p, k in (("x1", "p1", 2), ("x2", "p2", 4), ("x3", "p3", 4)):
        assert_between(TOL["pool"], rel(c[p], alo.pool(D(c[x]), k)), {})


@pytest.mark.parametrize("i", [2, 3, 4])
def test_downsample(chain, i):
    c, blk = chain, f"block{i}"
    p = c[f"p{i - 1}"]
    ref = alo.downsample(c["sd64"], blk, D(p))
    defects = {"lost bias": rel(alo.downsample(c["sd"], blk, p, nobias=True), ref)}
    if i == 4:
        defects["last partial 4-pixel group dropped"] = rel(alo.downsample(c["sd"], blk, p, drop_tail=True), ref)
    assert_between(TOL["conv"], rel(c[f"d{i}"], ref), defects)


@pytest.mark.parametrize("i", [2, 3, 4])
def test_first_convolution(chain, i):
    """t_i from p_{i-1}; block3 / block4: the offsets too, in float64 on the reference side."""
    c, blk = chain, f"block{i}"
    p = c[f"p{i - 1}"]
    ref = F.selu(alo.conv_bn(c["sd64"], blk, 1, D(p)))
    cases = {"lost BN bias": dict(nobias=True)}
    if i > 2:
        cases.update({"tap dy / dx swapped": dict(swap=True), "clamp-to-edge taps": dict(edge=True),
                      "offset group 16-17 dropped": dict(drop_group=True)})
        if p.shape[-2] != p.shape[-1]:  # on a square level min(h, w) = max(h, w)
            cases["offset clamp at min(h, w) / 4"] = dict(lim_min=True)
    defects = {k: rel(F.selu(alo.conv_bn(c["sd"], blk, 1, p, **v)), ref) for k, v in cases.items()}
    assert_between(TOL["dcn" if i > 2 else "conv"], rel(c[f"t{i}"], ref), defects)


@pytest.mark.parametrize("i", [3, 4])
def test_offset_convolution(chain, i):
    c, p = chain, f"block{i}.conv2"
    t = c[f"t{i}"]
    ref = alo.offsets(c["sd64"], p, D(t))
    cases = {"group 16-17 dropped": dict(drop_group=True)}
    if t.shape[-2] != t.shape[-1]:
        cases["clamp at min(h, w) / 4"] = dict(lim_min=True)
    if i == 4:
        cases["last partial 4-pixel group dropped"] = dict(drop_tail=True)
    defects = {k: rel(alo.offsets(c["sd"], p, t, **v), ref) for k, v in cases.items()}
    assert_between(TOL["offset"], rel(c[f"o{i}"], ref), defects)


@pytest.mark.parametrize("i", [2, 3, 4])
def test_block_output(chain, i):
    """x_i from the captured t_i, d_i (and o_i)."""
    c, blk = chain, f"block{i}"
    t, d, o = c[f"t{i}"], c[f"d{i}"], c.get(f"o{i}")
    ref = alo.block_out(c["sd64"], blk, D(t), D(d), None if o is None else D(o))
    cases = {"lost BN bias": dict(nobias=True), "dropped residual": dict(nores=True)}
    if i > 2:
        cases.update({"tap dy / dx swapped": dict(swap=True), "clamp-to-edge taps": dict(edge=True)})
    defects = {k: rel(alo.block_out(c["sd"], blk, t, d, o, **v), ref) for k, v in cases.items()}
    assert_between(TOL["conv"], rel(c[f"x{i}"], ref), defects)


@pytest.mark.parametrize("i", [2, 3, 4])
def test_aggregation(chain, i):
    c = chain
    x = c[f"x{i}"]
    ref = alo.aggregate(c["sd64"], i, D(x))
    defects = {}
    if i == 4:
        defects["last partial 4-pixel group dropped"] = rel(alo.aggregate(c["sd"], i, x, drop_tail=True), ref)
    assert_between(TOL["conv"], rel(c["a"][i - 1], ref), defects)


def test_head_layer_and_inverse_norm(chain):
    c = chain
    ref = c["x1234_64"]
    bad = alo.upsample(c["a"], align_corners=False)
    s1 = alo.score_layer(c["sd64"], 0, ref)
    assert_between(TOL["head"], rel(c["s"][0], s1), {"align_corners=False": rel(alo.score_layer(c["sd"], 0, bad), s1)})
    inv = alo.inv_norm(ref)
    assert_between(TOL["head"], rel(alo.inv_norm(c["x1234"]), inv), {"align_corners=False": rel(alo.inv_norm(bad), inv)})


def test_score_layers(chain):
    c = chain
    for j, k in enumerate((2, 4, 6), 1):
        assert_between(TOL["score"], rel(c["s"][j], alo.score_layer(c["sd64"], k, D(c["s"][j - 1]))), {})


def test_soft_argmax(chain):
    c = chain
    h, w = c["h"], c["w"]
    kp64, ks64, _ = alo.soft_argmax(D(c["score"][0]), c["pos"], 2)
    kp, ks, _ = alo.soft_argmax(c["score"][0], c["pos"], 2)
    kpt, kst, _ = alo.soft_argmax(c["score"][0], c["pos"], 2, temperature=0.11)
    px64, ext = alo.pixels(kp64, h, w), max(w - 1, h - 1)
    print(f"keypoints {absd(alo.pixels(kp, h, w), px64) / ext:.2e}")
    assert_between(TOL["kpt"], absd(alo.pixels(kp, h, w), px64) / ext,
                   {"temperature 0.11": absd(alo.pixels(kpt, h, w), px64) / ext})
    assert_between(TOL["kscore"], absd(ks, ks64), {"temperature 0.11": absd(kst, ks64)})


def _box(h, w):
    l, _, t, _ = alo._pads(h, w)
    return t, l, h, w


def test_sddh(chain):
    c = chain
    kp, _, _ = alo.soft_argmax(c["score"][0], c["pos"], 2)
    box = _box(c["h"], c["w"])
    featp = F.normalize(c["x1234"], dim=1)[0]
    ref = alo.sddh(c["sd64"], F.normalize(c["x1234_64"], dim=1)[0], box, D(kp), c["M"])
    cases = {"offsets read as (dy, dx)": dict(swap=True), "samples bounded by the padded frame": dict(padded=True),
             "agg_weights transposed": dict(agg_t=True)}
    defects = {k: absd(alo.sddh(c["sd"], featp, box, kp, c["M"], **v), ref) for k, v in cases.items()}
    assert_between(TOL["desc"], absd(alo.sddh(c["sd"], featp, box, kp, c["M"]), ref), defects)


def _kernel_mean(score):
    """The stats kernel's mean: the fp32 scores summed in double, divided by H W, rounded once to fp32."""
    b = score.shape[0]
    return (D(score).reshape(b, -1).sum(1) / score[0].numel()).float()


def test_mean(chain):
    """The mean tolerance covers the one rounding of the double sum; the margin covers a mean anywhere within it."""
    c = chain
    mean64 = D(c["score"]).mean()
    padded = D(c["s"][-1]).mean()  # the pre-crop map's
    assert_between(TOL["mean"], float((D(_kernel_mean(c["score"])) - mean64).abs() / mean64),
                   {"mean over the padded frame": float((padded - mean64).abs() / mean64)})
    assert TOL["mean_margin"] >= 3 * TOL["mean"]


@pytest.fixture(scope="module")
def big():
    """The network's fp32 maps at 768 x 1024 (the image of tests/test_gpu_aliked_layers.py, about 10 000 keypoints):
    where the fp32 rounding of normalised coordinates is coarsest."""
    torch.set_grad_enabled(False)
    sd = als.make_aliked_state_dict("aliked-n16", 0)
    sd64 = {k: D(v) for k, v in sd.items()}
    xs = alo.encoder(sd, alo.pad(als.make_image(768, 1024, 1, 91)))
    a = [alo.aggregate(sd, i, v) for i, v in enumerate(xs, 1)]
    x1234 = alo.upsample(a)
    score = alo.score_head(sd, x1234)  # no padding at 768 x 1024
    pos = alo.select(alo.nms_borders(score.clone(), 2), score, 0.2, -1)[0]
    assert len(pos) > 5000
    x64 = alo.upsample([alo.aggregate(sd64, 1, D(xs[0]))] + [D(v) for v in a[1:]])
    return {"sd": sd, "sd64": sd64, "score": score, "pos": pos, "featp": F.normalize(x1234, dim=1)[0],
            "featp64": F.normalize(x64, dim=1)[0]}


def test_soft_argmax_at_768x1024(big):
    """The keypoint error relative to the extent stays that of the small shapes; the keypoint score, sampled at the
    keypoint, grows with it (4.5e-5 px on the steepest slopes)."""
    score, pos = big["score"][0], big["pos"]
    kp64, ks64, _ = alo.soft_argmax(D(score), pos, 2)
    kp, ks, _ = alo.soft_argmax(score, pos, 2)
    kpt, kst, _ = alo.soft_argmax(score, pos, 2, temperature=0.11)
    px64 = alo.pixels(kp64, 768, 1024)
    assert_between(TOL["kpt"], absd(alo.pixels(kp, 768, 1024), px64) / 1023,
                   {"temperature 0.11": absd(alo.pixels(kpt, 768, 1024), px64) / 1023})
    assert_between(TOL["kscore"], absd(ks, ks64), {"temperature 0.11": absd(kst, ks64)})


def test_sddh_at_768x1024(big):
    """SDDH's sample positions (kp / 2 + 0.5) (w - 1) round more coarsely in fp32 the wider the image."""
    kp, _, _ = alo.soft_argmax(big["score"][0], big["pos"], 2)
    box = (0, 0, 768, 1024)
    ref = alo.sddh(big["sd64"], big["featp64"], box, D(kp), 16)
    cases = {"offsets read as (dy, dx)": dict(swap=True), "agg_weights transposed": dict(agg_t=True)}
    defects = {k: absd(alo.sddh(big["sd"], big["featp"], box, kp, 16, **v), ref) for k, v in cases.items()}
    assert_between(TOL["desc"], absd(alo.sddh(big["sd"], big["featp"], box, kp, 16), ref), defects)


def test_mean_at_768x1024(big):
    mean64 = D(big["score"]).mean()
    assert_between(TOL["mean"], float((D(_kernel_mean(big["score"])) - mean64).abs() / mean64), {})


def _end_to_end(sd, xp, h, w, pos, M, blk4=None, sddh=None, temperature=0.1, r=2):
    """(keypoints, scores, descriptors) of one padded image at the given flat positions; defects: ``blk4`` for block4's
    second convolution, ``sddh`` for SDDH, ``temperature`` for the soft-argmax."""
    x1, x2, x3, _ = alo.encoder(sd, xp)
    p3 = alo.pool(x3, 4)
    t4 = F.selu(alo.conv_bn(sd, "block4", 1, p3))
    x4 = alo.block_out(sd, "block4", t4, alo.downsample(sd, "block4", p3), **(blk4 or {}))
    x1234 = alo.upsample([alo.aggregate(sd, i, v) for i, v in enumerate((x1, x2, x3, x4), 1)])
    score = alo.crop(alo.score_head(sd, x1234), h, w)
    kp, ks, _ = alo.soft_argmax(score[0], pos, r, temperature)
    d = alo.sddh(sd, F.normalize(x1234, dim=1)[0], _box(h, w), kp, M, **(sddh or {}))
    return alo.pixels(kp, h, w), ks, d


def test_end_to_end_gates_resolve_the_defects(chain):
    """A lost BN bias in block4 (which reaches the descriptor through a quarter of the channels after a x32 upsample),
    SDDH's offsets read as (dy, dx) and a soft-argmax temperature of 0.11 move the outputs by >= 3x the gates."""
    c = chain
    args = (c["xp"], c["h"], c["w"], c["pos"], c["M"])
    ref = _end_to_end(c["sd64"], D(c["xp"]), *args[1:])
    defects = {"block4 lost BN bias": dict(blk4=dict(nobias=True)), "SDDH (dy, dx)": dict(sddh=dict(swap=True)),
               "temperature 0.11": dict(temperature=0.11)}
    dev = {k: [absd(a, r) for a, r in zip(_end_to_end(c["sd"], *args, **v), ref)] for k, v in defects.items()}
    moves_keypoints = ("block4 lost BN bias", "temperature 0.11")  # SDDH does not feed back into them
    assert_between(E2E_KPT, 0.0, {k: dev[k][0] for k in moves_keypoints})
    assert_between(E2E_SCORE, 0.0, {k: dev[k][1] for k in moves_keypoints})
    assert_between(E2E_DESC, 0.0, {k: v[2] for k, v in dev.items()})


FIXTURES = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "aliked")


@pytest.mark.parametrize("name", sorted(f[:-3] for f in os.listdir(FIXTURES) if f.startswith("al_") and f.endswith(".pt")))
def test_end_to_end_error_on_the_fixture_images(name):
    """One fp32 forward against float64 at its own keypoint positions, on the image and conf of each reference
    fixture that tests/test_gpu_aliked.py compares with: within the gates (at most 2.6e-5 px, 6.8e-6 and 5.4e-6, all
    on the t16 fixture)."""
    torch.set_grad_enabled(False)
    fix = torch.load(os.path.join(FIXTURES, name + ".pt"), weights_only=False)
    rc, conf = fix["recipe"], dict(fix["conf"])
    model_name = conf.pop("model_name")
    sd = als.make_aliked_state_dict(model_name, 0)
    sd64 = {k: D(v) for k, v in sd.items() if v.is_floating_point()}
    image = als.make_image(rc["h"], rc["w"], rc["b"], rc["seed"])
    image_size = torch.tensor(rc["image_size"]) if "image_size" in rc else None
    out = alo.forward(sd, image, model_name=model_name, image_size=image_size, **conf)
    M, r, h, w = alo.CFGS[model_name][6], conf["nms_radius"], rc["h"], rc["w"]
    err = [0.0, 0.0, 0.0]
    for b in range(rc["b"]):
        xp = alo.pad(image[b:b + 1])
        pos = out["nms_positions"][b][:, 1] * w + out["nms_positions"][b][:, 0]
        got = _end_to_end(sd, xp, h, w, pos, M, r=r)
        ref = _end_to_end(sd64, D(xp), h, w, pos, M, r=r)
        err = [max(e, absd(a, g)) for e, a, g in zip(err, got, ref)]
    assert err[0] < E2E_KPT and err[1] < E2E_SCORE and err[2] < E2E_DESC, err
