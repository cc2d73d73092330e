"""Constructed inputs for the keypoint-selection stages of SuperPoint (``sp_post``) and DISK (``disk_detect``), with the
stage-by-stage checks the CPU emulation and the GPU tests share.  TEST INFRASTRUCTURE ONLY.

SuperPoint inputs are detector logits [B, 65, Hc, Wc] and a descriptor map [B, 256, Hc, Wc].  A background cell has
logit 0 on its 64 pixel channels and BG on the dustbin, so each of its pixels scores 1 / (64 + e^BG) ~ 6e-6, below the
default threshold.  A peak sets one pixel's channel.  Equal scores come from identical logit vectors (same channels,
same values: the soft-max sums them in the same order); equal adjacent pixels of neighbouring cells come from equal
channels of identical vectors.

Every case carries a regime: a function of the captured stages that asserts the situation the case exists for (a tie
at the top-k cut that crosses a 1024-candidate chunk, a pixel re-admitted by round 2 of simple_nms, ...) and returns
a one-line description.  The checks compare each stage with the oracle applied to the captured output of the stage
before it: exactly for the NMS map, candidates and selection; within SCORE_TOL / DENSE_TOL / DESC_TOL for the
soft-max scores, the normalised map and the descriptors."""
from __future__ import annotations

import dataclasses
from typing import Callable, Optional

import torch
import torch.nn.functional as F

from oracle import disk_oracle as do
from oracle import superpoint_oracle as spo

BG = 12.0
PEAK = 14.0
# Gates, max|delta| / max|ref| per image for scores and the normalised map, absolute for unit descriptors: at least 3x
# the worst fp32 deviation seen on an H100 (2.3e-6 / 4.3e-7 / 3.1e-6) and at most a third of each listed defect (dropped
# dustbin, half-pixel sampler shift, align_corners=False) on every case that can show it
# (tests/test_keypoint_selection_emulation.py).
SCORE_TOL, DENSE_TOL, DESC_TOL = 1e-5, 2e-6, 1e-5
# sp_workspace_layout's buffers, in order (include/superpoint_b200.h)
SP_LAYOUT_NAMES = ("logits", "scores", "t0", "mask", "dense", "row_count", "row_start", "n_cand", "cand_pos", "cand_score",
                   "sel_pos", "sel_score", "n_sel")


# ------------------------------------------------------------------------------------------------------ SuperPoint
@dataclasses.dataclass
class SpCase:
    name: str
    logits: torch.Tensor
    dense: torch.Tensor
    regime: Callable[[dict], str]
    nms_radius: int = 4
    remove_borders: int = 4
    threshold: object = 0.0005  # or a function of a first run's captured stages (-> float)
    k: object = 0               # 0 = None; or a function of a first run's captured stages (-> int)

    @property
    def shape(self):
        b, _, hc, wc = self.logits.shape
        return b, 8 * hc, 8 * wc


def maps(b, h, w, seed=0, random_logits=False):
    """Background logits (or random ones: 3 N(0, 1) on every channel) and a random descriptor map."""
    g = torch.Generator().manual_seed(seed)
    if random_logits:
        logits = 3 * torch.randn(b, 65, h // 8, w // 8, generator=g)
    else:
        logits = torch.zeros(b, 65, h // 8, w // 8)
        logits[:, 64] = BG
    return logits, torch.randn(b, 256, h // 8, w // 8, generator=g)


def put(logits, y, x, v=PEAK, b=0):
    logits[b, (y % 8) * 8 + x % 8, y // 8, x // 8] = v


def levels(b, h, w, step=0.25):
    """Every cell identical, channel c at -(c % 8) step: the scores take 8 values by x % 8 (h w / 8 pixels each)."""
    logits, dense = maps(b, h, w)
    logits[:, :64] = (-(torch.arange(64) % 8) * step).view(1, 64, 1, 1)
    logits[:, 64] = 0.0
    return logits, dense


def kept(st, b=0):
    """Pixels (y, x) with a positive NMS value, and the NMS map of image b."""
    m = st["nms"][b]
    return {tuple(p) for p in (m > 0).nonzero().tolist()}, m


def sel_scores(st, b=0):
    return st["sel"][b][1]


def _pair_within_r(st):
    ks, m = kept(st)
    assert (12, 12) in ks and (12, 14) in ks and m[12, 12] == m[12, 14]
    return "two equal kept neighbours 2 <= r = 4 apart"


def _block(st):
    ks, m = kept(st)
    blk = {(y, x) for y in range(9, 12) for x in range(9, 12)}
    assert blk <= ks and len({float(m[p]) for p in blk}) == 1
    return "a flat 3x3 block, all nine kept"


def _r_plus_1(st):
    ks, m = kept(st)
    assert (10, 8) in ks and (10, 13) in ks and m[10, 8] == m[10, 13]
    return "equal maxima r + 1 = 5 apart, both kept"


def _cell_border(st):
    ks, m = kept(st)
    assert (10, 15) in ks and (10, 16) in ks and m[10, 15] == m[10, 16]
    return "equal adjacent pixels x = 15 | 16 across a cell border, both kept"


CHAIN = [(20, 4 + 8 * i) for i in range(7)]


def _chain(st):
    s = st["scores"][0].double()
    rounds = [spo.simple_nms(s[None], 8, rounds=n)[0] > 0 for n in range(4)]
    got = [[bool(r[p]) for p in CHAIN] for r in rounds]
    assert got[0][:5] == [True, False, False, False, False]
    assert got[1][:5] == [True, False, True, False, False]  # round 1 re-admits the third
    assert got[2][:5] == [True, False, True, False, True]   # round 2 re-admits the fifth
    assert not got[2][6] and got[3][6]                     # a third round would re-admit the seventh
    return "round 1 re-admits (20, 20), round 2 (20, 36); (20, 52) needs a third"


def _radius(r):
    def f(st):
        ks, m = kept(st)
        s = st["scores"][0]
        if r == 0:
            assert torch.equal(m > 0, s > 0)
            return "r = 0: every pixel kept"
        if 2 * r + 1 > 2 * max(s.shape):
            assert len(ks) == int((s == s.max()).sum()) >= 1
            return f"r = {r} wider than the map: only the global maximum"
        assert 1 < len(ks) < s.numel() // (r + 1)
        return f"r = {r}: {len(ks)} kept"
    return f


def _borders(p):
    def f(st):
        m = st["nms"][0]
        h, w = m.shape
        if p == 0:
            edge = torch.cat([m[0], m[-1], m[:, 0], m[:, -1]])
            assert (edge > st["thr"]).any()
            return "no border removal: candidates on the edge"
        assert (m[:p] == -1).all() and (m[:, -p:] == -1).all()
        if 2 * p >= min(h, w):
            assert (m == -1).all() and st["n_sel"][0] == 0
            return f"remove_borders = {p} >= half the map: no keypoint"
        return f"remove_borders = {p}"
    return f


def _median_kept(st):
    v = st["nms"][0][st["nms"][0] > 0.001].sort().values
    return float(v[v.numel() // 2])


def _thr_captured(st):
    m = st["nms"][0]
    eq = m == st["thr"]
    assert eq.sum() >= 1 and all(float(v) != st["thr"] for v in st["cand"][0][1])
    return f"threshold = a captured score ({int(eq.sum())} pixels), excluded"


def _thr_zero(st):
    m = st["nms"][0]
    vals = st["cand"][0][1]
    assert (m == 0).any() and (vals > 0).all() and (vals < 1e-5).any()
    assert vals.numel() > st["cap"] and st["n_sel"][0] == -1
    return (f"threshold 0: background plateaus are candidates, NMS zeros are not; {vals.numel()} candidates > "
            f"sp_max_keypoints {st['cap']}: count -1")


def _thr_negative(st):
    m, (pos, vals) = st["nms"][0], st["cand"][0]
    k = st["k"]
    assert pos.numel() == m.numel() and (vals == 0).sum() > 500 and (vals == -1).sum() > 100
    assert k < pos.numel() and sel_scores(st)[k - 1] == 0 and (vals == 0).sum() > (sel_scores(st) == 0).sum()
    return "threshold -2: NMS zeros and border -1s are candidates; the cut falls in the tie of zeros"


def _k_rel(d):
    def f(st):
        n = st["cand"][0][0].numel()
        assert st["k"] == n + d and n > 1
        return f"k = n {d:+d} (n = {n})"
    return f


def _k1(st):
    assert st["k"] == 1 < st["cand"][0][0].numel()
    return "k = 1"


def _all_equal(st):
    vals = st["cand"][0][1]
    assert (vals == vals[0]).all() and vals.numel() > st["k"]
    return f"all {vals.numel()} candidates equal, k = {st['k']}"


def _tie_at_cut(kmin=0, warp=True):
    def f(st):
        (pos, vals), k = st["cand"][0], st["k"]
        assert vals.numel() > k >= kmin
        kth = sel_scores(st)[k - 1]
        eq = (vals == kth).nonzero().reshape(-1)       # candidate indices of the tie
        taken = int((sel_scores(st) == kth).sum())
        assert 0 < taken < eq.numel()
        last_in, first_out = int(eq[taken - 1]), int(eq[taken])
        assert int(eq[0]) < 1024 <= last_in, "the kept part of the tie crosses a 1024-candidate chunk"
        assert not warp or last_in // 32 != first_out // 32, "the cut falls between two warps"
        return (f"k = {k} < n = {vals.numel()}: the tie at the k-th place has {eq.numel()} members, kept {taken} "
                f"(candidates {int(eq[0])} .. {last_in}), cut before candidate {first_out}")
    return f


def _shape(cond, text):
    def f(st):
        h, w = st["nms"][0].shape
        assert cond(h, w) and st["n_sel"][0] > 0
        return text
    return f


def _tall(st):
    rows = st["cand"][0][0] // st["nms"].shape[-1]
    assert st["nms"].shape[1] > 1024 and (rows < 1024).any() and (rows >= 1024).any()
    return f"{st['nms'].shape[1]} rows: candidates on both sides of row 1024 (the row scan's carry)"


def _batch(st):
    n = [int(v) for v in st["n_sel"]]
    assert n[0] == 0 and 0 < n[1] <= 5 and n[2] > 100
    return f"B = 3 with {n} keypoints"


def _edges(st):
    ks = {(int(p) // st["nms"].shape[-1], int(p) % st["nms"].shape[-1]) for p in st["sel"][0][0]}
    assert EDGE_POINTS <= ks
    return "keypoints at the four corners and on every edge"


def _zero_cell(st):
    ws = st["nms"].shape[-1]
    pos = st["sel"][0][0].tolist()
    assert 20 * ws + 20 in pos
    return "a keypoint whose neighbouring cells' descriptors are all zero"


EDGE_POINTS = {(0, 0), (0, 47), (31, 0), (31, 47), (0, 20), (31, 28), (12, 0), (20, 47)}


def sp_cases():
    cases = []

    def add(name, lg_dense, regime, **kw):
        cases.append(SpCase(name, lg_dense[0], lg_dense[1], regime, **kw))

    lg, de = maps(1, 32, 32, 1)
    put(lg, 12, 12), put(lg, 12, 14)
    add("plateau: equal neighbours within r", (lg, de), _pair_within_r)
    lg, de = maps(1, 32, 32, 2)
    for y in range(9, 12):
        for x in range(9, 12):
            put(lg, y, x)
    add("plateau: flat 3x3 block", (lg, de), _block)
    lg, de = maps(1, 32, 32, 3)
    put(lg, 10, 8), put(lg, 10, 13)
    add("plateau: equal values r + 1 apart", (lg, de), _r_plus_1)
    lg, de = maps(1, 32, 32, 4)
    for x in (8, 15, 16, 23):  # cells (1, 1) and (1, 2): identical vectors, channels (2, 0) and (2, 7) equal
        put(lg, 10, x)
    add("plateau: across a cell border", (lg, de), _cell_border)
    lg, de = maps(1, 48, 80, 5)
    for i, (y, x) in enumerate(CHAIN):
        put(lg, y, x, 16.0 - 0.5 * i)
    add("simple_nms: rounds 1 and 2 re-admit", (lg, de), _chain, nms_radius=8, remove_borders=0)
    for r in (0, 1, 4, 40):
        add(f"nms_radius {r}", maps(1, 24, 32, 10 + r, random_logits=True), _radius(r), nms_radius=r, remove_borders=0)
    for p in (0, 4, 16):
        add(f"remove_borders {p}", maps(1, 32, 32, 20 + p, random_logits=True), _borders(p), nms_radius=2,
            remove_borders=p)
    add("threshold: a captured score", maps(1, 32, 40, 30, random_logits=True), _thr_captured, nms_radius=2,
        threshold=_median_kept)
    lg, de = maps(1, 40, 40, 31)
    put(lg, 20, 20), put(lg, 12, 30, 13.0)
    add("threshold 0", (lg, de), _thr_zero, nms_radius=2, threshold=0.0)
    add("threshold -2: huge tie sets", maps(1, 40, 48, 32, random_logits=True), _thr_negative, nms_radius=2,
        threshold=-2.0, k=lambda st: int((st["nms"][0] > 0).sum()) + 100)
    for d in (-1, 0, 1):
        add(f"top-k: k = n {d:+d}", maps(1, 32, 48, 40, random_logits=True), _k_rel(d), nms_radius=2,
            k=lambda st, d=d: st["cand"][0][0].numel() + d)
    add("top-k: k = 1", maps(1, 32, 48, 41, random_logits=True), _k1, nms_radius=2, k=1)
    lg, de = maps(1, 64, 64, 42)
    lg[:, 4 * 8 + 4] = PEAK  # every cell: the same peak at (4, 4)
    add("top-k: all candidates equal", (lg, de), _all_equal, k=10)
    add("top-k: tie across the cut, a 1024 chunk and a warp", levels(1, 64, 64), _tie_at_cut(), nms_radius=0,
        remove_borders=0, threshold=0.0, k=812)
    for k in (4096, 4097):
        add(f"top-k: k = {k} (n = 5184)", levels(1, 72, 72), _tie_at_cut(k, warp=k == 4096), nms_radius=0, remove_borders=0,
            threshold=0.0, k=k)
    lg, de = maps(1, 8, 8, 50)
    put(lg, 2, 2), put(lg, 5, 6, 13.0), put(lg, 7, 0, 12.5)
    add("shape: 8x8, one cell", (lg, de), _shape(lambda h, w: h == w == 8, "one cell: Wc - 1 = Hc - 1 = 0 in the sampler"),
        nms_radius=1, remove_borders=0)
    add("shape: width 8", maps(1, 64, 8, 51, random_logits=True), _shape(lambda h, w: w == 8, "W = 8: one ballot tail"),
        nms_radius=1, remove_borders=0)
    add("shape: width 40", maps(1, 48, 40, 52, random_logits=True),
        _shape(lambda h, w: w % 32 == 8, "W = 40: a full warp and a tail of 8"), nms_radius=1, remove_borders=0)
    add("shape: 1040x16", maps(1, 1040, 16, 53, random_logits=True), _tall, nms_radius=1, remove_borders=0)
    lg, de = maps(3, 48, 64, 54)
    lg[2] = maps(1, 48, 64, 55, random_logits=True)[0][0]
    for y, x in ((10, 10), (30, 40), (20, 50)):
        put(lg, y, x, b=1)
    add("shape: B = 3, zero / few / many", (lg, de), _batch, nms_radius=2)
    lg, de = maps(1, 32, 48, 60)
    for y, x in EDGE_POINTS:
        put(lg, y, x)
    add("sampling: corners and edges", (lg, de), _edges, nms_radius=1, remove_borders=0)
    lg, de = maps(1, 32, 32, 61)
    put(lg, 20, 20), put(lg, 6, 26)
    de[:, :, 1:4, 1:4] = 0.0
    add("sampling: zero descriptor cells", (lg, de), _zero_cell, nms_radius=2)
    return cases


def sp_conf(case, threshold, k):
    return dict(nms_radius=case.nms_radius, remove_borders=case.remove_borders, detection_threshold=threshold,
                max_num_keypoints=k)


def sp_views(ws, offsets, sizes, b, h, w, cap):
    """Views of a SuperPoint workspace (CPU or CUDA uint8 tensor) by sp_workspace_layout's names, shaped for a score map
    h x w (multiples of 8) and `cap` output rows."""
    v = {}
    for name, o, n in zip(SP_LAYOUT_NAMES, offsets, sizes):
        dt = torch.int32 if name in ("row_count", "row_start", "n_cand", "cand_pos", "sel_pos", "n_sel") else torch.float32
        v[name] = ws[o:o + n].view(dt)
    hc, wc = h // 8, w // 8
    v["logits"] = v["logits"][:b * 65 * hc * wc].view(b, 65, hc, wc)
    v["dense"] = v["dense"][:b * 256 * hc * wc].view(b, 256, hc, wc)
    for name in ("scores", "t0", "mask"):
        v[name] = v[name][:b * h * w].view(b, h, w)
    for name in ("row_count", "row_start"):
        v[name] = v[name][:b * h].view(b, h)
    for name in ("sel_pos", "sel_score"):
        v[name] = v[name][:b * cap].view(b, cap)
    return v


def captured_stages(v, out, thr, k):
    """The stages as the regimes and the oracle read them (on the CPU)."""
    b, h, w = v["t0"].shape
    n_cand, n_sel = v["n_cand"][:b].cpu(), v["n_sel"][:b].cpu()
    cp, cs = v["cand_pos"].cpu(), v["cand_score"].cpu()
    cand = [(cp[i * h * w:i * h * w + int(n_cand[i])].long(), cs[i * h * w:i * h * w + int(n_cand[i])].double())
            for i in range(b)]
    sel = [(v["sel_pos"][i, :max(int(n_sel[i]), 0)].cpu().long(), v["sel_score"][i, :max(int(n_sel[i]), 0)].cpu().double())
           for i in range(b)]
    return {"scores": v["scores"].cpu(), "nms": v["t0"].cpu().double(), "mask": v["mask"].cpu(),
            "dense": v["dense"].cpu(), "cand": cand, "sel": sel, "n_sel": n_sel, "thr": thr, "k": k,
            "cap": v["sel_pos"].shape[1], "out": [t.cpu() for t in out]}


def rel(a, ref):
    d = (a.double() - ref).abs().flatten(1).amax(1) / ref.abs().flatten(1).amax(1).clamp_min(1e-300)
    return float(d.max())


def check_sp(case, st, worst):
    """Every stage of one captured post-processing run against the oracle on its captured input.  Returns the list of
    failed checks; `worst` collects the deviations of the checks within a tolerance."""
    bad = []
    conf = sp_conf(case, st["thr"], st["k"])
    ref = spo.post(case.logits, case.dense, given=st, **conf)
    b = case.logits.shape[0]

    def within(name, err, tol):
        worst[name] = max(worst.get(name, 0.0), err)
        if not err <= tol:
            bad.append((name, err, tol))

    within("scores", rel(st["scores"], ref["scores"]), SCORE_TOL)
    within("dense", rel(st["dense"].reshape(b, -1), ref["dense"].reshape(b, -1)), DENSE_TOL)
    if not torch.equal(st["nms"], ref["nms"]):
        bad.append("nms map")
    keep = spo.simple_nms(st["scores"].double(), case.nms_radius) > 0
    if not torch.equal(st["mask"] > 0, keep):
        bad.append("nms mask")
    kp, ks, de, cnt = st["out"]
    for i in range(b):
        (cp, cs), (rp, rs) = st["cand"][i], ref["cand"][i]
        if not (torch.equal(cp, rp) and torch.equal(cs, rs)):
            bad.append(f"image {i}: candidates")
        n = int(st["n_sel"][i])
        if int(cnt[i]) != n:
            bad.append(f"image {i}: counts")
        if not st["k"] and cp.numel() > st["cap"]:  # more NMS survivors than the outputs hold: count -1, zero rows
            if n != -1 or kp[i].any() or ks[i].any() or de[i].any():
                bad.append(f"image {i}: overflow")
            continue
        (sp_, ss), (tp, ts) = st["sel"][i], ref["sel"][i]
        if not (torch.equal(sp_, tp) and torch.equal(ss, ts)):
            bad.append(f"image {i}: selection")
        if not torch.equal(kp[i, :n].double(), ref["keypoints"][i]) or not torch.equal(ks[i, :n].double(), ss):
            bad.append(f"image {i}: keypoints / scores")
        if kp[i, n:].any() or ks[i, n:].any() or de[i, n:].any():
            bad.append(f"image {i}: padding rows")
        if n:
            within("descriptors", float((de[i, :n].double() - ref["descriptors"][i]).abs().max()), DESC_TOL)
    return bad


def sp_defects(case, st):
    """The listed defects on this case's captured data, in the units of the gates: a dropped dustbin (scores), a
    half-pixel shift of the sampler and align_corners=False (descriptors).  None where the case cannot show one."""
    out = {}
    p = torch.softmax(case.logits.double()[:, :64], dim=1)
    ref = spo.dense_scores(case.logits.double())
    hc, wc = case.logits.shape[-2:]
    nodust = p.permute(0, 2, 3, 1).reshape(-1, hc, wc, 8, 8).permute(0, 1, 3, 2, 4).reshape(ref.shape)
    out["scores"] = rel(nodust, ref)
    dn = F.normalize(case.dense.double(), dim=1)
    shift, corners = 0.0, 0.0
    for i, (pos, _) in enumerate(st["sel"]):
        if pos.numel() == 0 or hc == 1 or wc == 1:
            continue
        ws = 8 * wc
        xy = torch.stack([pos % ws, pos // ws], dim=-1).double()
        good = spo.sample_descriptors(xy, dn[i])
        shift = max(shift, float((spo.sample_descriptors(xy + 0.5, dn[i]) - good).abs().max()))
        g = (xy - 3.5) / torch.tensor([wc * 8 - 4.5, hc * 8 - 4.5]).double() * 2 - 1
        bad = F.grid_sample(dn[i][None], g.view(1, 1, -1, 2), mode="bilinear", align_corners=False)
        bad = F.normalize(bad.reshape(256, -1), dim=0).t()
        corners = max(corners, float((bad - good).abs().max()))
    if shift:
        out["half-pixel shift"], out["align_corners=False"] = shift, corners
    return out


# ------------------------------------------------------------------------------------------------------ DISK
@dataclasses.dataclass
class DiskCase:
    name: str
    heat: torch.Tensor  # [B, H, W]
    window: int
    threshold: float
    n: object           # None, int, or a function of the candidate count of image 0
    regime: Callable[[list, list], str]  # (per-image candidate (y, x, value) lists, per-image selected (x, y)) -> text


def disk_candidates(heat, window, threshold):
    """[H, W] -> the NMS survivors above the threshold: flat indices, row-major."""
    keep = do.nms_mask(heat, window) & (heat > threshold)
    return keep.reshape(-1).nonzero().reshape(-1)


def disk_expected(heat, window, threshold, n):
    """disk_oracle.detect for one image, as (flat indices, scores); an image without candidates keeps nothing (the
    reference's kthvalue raises there)."""
    if n is not None and disk_candidates(heat, window, threshold).numel() == 0:
        return torch.zeros(0, dtype=torch.long), torch.zeros(0, dtype=heat.dtype)
    xy, logp = do.detect(heat, window, threshold, n)
    return xy[:, 1] * heat.shape[1] + xy[:, 0], logp


def _bg(b, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    return -1.0 - torch.rand(b, h, w, generator=g)


def _plateau(window):
    r = window // 2

    def f(cands, sel):
        ys = set(map(tuple, sel[0]))
        first, outside = (10, 10), (10, 11 + r + 1)
        if window == 1:
            assert {(10, 10), (10, 11), (11, 10), (11, 11), (0, 0), (0, 1)} <= {(y, x) for x, y in ys}
            return "window 1: every plateau pixel kept"
        assert {(x, y) for y, x in (first, outside, (0, 0))} <= ys
        assert not {(11, 10), (10, 11), (11, 11), (1, 0), (0, 1)} & ys
        return f"window {window}: only each plateau's first pixel (one cut by the edge) and the equal value r + 1 away"
    return f


def _kcount(expect):
    def f(cands, sel):
        c = len(cands[0])
        want = expect(c)
        assert len(sel[0]) == want, (len(sel[0]), want)
        return f"{c} candidates -> {want} kept"
    return f


def _tie_n1(cands, sel):
    assert len(sel[0]) == 2
    return "a tie at the (n + 1)-th score: 2 kept for n = 3"


def _chunk_tie(cands, sel):
    idx = [y * 64 + x for x, y in sel[0]]
    assert len(sel[0]) == 1024 < 1500 and max(idx) >= 1024
    return "1024 of 4096 kept across every 1024-candidate chunk, n = 1500 (the 1501st is tied)"


def _thr_eq(cands, sel):
    assert (5, 5) not in set(map(tuple, sel[0])) and (20, 5) in set(map(tuple, sel[0]))
    return "a heat value equal to the threshold is dropped"


def _tall_disk(cands, sel):
    ys = [y for _, y in sel[0]]
    assert min(ys) < 1024 <= max(ys)
    return "1040 rows: keypoints on both sides of row 1024"


def _batch_disk(cands, sel):
    n = [len(s) for s in sel]
    assert n[0] == 0 and 0 < n[1] <= 5 and n[2] > 50
    return f"B = 3 with {n} keypoints"


def disk_cases():
    cases = []
    for window in (1, 3, 5, 7):
        r = window // 2
        heat = _bg(1, 32, 48, window)
        heat[0, 10:12, 10:12] = 1.0
        heat[0, 0:2, 0:2] = 1.0
        heat[0, 10, 11 + r + 1] = 1.0
        cases.append(DiskCase(f"plateau, window {window}", heat, window, 0.0, None, _plateau(window)))
    heat = _bg(1, 48, 64, 9)
    g = torch.Generator().manual_seed(9)
    for i in range(20):
        heat[0, 6 + 8 * (i // 6), 5 + 10 * (i % 6)] = 1.0 + torch.rand(1, generator=g).item()
    for name, n, want in (("None", None, lambda c: c), ("0", 0, lambda c: 0), ("count - 1", lambda c: c - 1, lambda c: c - 1),
                          ("count", lambda c: c, lambda c: c - 1), ("count + 1", lambda c: c + 1, lambda c: c - 1)):
        cases.append(DiskCase(f"top-k: n = {name}", heat, 5, 0.0, n, _kcount(want)))
    heat = _bg(1, 16, 64, 10)
    for x, v in zip(range(4, 64, 8), (5.0, 4.0, 3.0, 3.0, 3.0, 2.0, 1.0)):
        heat[0, 8, x] = v
    cases.append(DiskCase("top-k: tie at the (n + 1)-th score", heat, 5, 0.0, 3, _tie_n1))
    heat = (-(torch.arange(64) % 8) * 0.25).view(1, 1, 64).expand(1, 64, 64).contiguous()
    cases.append(DiskCase("top-k: tie across a 1024 chunk", heat, 1, -10.0, 1500, _chunk_tie))
    heat = _bg(1, 32, 32, 11)
    heat[0, 5, 5], heat[0, 5, 20] = 0.5, 0.75
    cases.append(DiskCase("threshold equal to a heat value", heat, 5, 0.5, None, _thr_eq))
    g = torch.Generator().manual_seed(12)
    cases.append(DiskCase("1040x32", torch.randn(1, 1040, 32, generator=g), 5, 0.0, None, _tall_disk))
    heat = _bg(3, 48, 64, 13)
    heat[1, 10, 10], heat[1, 30, 40] = 2.0, 3.0
    heat[2] = torch.randn(48, 64, generator=g)
    cases.append(DiskCase("B = 3, one image without candidates", heat, 5, 0.0, None, _batch_disk))
    return cases


def disk_n(case):
    if callable(case.n):
        return case.n(disk_candidates(case.heat[0], case.window, case.threshold).numel())
    return case.n
