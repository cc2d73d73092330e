"""Every GPU estimator of include/geometry_b200.h at its launch-shape and value bounds against its numpy oracle, pair by
pair: find_homography, find_fundamental, find_homography_lo, estimate_relative_pose, estimate_relative_pose_lo and
estimate_absolute_pose.

The other GPU geometry files test a 640x480 frame, M <= 4096, B <= 32, 1-8 px thresholds and finite keypoints.  Here:
score kernels with one split of several shared-memory tiles and with the most splits; more pairs than a grid's y extent
(65 535); the chunk edges of the sample budget; empty pairs; the LO bound M = GEO_LO_MAX_MATCHES; squared thresholds of
0, a subnormal, FLT_MIN and +inf in fp32; large, far-off and integer coordinates; non-finite keypoints; duplicates.
Each launch-shape case asserts the regime it reaches from the score kernels' split rule, so a change of that rule
cannot make a case vacuous unnoticed."""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Callable

import numpy as np
import pytest
import torch

from lightglue_b200 import _cabi
from lightglue_b200.geometry import (estimate_absolute_pose, estimate_relative_pose, estimate_relative_pose_lo,
                                     find_fundamental, find_homography, find_homography_lo)
from oracle import geometry_oracle as go
from oracle import geometry_synth as gs
from oracle import lo_homography_oracle as lh
from oracle import lo_pose_oracle as lo
from oracle import pnp_oracle as pp
from oracle import pose_oracle as po

pytestmark = pytest.mark.gpu

FLT_MIN = float(np.finfo(np.float32).tiny)  # 2^-126
SUBNORMAL = 2.0 ** -140                      # an fp32 subnormal: QSCALE / it overflows to +inf


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


@dataclass(frozen=True)
class Est:
    """One estimator: its entry point, its oracle's per-pair function, the outputs that must match exactly, the masks,
    the models held to 1e-8 (GPU key -> oracle key), a seeded scene, and the constants of its score kernel."""
    name: str
    gpu: Callable          # (a, b, m0, K, **kw) -> dict of device tensors
    oracle: Callable       # (a, b, m0, K, threshold, max_iters, confidence, seed) -> dict for one pair
    exact: tuple
    masks: tuple
    models: dict
    scene: Callable        # (m, outliers, seed, unmatched) -> (a, b, m0, K)
    threshold: float       # default, pixels
    focal: bool            # thr2 = (float)((threshold / f)^2), f the mean focal length
    tile: int              # points per shared-memory tile of the score kernel
    workspace: str         # the *_workspace_bytes entry point
    lo: bool = False
    relative: bool = True  # models compared relative to their largest entry, else absolutely


def _planar(m, outliers, seed, unmatched):
    k0, k1, m0, _, _ = gs.planar(m, outliers, seed, noise=1.0, unmatched=unmatched)
    return k0, k1, m0, None


def _two_view(m, outliers, seed, unmatched):
    k0, k1, m0, _, _ = gs.two_view(m, outliers, seed, unmatched=unmatched)
    return k0, k1, m0, None


def _calibrated(m, outliers, seed, unmatched):
    k0, k1, m0, _, K, _, _, _ = po.calibrated_two_view(m, outliers, seed, unmatched=unmatched)
    return k0, k1, m0, K


def _localization(m, outliers, seed, unmatched):
    k0, p3, m0, _, K, _, _ = pp.localization_scene(m, outliers, seed, unmatched=unmatched)
    return k0, p3, m0, K


_H_EXACT = ("best_hypothesis", "num_hypotheses", "num_inliers", "success")
_POSE_EXACT = ("best_hypothesis", "best_solution", "num_hypotheses", "num_inliers", "num_pose_inliers", "success")
_LO = ("num_local_optimizations", "cost")

ESTIMATORS = {e.name: e for e in (
    Est("H", lambda a, b, m0, K, **kw: find_homography(_t(a), _t(b), _t(m0), **kw),
        lambda a, b, m0, K, thr, it, conf, seed: go.estimate_pair(go.HOMOGRAPHY, a, b, m0, thr, it, conf, seed),
        _H_EXACT, ("inliers",), {"H": "model"}, _planar, 3.0, False, 1024, "geo_workspace_bytes"),
    Est("F", lambda a, b, m0, K, **kw: find_fundamental(_t(a), _t(b), _t(m0), **kw),
        lambda a, b, m0, K, thr, it, conf, seed: go.estimate_pair(go.FUNDAMENTAL, a, b, m0, thr, it, conf, seed),
        _H_EXACT, ("inliers",), {"F": "model"}, _two_view, 3.0, False, 1024, "geo_workspace_bytes"),
    Est("LO-H", lambda a, b, m0, K, **kw: find_homography_lo(_t(a), _t(b), _t(m0), **kw),
        lambda a, b, m0, K, thr, it, conf, seed: lh.lo_homography_pair(a, b, m0, thr, it, conf, seed),
        _H_EXACT + _LO, ("inliers",), {"H": "H"}, _planar, 3.0, False, 1024, "geo_lo_homography_workspace_bytes",
        lo=True),
    Est("pose", lambda a, b, m0, K, **kw: estimate_relative_pose(_t(a), _t(b), _t(m0), _t(K), **kw),
        lambda a, b, m0, K, thr, it, conf, seed: po.relative_pose_pair(a, b, m0, K, K, thr, it, conf, 50.0, seed),
        _POSE_EXACT, ("inliers", "pose_inliers"), {"E": "E", "R": "R", "t": "t"}, _calibrated, 1.0, True, 1024,
        "geo_pose_workspace_bytes", relative=False),
    Est("LO-pose", lambda a, b, m0, K, **kw: estimate_relative_pose_lo(_t(a), _t(b), _t(m0), _t(K), **kw),
        lambda a, b, m0, K, thr, it, conf, seed: lo.lo_relative_pose_pair(a, b, m0, K, K, thr, it, conf, 50.0, seed),
        _POSE_EXACT + _LO, ("inliers", "pose_inliers"), {"E": "E", "R": "R", "t": "t"}, _calibrated, 1.0, True, 1024,
        "geo_lo_pose_workspace_bytes", lo=True, relative=False),
    Est("PnP", lambda a, b, m0, K, **kw: estimate_absolute_pose(_t(a), _t(b), _t(m0), _t(K), **kw),
        lambda a, b, m0, K, thr, it, conf, seed: pp.absolute_pose_pair(a, b, m0, K, thr, it, conf, seed),
        ("best_hypothesis", "best_solution", "num_hypotheses", "num_inliers", "success"), ("inliers",),
        {"R": "R", "t": "t"}, _localization, 8.0, False, 512, "geo_pnp_workspace_bytes", relative=False),
)}
NAMES = list(ESTIMATORS)
TWO_VIEW = ["H", "F", "LO-H", "pose", "LO-pose"]


def _batch(e: Est, m, seeds, outliers=0.3, unmatched=0.1):
    """Stacked scenes: (a [B, m, 2], b [B, N, 2 or 3], m0 [B, m], K [3, 3] or None)."""
    outs = np.broadcast_to(np.asarray(outliers, dtype=float), (len(seeds),))
    unm = np.broadcast_to(np.asarray(unmatched, dtype=float), (len(seeds),))
    scenes = [e.scene(m, o, s, u) for s, o, u in zip(seeds, outs, unm)]
    return (*(np.stack([sc[i] for sc in scenes]) for i in range(3)), scenes[0][3])


def _kw(e: Est, threshold=None, max_iters=256, confidence=1.0, seed=0):
    return dict(ransac_reproj_threshold=e.threshold if threshold is None else threshold, max_iters=max_iters,
                confidence=confidence, seed=seed)


def _run(e: Est, a, b, m0, K, **kw):
    return {k: v.cpu().numpy() for k, v in e.gpu(a, b, m0, K, **kw).items()}


def _oracle(e: Est, a, b, m0, K, pairs, ransac_reproj_threshold, max_iters, confidence, seed):
    return [e.oracle(a[p], b[p], m0[p], K, ransac_reproj_threshold, max_iters, confidence, seed) for p in pairs]


def _assert_equal(e: Est, got, refs, pairs):
    for r, p in zip(refs, pairs):
        for k in e.exact:
            assert got[k][p] == r[k], (e.name, p, k, got[k][p], r[k])
        for k in e.masks:
            assert np.array_equal(got[k][p], r[k]), (e.name, p, k, int((got[k][p] != r[k]).sum()))
        for gk, rk in e.models.items():
            ref = np.asarray(r[rk])
            assert np.isfinite(got[gk][p]).all(), (e.name, p, gk)
            tol = 1e-8 * max(np.abs(ref).max(), 1e-300) if e.relative else 1e-8
            assert np.abs(got[gk][p] - ref).max() <= tol, (e.name, p, gk, got[gk][p], ref)


def _check(e: Est, a, b, m0, K, pairs=None, **kw):
    """Run the batch on the GPU and compare the given pairs (default: all) with the oracle; returns the GPU outputs."""
    got = _run(e, a, b, m0, K, **kw)
    pairs = range(len(m0)) if pairs is None else pairs
    _assert_equal(e, got, _oracle(e, a, b, m0, K, pairs, **kw), pairs)
    return got


def _valid(e: Est, a, b, m0):
    """Per pair, the number of valid matches n of header steps 1 and A1."""
    n1 = b.shape[1]
    ok = (m0 >= 0) & (m0 < n1)
    rows = np.take_along_axis(b, np.clip(m0, 0, max(n1 - 1, 0))[..., None], 1) if n1 else np.zeros(a.shape[:2] + (1,))
    return (ok & np.isfinite(a).all(-1) & np.isfinite(rows).all(-1)).sum(1)


def _splits(B, M):
    """The score kernels' CTAs per pair: enough to cover the SMs twice, at least 128 rows per slice."""
    want = -(-2 * torch.cuda.get_device_properties(0).multi_processor_count // B)
    return max(1, min(-(-M // 128), want))


def _thr2(e: Est, threshold, K):
    """The fp32 squared threshold the estimator compares against."""
    if e.focal:
        return po.threshold2(np.asarray(K).reshape(9), np.asarray(K).reshape(9), threshold)
    return np.float32(threshold * threshold)


def _threshold_for(e: Est, thr2, K):
    """A pixel threshold whose squared fp32 comparison value is thr2 (a power of two, so the square is exact)."""
    f = (((K[0, 0] + K[1, 1]) + K[0, 0]) + K[1, 1]) / 4.0 if e.focal else 1.0
    return math.sqrt(thr2) * f


def _assert_lo_sane(e: Est, got, n):
    if e.lo:
        assert (got["cost"] >= 0).all() and (got["cost"] < 1 << 40).all(), got["cost"]
        assert (got["num_inliers"] <= n).all(), (got["num_inliers"], n)


# ----------------------------------------------------------------------------------------------------- launch shapes


@pytest.mark.parametrize("name", NAMES)
def test_one_split_of_several_tiles(name):
    # B = 2 SMs + 1 pairs: one score CTA per pair, which streams its ~2700 points through three tiles (six for PnP's
    # 512-point tile), the last one partial
    e = ESTIMATORS[name]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    B, M = 2 * sms + 1, 3000
    a, b, m0, K = _batch(e, M, [1000 + i for i in range(B)], outliers=[0.2, 0.5, 0.35] * (B // 3) + [0.2] * (B % 3))
    n = _valid(e, a, b, m0)
    assert _splits(B, M) == 1
    assert (n > 2 * e.tile).all() and (n % e.tile != 0).any(), n
    kw = _kw(e)
    pairs = np.linspace(0, B - 1, 8).astype(int).tolist()
    got = _check(e, a, b, m0, K, pairs=pairs, **kw)
    assert got["success"].all()
    for p in range(B):
        one = _run(e, a[p:p + 1], b[p:p + 1], m0[p:p + 1], K, **kw)
        for k in got:
            assert np.array_equal(got[k][p], one[k][0]), (p, k)


@pytest.mark.parametrize("name,m,unmatched", [(n, (1 << 17) + 37, 0.1) for n in NAMES]
                         + [("H", 300_000, 0.0), ("F", 300_000, 0.0), ("PnP", 300_000, 0.0)])
def test_most_splits(name, m, unmatched):
    # B = 1: 2 SMs splits per pair.  At 2^17 + 37 rows each split holds under one tile; at 300 000 fully matched rows
    # each holds more than one, so every split also runs a second, partial tile.  For the LO estimators this is also
    # the realistic large case: 2^17 matches at the default 3 px (H) and 1 px (pose).
    e = ESTIMATORS[name]
    a, b, m0, K = _batch(e, m, [77], outliers=0.4, unmatched=unmatched)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    splits = _splits(1, m)
    assert splits == 2 * sms
    n = int(_valid(e, a, b, m0)[0])
    if m == 300_000:
        assert n // splits > e.tile, (n, splits)
    got = _check(e, a, b, m0, K, **_kw(e))
    assert got["success"][0] and got["num_hypotheses"][0] == 256


def _many_pairs(e: Est, B, M, seed=5):
    """B pairs of M rows: 256 seeded scenes tiled over the batch, each pair with its own random unmatched rows."""
    a, b, m0, K = _batch(e, M, [seed * 1000 + i for i in range(256)], outliers=0.25, unmatched=0.0)
    idx = np.arange(B) % 256
    a, b, m0 = a[idx], b[idx], m0[idx].copy()
    m0[np.random.default_rng(seed).random(m0.shape) < 0.15] = -1
    return a, b, m0, K


@pytest.mark.parametrize("name", NAMES)
def test_more_pairs_than_a_grid_column(name):
    # B = 65 537 > 65 535, the largest grid y extent: the pair index must sit on grid x
    e = ESTIMATORS[name]
    B, M = 65_537, 16
    kw = _kw(e)
    ws = getattr(_cabi.load(), e.workspace)(B, M, kw["max_iters"])
    assert 0 < ws < 16 << 30, ws
    a, b, m0, K = _many_pairs(e, B, M)
    assert _splits(B, M) == 1
    got = _check(e, a, b, m0, K, pairs=[0, B // 2, B - 1], **kw)
    assert got["success"].mean() > 0.5
    for s in range(0, B, 4096):
        part = _run(e, a[s:s + 4096], b[s:s + 4096], m0[s:s + 4096], K, **kw)
        for k in got:
            assert np.array_equal(got[k][s:s + 4096], part[k]), (s, k)


# ------------------------------------------------------------------------------------------------------ sample budget


@pytest.mark.parametrize("max_iters", [1, 255, 257, 513])
@pytest.mark.parametrize("name", NAMES)
def test_chunk_edges(name, max_iters):
    e = ESTIMATORS[name]
    a, b, m0, K = _batch(e, 400, [31, 32], outliers=[0.3, 0.6])
    got = _check(e, a, b, m0, K, **_kw(e, max_iters=max_iters))
    assert (got["num_hypotheses"] == max_iters).all(), got["num_hypotheses"]


@pytest.mark.parametrize("name", NAMES)
def test_adaptive_stop_mid_budget(name):
    e = ESTIMATORS[name]
    a, b, m0, K = _batch(e, 600, [41, 42], outliers=0.15)
    got = _check(e, a, b, m0, K, **_kw(e, max_iters=2000, confidence=0.99))
    h = got["num_hypotheses"]
    assert ((h >= 256) & (h < 2000) & (h % 256 == 0)).all(), h


@pytest.mark.parametrize("name", NAMES)
def test_empty_pairs(name):
    e = ESTIMATORS[name]
    a, b, m0, K = _batch(e, 300, [51, 52, 53])
    m0[1] = -1  # no valid match in the middle pair
    got = _check(e, a, b, m0, K, **_kw(e))
    assert got["success"][0] and got["success"][2] and not got["success"][1] and got["num_hypotheses"][1] == 0
    # M = 0 and N = 0 for the whole batch: every pair fails without drawing
    for aa, bb, mm in ((a[:, :0], b, m0[:, :0]), (a, b[:, :0], m0)):
        got = _check(e, aa, bb, mm, K, **_kw(e))
        assert not got["success"].any() and not got["num_hypotheses"].any()


# ------------------------------------------------------------------------------------------------------------ values


@pytest.mark.parametrize("name", ["LO-H", "LO-pose"])
def test_lo_bound_with_every_point_an_outlier(name):
    # M = GEO_LO_MAX_MATCHES fully matched rows and a threshold whose fp32 square is 0: every hypothesis scores
    # QSCALE * n, the largest score the packed (score, h) key must hold
    e = ESTIMATORS[name]
    M = _cabi.GEO_LO_MAX_MATCHES
    a, b, m0, K = _batch(e, M, [61], outliers=0.3, unmatched=0.0)
    threshold = 1e-30
    assert _thr2(e, threshold, K) == 0.0
    got = _check(e, a, b, m0, K, **_kw(e, threshold=threshold, max_iters=8))
    assert got["success"][0] and got["num_inliers"][0] == 0
    assert got["cost"][0] == lo.QSCALE * M


@pytest.mark.parametrize("thr2", [0.0, SUBNORMAL, FLT_MIN, math.inf], ids=["zero", "subnormal", "flt_min", "inf"])
@pytest.mark.parametrize("name", NAMES)
def test_threshold_extremes(name, thr2):
    e = ESTIMATORS[name]
    a, b, m0, K = _batch(e, 500, [71, 72], outliers=[0.2, 0.5])
    Kn = np.eye(3) if K is None else K
    threshold = {0.0: 1e-30, math.inf: 1e20 * (500.0 if e.focal else 1.0)}.get(thr2) or _threshold_for(e, thr2, Kn)
    got_thr2 = _thr2(e, threshold, Kn)
    assert got_thr2 == np.float32(thr2), (got_thr2, thr2)
    if thr2 == SUBNORMAL:
        assert 0.0 < got_thr2 < FLT_MIN
    got = _check(e, a, b, m0, K, **_kw(e, threshold=threshold))
    n = _valid(e, a, b, m0)
    _assert_lo_sane(e, got, n)
    if thr2 == math.inf and name in TWO_VIEW:  # every finite error is an inlier (PnP's also need positive depth)
        assert (got["num_inliers"] == n).all() and (not e.lo or not got["cost"].any())


def _frame(e: Est, a, b, K, scale, offset):
    """The scene in pixels scaled by scale and shifted by offset in both images (K follows), float32."""
    S = np.array([[scale, 0.0, offset[0]], [0.0, scale, offset[1]], [0.0, 0.0, 1.0]])
    a = (a.astype(np.float64) * scale + offset).astype(np.float32)
    if b.shape[-1] == 2:
        b = (b.astype(np.float64) * scale + offset).astype(np.float32)
    return a, b, None if K is None else S @ K, S


@pytest.mark.parametrize("case", ["8192x6144", "offset", "integer"])
@pytest.mark.parametrize("name", NAMES)
def test_coordinates(name, case):
    e = ESTIMATORS[name]
    M = 800
    a, b, m0, K = _batch(e, M, [81, 82], outliers=[0.2, 0.4])
    threshold = e.threshold
    if case == "8192x6144":
        a, b, K, _ = _frame(e, a, b, K, 12.8, (0.0, 0.0))
        threshold = e.threshold * 12.8
    elif case == "offset":
        a, b, K, S = _frame(e, a, b, K, 1.0, (1e5, -1e5))
    else:
        rng = np.random.default_rng(83)
        a = np.rint(a).astype(np.float32)
        if b.shape[-1] == 2:  # image 1 is image 0 moved by whole pixels: exact zero errors for the true model
            moved = a + np.array([17.0, -5.0], dtype=np.float32)
            for p in range(len(m0)):
                ok = m0[p] >= 0
                b[p, m0[p, ok]] = moved[p, ok]
                out = ok & (rng.random(M) < 0.3)
                b[p, m0[p, out]] = rng.integers(0, 600, (int(out.sum()), 2)).astype(np.float32)
    got = _check(e, a, b, m0, K, **_kw(e, threshold=threshold))
    if case == "offset" and name in ("H", "LO-H"):
        corners = gs.CORNERS + np.array([1e5, -1e5])
        for p, Hm in enumerate(gs.planar(M, 0.0, s)[4] for s in (81, 82)):  # the scene's H: its first draws
            Ht = S @ Hm @ np.linalg.inv(S)
            assert np.abs(gs.apply_h(got["H"][p], corners) - gs.apply_h(Ht, corners)).max() <= 1.0, p
    if case == "integer" and name in ("H", "LO-H"):
        assert got["success"].all() and (got["num_inliers"] > 0).all()


@pytest.mark.parametrize("name", NAMES)
def test_non_finite_keypoints_are_invalid(name):
    # NaN, +inf and -inf in a kpts0 row or in the kpts1 (PnP: points3d1) row of a valid match, at one row and at 10 %
    # of the rows: such a match is no inlier and does not count, exactly as if matches0 were -1 there
    e = ESTIMATORS[name]
    M = 500
    cases = [(v, side, frac) for v in (np.nan, np.inf, -np.inf) for side in (0, 1) for frac in (None, 0.1)]
    a, b, m0, K = _batch(e, M, [90 + i for i in range(len(cases))], outliers=0.3)
    a, b = a.copy(), b.copy()
    clean = m0.copy()
    rng = np.random.default_rng(91)
    bad = np.zeros(m0.shape, dtype=bool)
    for p, (v, side, frac) in enumerate(cases):
        valid = np.nonzero((m0[p] >= 0) & np.isfinite(b[p, np.maximum(m0[p], 0)]).all(1))[0]
        rows = rng.choice(valid, 1 if frac is None else int(frac * M), replace=False)
        coord = rng.integers(0, b.shape[-1] if side else 2, rows.size)
        if side == 0:
            a[p, rows, coord] = v
        else:
            b[p, m0[p, rows], coord] = v
        clean[p, rows] = -1
        bad[p, rows] = True
    kw = _kw(e)
    got = _run(e, a, b, m0, K, **kw)
    ref = _run(e, a, b, clean, K, **kw)
    for k in got:
        assert np.array_equal(got[k], ref[k]), k
    for k in e.masks:
        assert not got[k][bad].any(), k
    pairs = range(len(cases))
    _assert_equal(e, got, _oracle(e, a, b, clean, K, pairs, **kw), pairs)
    assert got["success"].all()


@pytest.mark.parametrize("name", NAMES)
def test_duplicate_points_and_matches(name):
    # half of the rows of image 0 share 20 coordinates, and 64 rows of matches0 point at one column
    e = ESTIMATORS[name]
    M = 512
    a, b, m0, K = _batch(e, M, [95, 96], outliers=0.2)
    a, m0 = a.copy(), m0.copy()
    rng = np.random.default_rng(97)
    for p in range(len(m0)):
        half = rng.choice(M, M // 2, replace=False)
        pool = rng.choice(M, 20, replace=False)
        a[p, half] = a[p, pool[rng.integers(0, 20, half.size)]]
        j = m0[p, np.nonzero(m0[p] >= 0)[0][0]]
        m0[p, rng.choice(M, 64, replace=False)] = j
    _check(e, a, b, m0, K, **_kw(e, confidence=0.99, max_iters=600))
