"""The value bounds of the geometry estimators without a GPU: the LO match bound and the key it protects, the MSAC
score term at a subnormal threshold (w = +inf) and at a zero error, and the rule that a non-finite keypoint or 3D point
invalidates its match at compaction (include/geometry_b200.h steps 1, A1, L3 and LH3; the oracles restate them)."""
import ctypes
import os
import re

import numpy as np
import pytest

from lightglue_b200 import _cabi
from oracle import geometry_oracle as go
from oracle import lo_homography_oracle as lh
from oracle import lo_pose_oracle as lo
from oracle import pnp_oracle as pp
from oracle import pose_oracle as po

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SUBNORMAL = np.float32(2.0 ** -140)
FLT_MIN = np.finfo(np.float32).tiny


def _header():
    with open(os.path.join(ROOT, "include", "geometry_b200.h")) as f:
        return f.read()


def test_lo_bound_keeps_the_largest_score_inside_the_key():
    # the LO kernels pack (score, h) as score << 28 | h in 64 bits: the largest score, QSCALE * M, must stay below 2^36
    m = (1 << 20) - 1
    assert _cabi.GEO_LO_MAX_MATCHES == m
    assert re.search(r"#define GEO_LO_MAX_MATCHES \(\(1 << 20\) - 1\)", _header())
    assert lo.QSCALE * m < 1 << 36 and (lo.QSCALE * m) << 28 < 1 << 64
    assert (lo.QSCALE * (m + 1)) << 28 == 1 << 64  # one more row would wrap to a zero key
    # the score field of a sum holds the same bound below the count at bit 40
    assert lo.QSCALE * m < 1 << 40 and m < 1 << 24


@pytest.mark.parametrize("entry", ["geo_homography_lo", "geo_relative_pose_lo"])
def test_the_c_abi_accepts_the_bound_and_rejects_one_more_row(entry):
    lib = _cabi.load()
    if entry == "geo_homography_lo":
        cfg = _cabi.GeoConfig(_cabi.GEO_ABI_VERSION, _cabi.GEO_HOMOGRAPHY, 100, 0, 3.0, 0.99)
        ins = lambda m: _cabi.GeoInputs(0, m, 4, 0, 0, 0)  # noqa: E731
        outs = _cabi.GeoLoOutputs()
    else:
        cfg = _cabi.GeoLoPoseConfig(_cabi.GEO_ABI_VERSION, 100, 0, 0, 1.0, 0.99, 50.0)
        ins = lambda m: _cabi.GeoPoseInputs(0, m, 4, 0, 0, 0, 0, 0)  # noqa: E731
        outs = _cabi.GeoLoPoseOutputs()
    fn = getattr(lib, entry)
    # B = 0: the size checks run and nothing launches
    call = lambda m: fn(ctypes.byref(cfg), ctypes.byref(ins(m)), ctypes.byref(outs), None, 0, None)  # noqa: E731
    assert call(_cabi.GEO_LO_MAX_MATCHES) == 0
    assert call(_cabi.GEO_LO_MAX_MATCHES + 1) != 0
    assert "GEO_LO_MAX_MATCHES" in lib.lg_last_error().decode()


def test_score_term_is_clamped_when_w_is_infinite():
    # thr2 subnormal or FLT_MIN: w = QSCALE / thr2 = +inf; an inlier with 0 < err scores QSCALE, err == 0 scores 0
    for thr2 in (SUBNORMAL, np.float32(FLT_MIN)):
        with np.errstate(over="ignore"):
            assert np.isinf(np.float32(lo.QSCALE) / thr2)
        err = np.array([0.0, thr2 / np.float32(2), thr2, np.inf, np.nan], dtype=np.float32)
        s, c = lo.score(err, thr2)
        assert int(c) == 2
        assert int(s) == 0 + lo.QSCALE + lo.QSCALE + lo.QSCALE + lo.QSCALE


def test_score_term_at_zero_error_and_thresholds_zero_and_infinite():
    err = np.array([0.0, 1.0, 4.0], dtype=np.float32)
    s, c = lo.score(err, np.float32(0.0))  # nothing is below 0: every point is an outlier
    assert int(c) == 0 and int(s) == 3 * lo.QSCALE
    s, c = lo.score(err, np.float32(np.inf))  # w = 0: every finite point is an inlier scoring 0
    assert int(c) == 3 and int(s) == 0
    s, c = lo.score(np.array([np.inf], dtype=np.float32), np.float32(np.inf))
    assert int(c) == 0 and int(s) == lo.QSCALE


def test_score_term_is_unchanged_for_finite_w():
    # for a normal thr2 an inlier's product truncates to at most QSCALE, so the clamp moves nothing
    rng = np.random.default_rng(0)
    for thr2 in (np.float32(9.0), np.float32(1e-6), np.float32(4e-34)):
        w = np.float32(lo.QSCALE) / thr2
        assert np.isfinite(w)
        err = np.concatenate([rng.random(4096).astype(np.float32) * thr2, [thr2 * np.float32(0.99999994), 0.0]])
        err = err.astype(np.float32)
        inl = err < thr2
        plain = np.where(inl, (err * w).astype(np.uint32), np.uint32(lo.QSCALE)).astype(np.uint64)
        s, c = lo.score(err, thr2)
        assert int(s) == int(plain.sum()) and int(c) == int(inl.sum())
        assert (err[inl] * w <= lo.QSCALE).all()


def test_score_terms_are_batched_over_leading_axes():
    err = np.array([[0.0, 0.5, 2.0], [1.0, 0.0, np.nan]], dtype=np.float32)
    s, c = lo.score(err, np.float32(1.0))
    assert s.tolist() == [0 + 32768 + lo.QSCALE, lo.QSCALE + 0 + lo.QSCALE] and c.tolist() == [2, 1]


@pytest.mark.parametrize("value", [np.nan, np.inf, -np.inf])
def test_compaction_drops_non_finite_keypoints(value):
    rng = np.random.default_rng(1)
    k0 = rng.uniform(0, 640, (10, 2)).astype(np.float32)
    k1 = rng.uniform(0, 640, (8, 2)).astype(np.float32)
    m0 = np.array([0, 1, -1, 3, 4, 5, 9, 7, 2, 6], dtype=np.int64)  # row 6 is out of range
    k0[1, 0] = value      # row 1 invalid through kpts0
    k1[4, 1] = value      # row 4 invalid through kpts1[4]
    k0[2, 1] = value      # row 2 is unmatched anyway
    rows, pts = go.compact(k0, k1, m0)
    assert rows.tolist() == [0, 3, 5, 7, 8, 9]
    assert np.isfinite(pts).all() and np.array_equal(pts[:, :2], k0[rows])
    assert np.array_equal(pts[:, 2:], k1[m0[rows]])


def test_compaction_ignores_non_finite_rows_nobody_matches():
    k0 = np.zeros((3, 2), dtype=np.float32)
    k1 = np.array([[np.nan, 0.0], [1.0, 1.0], [2.0, 2.0]], dtype=np.float32)
    rows, _ = go.compact(k0, k1, np.array([1, 2, 1], dtype=np.int64))
    assert rows.tolist() == [0, 1, 2]
    rows, pts = go.compact(k0[:0], k1, np.zeros(0, dtype=np.int64))
    assert rows.size == 0 and pts.shape == (0, 4)
    rows, pts = go.compact(k0, k1[:0], np.array([0, 1, -1], dtype=np.int64))
    assert rows.size == 0 and pts.shape == (0, 4)


@pytest.mark.parametrize("value", [np.nan, np.inf, -np.inf])
def test_pnp_compaction_drops_non_finite_pixels_and_points(value):
    rng = np.random.default_rng(2)
    k0 = rng.uniform(0, 640, (6, 2)).astype(np.float32)
    p3 = rng.uniform(-1, 1, (6, 3)).astype(np.float32)
    m0 = np.array([5, 4, 3, 2, 1, 0], dtype=np.int64)
    k0[0, 1] = value   # row 0: non-finite pixel
    p3[3, 2] = value   # row 2: non-finite 3D point
    rows, pix, wld = pp.compact(k0, p3, m0)
    assert rows.tolist() == [1, 3, 4, 5]
    assert np.isfinite(pix).all() and np.isfinite(wld).all()


def _poisoned(rows_frac, seed, make):
    k0, k1, m0, *rest = make(seed)
    k0, k1 = k0.copy(), k1.copy()
    rng = np.random.default_rng(seed)
    valid = np.nonzero((m0 >= 0) & np.isfinite(k1[np.maximum(m0, 0)]).all(1))[0]
    rows = rng.choice(valid, max(1, int(rows_frac * len(m0))), replace=False)
    half = rows.size // 2
    k0[rows[:half], 0] = np.nan
    k1[m0[rows[half:]], 1] = np.inf
    clean = m0.copy()
    clean[rows] = -1
    return k0, k1, m0, clean, rows, rest


def _same(a, b):
    for k in a:
        assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), k


@pytest.mark.parametrize("frac", [0.0, 0.1])
def test_estimators_treat_a_non_finite_match_as_unmatched(frac):
    # one row (frac 0) or 10 % of the rows: every oracle equals itself on the input with those rows unmatched
    k0, k1, m0, clean, rows, _ = _poisoned(frac, 3, lambda s: po.calibrated_two_view(300, 0.3, s)[:3])
    K = np.array([[500.0, 0.0, 320.0], [0.0, 500.0, 240.0], [0.0, 0.0, 1.0]])
    for fn in (lambda m: go.estimate_pair(go.HOMOGRAPHY, k0, k1, m, 3.0, 256, 1.0, 0),
               lambda m: go.estimate_pair(go.FUNDAMENTAL, k0, k1, m, 3.0, 256, 1.0, 0),
               lambda m: lh.lo_homography_pair(k0, k1, m, 3.0, 256, 1.0, 0),
               lambda m: po.relative_pose_pair(k0, k1, m, K, K, 1.0, 256, 1.0, 50.0, 0),
               lambda m: lo.lo_relative_pose_pair(k0, k1, m, K, K, 1.0, 256, 1.0, 50.0, 0)):
        a, b = fn(m0), fn(clean)
        _same(a, b)
        assert a["success"] and not a["inliers"][rows].any()
    k0, p3, m0, clean, rows, _ = _poisoned(frac, 4, lambda s: pp.localization_scene(300, 0.3, s)[:3])
    a = pp.absolute_pose_pair(k0, p3, m0, K, 8.0, 256, 1.0, 0)
    _same(a, pp.absolute_pose_pair(k0, p3, clean, K, 8.0, 256, 1.0, 0))
    assert a["success"] and not a["inliers"][rows].any()


def test_inlier_masks_may_be_null_only_when_empty():
    # an empty [B, 0] mask has no storage; with M > 0 a null mask is still refused before anything launches
    lib = _cabi.load()
    cfg = _cabi.GeoConfig(_cabi.GEO_ABI_VERSION, _cabi.GEO_HOMOGRAPHY, 100, 0, 3.0, 0.99)
    ins = _cabi.GeoInputs(1, 4, 4, 8, 8, 8)  # non-null placeholders: the output check comes first
    outs = _cabi.GeoOutputs(8, 0, 8, 8, 8, 8)
    assert lib.geo_estimate(ctypes.byref(cfg), ctypes.byref(ins), ctypes.byref(outs), None, 0, None) != 0
    assert "null output" in lib.lg_last_error().decode()
