"""The affine and partial affine oracle (oracle/affine_oracle.py, include/geometry_b200.h steps AF1-AF7) without a GPU:
the refinement reaches the linear least-squares fit, noise-free scenes give the true transform and OpenCV's, synthetic
scenes are estimated at least as well as cv2.estimateAffine2D / estimateAffinePartial2D, degenerate samples and pairs
fail as AF3 and AF7 say, and the inlier test is step 5's homography error on [A; 0 0 1] bit for bit."""
import numpy as np
import pytest

from oracle import affine_oracle as ao
from oracle import geometry_oracle as go

cv2 = pytest.importorskip("cv2")

KINDS = [ao.AFFINE, ao.PARTIAL]
CV = {ao.AFFINE: "estimateAffine2D", ao.PARTIAL: "estimateAffinePartial2D"}
CORNERS = np.array([[0.0, 0.0, 1.0], [640.0, 0.0, 1.0], [640.0, 480.0, 1.0], [0.0, 480.0, 1.0]])


def _cv(kind, k0, k1, m0, threshold=3.0):
    v = m0 >= 0
    A, mask = getattr(cv2, CV[kind])(k0[v], k1[m0[v]], method=cv2.RANSAC, ransacReprojThreshold=threshold,
                                     maxIters=2000, confidence=0.99, refineIters=10)
    full = np.zeros(m0.shape, dtype=bool)
    full[np.flatnonzero(v)] = mask.ravel().astype(bool)
    return A, full


def _corner_error(A, truth):
    return float(np.linalg.norm((A - truth) @ CORNERS.T, axis=0).mean())


def _iou(a, b):
    return float((a & b).sum() / max((a | b).sum(), 1))


def _lstsq(kind, pts, inl):
    """The linear least-squares transform of the inliers, in pixels, by numpy.linalg.lstsq."""
    x, y, u, v = (pts[inl, q].astype(np.float64) for q in range(4))
    one, zero = np.ones_like(x), np.zeros_like(x)
    if kind == ao.PARTIAL:  # u = a x - b y + tx, v = b x + a y + ty
        D = np.concatenate([np.stack([x, -y, one, zero], 1), np.stack([y, x, zero, one], 1)])
        a, b, tx, ty = np.linalg.lstsq(D, np.concatenate([u, v]), rcond=None)[0]
        return np.array([[a, -b, tx], [b, a, ty]])
    D = np.stack([x, y, one], 1)
    return np.stack([np.linalg.lstsq(D, u, rcond=None)[0], np.linalg.lstsq(D, v, rcond=None)[0]])


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_refinement_reaches_the_least_squares_fit(kind, seed):
    k0, k1, m0, truth, _ = ao.scene(kind, 1024, 0.3, seed, noise=0.8)
    r = ao.estimate_pair(kind, k0, k1, m0)
    _, pts = go.compact(k0, k1, m0)
    norm = go.normalisation(pts)
    X, A, _ = ao.hypotheses(kind, 0, np.array([r["best_hypothesis"]]), pts, norm)
    inl = ao.errors(A, pts)[0] < np.float32(9.0)  # the hypothesis's inliers: the refinement's fixed set
    refined = ao.pixels(kind, norm, ao.refine(kind, norm, pts, inl, X[0], 10)[None])[0].reshape(2, 3)
    want = _lstsq(kind, pts, inl)
    assert np.abs(refined - want).max() <= 1e-9 * np.abs(want).max()
    # the final model is the refined one unless that has fewer inliers than the hypothesis (AF6)
    final = refined if int((ao.errors(refined.reshape(1, 6), pts)[0] < np.float32(9.0)).sum()) >= inl.sum() else A[0]
    assert np.array_equal(r["model"][:2], final.reshape(2, 3))
    assert np.abs(_lstsq(kind, pts, inl) - truth).max() < 1.0


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("seed", [5, 6])
def test_noise_free_scenes_give_the_true_transform(kind, seed):
    k0, k1, m0, truth, _ = ao.scene(kind, 400, 0.0, seed, noise=0.0, unmatched=0.0)
    r = ao.estimate_pair(kind, k0, k1, m0)
    assert r["success"] and r["num_inliers"] == 400 and r["inliers"].all()
    A = r["model"][:2]
    assert np.array_equal(r["model"][2], [0.0, 0.0, 1.0])
    assert np.abs(A - truth).max() <= 1e-6 * max(1.0, np.abs(truth).max()) * 100  # float32 keypoints
    Acv, _ = _cv(kind, k0, k1, m0)
    assert np.abs(A - Acv).max() <= 1e-6 * np.abs(Acv).max()
    if kind == ao.PARTIAL:
        assert A[0, 0] == A[1, 1] and A[0, 1] == -A[1, 0]


def measure(kind, noise, outliers, seeds=range(16)):
    """Mean-corner error (px) against the true transform, and IoU of the inlier mask with the true inliers, for the
    oracle and for cv2 on the same scenes: lists over the seeds."""
    out = {"ours_err": [], "cv_err": [], "ours_iou": [], "cv_iou": []}
    for s in seeds:
        k0, k1, m0, truth, gt = ao.scene(kind, 1024, outliers, 7000 + s, noise=noise)
        r = ao.estimate_pair(kind, k0, k1, m0)
        Acv, mcv = _cv(kind, k0, k1, m0)
        out["ours_err"].append(_corner_error(r["model"][:2], truth))
        out["cv_err"].append(_corner_error(Acv, truth))
        out["ours_iou"].append(_iou(r["inliers"], gt))
        out["cv_iou"].append(_iou(mcv, gt))
    return out


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("noise", [0.5, 1.5])
@pytest.mark.parametrize("outliers", [0.2, 0.5])
def test_synthetic_scenes_against_opencv(kind, noise, outliers):
    m = measure(kind, noise, outliers)
    # both refine on the inliers of the best minimal model, so their median corner errors are alike.  The worst case
    # is a pair whose refinement counts fewer inliers than its minimal model, which then stays (AF6; OpenCV keeps the
    # refinement): up to 1.3 px on these scenes (INTEGRATION.md).  The mask is the final model's, at least as close to
    # the true inliers as cv2's minimal-model mask.
    assert np.median(m["ours_err"]) <= 1.25 * np.median(m["cv_err"]) + 0.05, m
    assert max(m["ours_err"]) <= 1.5, m
    assert np.median(m["ours_iou"]) >= np.median(m["cv_iou"]) - 1e-3, m
    assert min(m["ours_iou"]) >= min(m["cv_iou"]), m


def _pts(x0, x1):
    return np.asarray(x0, np.float32), np.asarray(x1, np.float32)


def test_collinear_triples_are_degenerate_in_either_image():
    norm = (0.0, 0.0, 1.0, 0.0, 0.0, 1.0)
    line = [[0.0, 0.0], [1.0, 2.0], [3.0, 6.0]]
    tri = [[0.0, 0.0], [1.0, 0.0], [0.0, 1.0]]
    for a, b in ((line, tri), (tri, line), (tri, tri)):
        sp = np.concatenate(_pts(a, b), 1)[None]
        _, ok = ao.solve(ao.AFFINE, norm, sp)
        assert bool(ok[0]) == (a is tri and b is tri)


def test_coincident_partial_points_are_degenerate_in_either_image():
    norm = (0.0, 0.0, 1.0, 0.0, 0.0, 1.0)
    cases = {((0, 0), (0, 0), (1, 1), (2, 3)): False,  # coincident in image 0
             ((0, 0), (1, 1), (2, 3), (2, 3)): False,  # coincident in image 1: zero scale
             ((0, 0), (1, 1), (2, 3), (4, 3)): True}
    for (p, q, r, s), want in cases.items():
        sp = np.array([[[*p, *r], [*q, *s]]], np.float32)
        X, ok = ao.solve(ao.PARTIAL, norm, sp)
        assert bool(ok[0]) == want
    X, ok = ao.solve(ao.PARTIAL, norm, np.array([[[0, 0, 0, 0], [1, 0, 0, 2]]], np.float32))  # a 90-degree turn, x2
    assert ok[0] and np.array_equal(X[0], [0.0, 2.0, 0.0, 0.0])


@pytest.mark.parametrize("kind", KINDS)
def test_failed_pairs(kind):
    g = np.random.default_rng(0)
    k0 = g.uniform(0, 100, (10, 2)).astype(np.float32)
    k1 = k0 * np.float32(2.0)
    s = ao.sample_size(kind)
    few = np.where(np.arange(10) < s - 1, np.arange(10), -1)
    for m0, kk0 in ((few, k0), (np.arange(10), np.full_like(k0, np.nan)), (np.arange(10), np.tile(k0[:1], (10, 1))),
                    (np.zeros(0, np.int64), k0[:0])):
        r = ao.estimate_pair(kind, kk0, k1, m0)
        assert not r["success"] and r["best_hypothesis"] == -1 and r["num_inliers"] == 0
        assert not r["inliers"].any() and (r["model"] == 0).all() and r["num_hypotheses"] == 0
    # every affine sample of collinear points is degenerate: the pair draws its budget and fails
    line = np.stack([np.arange(10.0), 3.0 * np.arange(10.0)], 1).astype(np.float32)
    r = ao.estimate_pair(kind, line, line * np.float32(2.0), np.arange(10), max_iters=300)
    assert r["success"] == (kind == ao.PARTIAL) and r["num_hypotheses"] == (300 if kind == ao.AFFINE else 256)
    # n == s: no special case, the one sample is drawn like any other
    r = ao.estimate_pair(kind, k0, k1, np.where(np.arange(10) < s, np.arange(10), -1), max_iters=5, confidence=1.0)
    assert r["success"] and r["num_inliers"] == s and r["num_hypotheses"] == 5


@pytest.mark.parametrize("kind", KINDS)
def test_the_inlier_test_is_the_homography_error_on_the_bottom_row_0_0_1(kind):
    for seed in range(4):
        k0, k1, m0, _, _ = ao.scene(kind, 2000, 0.4, 300 + seed, noise=2.0)
        r = ao.estimate_pair(kind, k0, k1, m0)
        _, pts = go.compact(k0, k1, m0)
        A = r["model"].reshape(1, 9).astype(np.float32)
        x0, y0, x1, y1 = (pts[:, q] for q in range(4))
        dx = x1 - ((A[0, 0] * x0 + A[0, 1] * y0) + A[0, 2])  # AF4's affine form, as the score kernel evaluates it
        dy = y1 - ((A[0, 3] * x0 + A[0, 4] * y0) + A[0, 5])
        h = go.errors(go.HOMOGRAPHY, r["model"].reshape(1, 9), pts)[0]
        assert np.array_equal(dx * dx + dy * dy, h)
        assert int((h < np.float32(9.0)).sum()) == r["num_inliers"] == int(r["inliers"].sum())
