"""The absolute-pose oracle (oracle/pnp_oracle.py, the numpy statement of geo_absolute_pose in include/geometry_b200.h)
against the ground truth of seeded localization scenes, and against OpenCV's P3P, solvePnPRefineLM and
solvePnPRansac."""
import numpy as np
import pytest

from oracle import pnp_oracle as pp

M = 2048


def _errors(r, R, t):
    cos = (np.trace(r["R"].T @ R) - 1.0) / 2.0
    return np.degrees(np.arccos(min(1.0, cos))), np.linalg.norm(r["t"] - t)


# Measured here (rotation error, translation error in scene units, inlier recall) at seeds 1-3, 8 px, confidence 0.99:
#   20 % (100 samples):  0.004-0.008 deg, 0.0004-0.0016, 1.0
#   50 % (100 samples):  0.002-0.305 deg, 0.0003-0.040, 1.0
#   70 % (1000 samples): 0.012-0.020 deg, 0.0014-0.0027, 1.0
# The 0.305 deg at 50 %, seed 1, is the minimal solution's: the refit reaches 0.014 deg with one inlier fewer (838
# against 839, an outlier within 8 px of its true projection), so the rule "the refit replaces the solution unless it has
# fewer inliers" keeps the P3P pose.
@pytest.mark.parametrize("o,iters", [(0.2, 100), (0.5, 100), (0.7, 1000)])
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_recovers_the_truth(o, iters, seed):
    k0, p3, m0, truth, K, R, t = pp.localization_scene(M, o, seed)
    r = pp.absolute_pose_pair(k0, p3, m0, K, 8.0, iters, 0.99, 0)
    assert r["success"]
    rot, tra = _errors(r, R, t)
    assert rot <= 0.4 and tra <= 0.05
    assert (r["inliers"] & truth).sum() / truth.sum() >= 0.99
    assert r["num_inliers"] == r["inliers"].sum() and not r["inliers"][m0 < 0].any()
    assert not r["inliers"][~np.isfinite(p3[np.maximum(m0, 0)]).all(1)].any()
    assert np.abs(r["R"] @ r["R"].T - np.eye(3)).max() < 1e-9 and abs(np.linalg.det(r["R"]) - 1.0) < 1e-9


# A planar scene (the points on one plane, 40 % outliers, seeds 4 and 5): 0.024 and 0.051 deg, translation error 0.0035
# and 0.0070, recall 1.0, recorded here.
@pytest.mark.parametrize("seed", [4, 5])
def test_planar_scene(seed):
    k0, p3, m0, truth, K, R, t = pp.localization_scene(M, 0.4, seed, planar=True)
    r = pp.absolute_pose_pair(k0, p3, m0, K, 8.0, 100, 0.99, 0)
    rot, tra = _errors(r, R, t)
    assert r["success"] and rot <= 0.1 and tra <= 0.02
    assert (r["inliers"] & truth).sum() / truth.sum() >= 0.99


def test_failures():
    k0, p3, m0, *_ = pp.localization_scene(64, 0.0, 1, unmatched=0.0, missing3d=0.0)
    K = np.array([[500.0, 0.0, 320.0], [0.0, 500.0, 240.0], [0.0, 0.0, 1.0]])
    m = np.full(64, -1)
    m[:2] = m0[:2]
    r = pp.absolute_pose_pair(k0, p3, m, K, 8.0, 100, 0.99, 0)
    assert not r["success"] and r["best_hypothesis"] == r["best_solution"] == -1 and r["num_hypotheses"] == 0
    bad = K.copy()
    bad[2, 2] = 0.5
    r = pp.absolute_pose_pair(k0, p3, m0, bad, 8.0, 100, 0.99, 0)
    assert not r["success"] and not r["inliers"].any() and not r["R"].any() and not r["t"].any()
    nan = p3.copy()
    nan[m0[2:]] = np.nan  # two matches keep a 3D point
    r = pp.absolute_pose_pair(k0, nan, m0, K, 8.0, 100, 0.99, 0)
    assert not r["success"] and r["num_hypotheses"] == 0
    same = np.ones((64, 3), dtype=np.float32)  # coincident world points
    r = pp.absolute_pose_pair(k0, same, m0, K, 8.0, 300, 0.99, 0)
    assert not r["success"] and r["num_hypotheses"] == 300


def _samples(n):
    rng = np.random.default_rng(0)
    out = []
    for i in range(n):
        k0, p3, m0, _, K, _, _ = pp.localization_scene(64, 0.0, 1000 + i, noise=0.0 if i % 2 else 0.5, unmatched=0.0,
                                                       missing3d=0.0)
        _, pix, wld = pp.compact(k0, p3, m0)
        sel = rng.choice(len(pix), 3, replace=False)
        out.append((pp.calibrate(K, pix[sel]), wld[sel]))
    return out


# 600 samples, half noise-free, given to cv2.solveP3P(SOLVEPNP_P3P) as the same float calibrated coordinates with K = I:
# OpenCV returns 1, 2, 3 or 4 solutions (65, 469, 7 and 59 samples) and this solver the same number in every sample,
# every solution's R and t within 1e-6 of one of OpenCV's in all 600 (100 %), recorded with OpenCV 4.13.  Given the
# pixels instead, 484 agree (80.7 %): the solver reads the calibrated coordinates rounded to float (step A2), which moves
# a solution by up to ~1e-5 px of reprojection, 1e-6 .. 6e-4 in R and t.
def test_minimal_solver_agrees_with_opencv():
    cv2 = pytest.importorskip("cv2")
    agree = 0
    for bear, wld in _samples(600):
        R, t, kept = pp.p3p(bear[None], wld[None])
        got = [(R[0, j], t[0, j]) for j in range(4) if kept[0, j]]
        _, rv, tv = cv2.solveP3P(wld.astype(np.float64), bear.astype(np.float64), np.eye(3), None,
                                 flags=cv2.SOLVEPNP_P3P)
        ref = [(cv2.Rodrigues(r)[0].reshape(9), tt.ravel()) for r, tt in zip(rv, tv)]
        agree += len(ref) == len(got) and all(
            min(max(np.abs(g[0] - r[0]).max(), np.abs(g[1] - r[1]).max()) for r in ref) <= 1e-6 for g in got)
    assert agree >= 0.99 * 600, agree


# From the same start on the same inliers, OpenCV's LM lands within 6e-13 in R and 5e-12 in t of this refit on scene
# seed 1 at 50 % outliers (recorded with OpenCV 4.13); both converge to the same minimum of the squared pixel error.
@pytest.mark.parametrize("o,seed", [(0.5, 1), (0.2, 2), (0.7, 3)])
def test_refit_agrees_with_opencv(o, seed):
    cv2 = pytest.importorskip("cv2")
    k0, p3, m0, _, K, _, _ = pp.localization_scene(M, o, seed)
    _, pix, wld = pp.compact(k0, p3, m0)
    bear = pp.calibrate(K, pix)
    r = pp.absolute_pose_pair(k0, p3, m0, K, 8.0, 1000, 0.99, 0)
    R, t, _ = pp.solutions(0, np.array([r["best_hypothesis"]]), bear, wld)
    R0, t0 = R[0, r["best_solution"]], t[0, r["best_solution"]]
    inl = pp.reproj_inliers(pp.projection(R0, t0, K)[None], pix, wld, np.float32(64.0))[0]
    Rr, tr = pp.refine_lm(R0, t0, K.reshape(9), pix, wld, inl)
    rv, _ = cv2.Rodrigues(R0.reshape(3, 3))
    rv, tv = cv2.solvePnPRefineLM(wld[inl].astype(np.float64), pix[inl].astype(np.float64), K, None, rv.copy(),
                                  t0.reshape(3, 1).copy())
    assert np.abs(cv2.Rodrigues(rv)[0].reshape(9) - Rr).max() <= 1e-9
    assert np.abs(tv.ravel() - tr).max() <= 1e-8


def _iou(a, b):
    return (a & b).sum() / max((a | b).sum(), 1)


# Inlier-set IoU with cv2.solvePnPRansac (same threshold, confidence and budget) on scene seed 5, recorded with OpenCV
# 4.13: 1.0, 1.0 and 1.0 at 0.2, 0.5 and 0.7 outliers.  Both refine on the inliers and recount them, and a 8 px band
# leaves little room for the two samplers to end on different sets; the bound leaves some.
@pytest.mark.parametrize("o", [0.2, 0.5, 0.7])
def test_inliers_against_opencv(o):
    cv2 = pytest.importorskip("cv2")
    k0, p3, m0, _, K, _, _ = pp.localization_scene(M, o, 5)
    iters = 1000 if o > 0.6 else 100
    r = pp.absolute_pose_pair(k0, p3, m0, K, 8.0, iters, 0.99, 0)
    rows, pix, wld = pp.compact(k0, p3, m0)
    _, _, _, inl = cv2.solvePnPRansac(wld.astype(np.float64), pix.astype(np.float64), K, None, iterationsCount=iters,
                                      reprojectionError=8.0, confidence=0.99)
    ref = np.zeros(M, dtype=bool)
    ref[rows[inl.ravel()]] = True
    assert _iou(r["inliers"], ref) >= 0.98
