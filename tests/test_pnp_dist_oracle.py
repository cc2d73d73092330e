"""The distortion-aware absolute-pose oracle (oracle/pnp_dist_oracle.py, header steps AD1-AD4) against OpenCV and
against the pinhole oracles."""
import numpy as np
import pytest

from oracle import lo_pnp_oracle as lp
from oracle import pnp_dist_oracle as pd
from oracle import pnp_oracle as pp

M = 500
D = np.array([-0.3, 0.09, 1e-3, -5e-4, -0.01])


def _scene(o, seed, dist=D):
    return pd.scene(M, o, seed, dist)


@pytest.mark.parametrize("o,seed", [(0.2, 1), (0.5, 2)])
def test_refit_agrees_with_opencv(o, seed):
    cv2 = pytest.importorskip("cv2")
    k0, p3, m0, _, K, _, _ = _scene(o, seed)
    _, pix, wld = pp.compact(k0, p3, m0)
    bear = pd.bearings(K, pix, D)
    r = pd.absolute_pose_pair(k0, p3, m0, K, 8.0, 1000, 0.99, 0, D)
    R, t, _ = pp.solutions(0, np.array([r["best_hypothesis"]]), bear, wld)
    R0, t0 = R[0, r["best_solution"]], t[0, r["best_solution"]]
    inl = pd.inliers(pd.model(R0, t0)[None], pix, wld, np.float32(64.0), K, D)[0]
    Rr, tr = pd.refine_lm(R0, t0, K.reshape(9), pix, wld, inl, D)
    rv, _ = cv2.Rodrigues(R0.reshape(3, 3))
    rv, tv = cv2.solvePnPRefineLM(wld[inl].astype(np.float64), pix[inl].astype(np.float64), K, D, rv.copy(),
                                  t0.reshape(3, 1).copy())
    assert np.abs(cv2.Rodrigues(rv)[0].reshape(9) - Rr).max() <= 1e-9
    assert np.abs(tv.ravel() - tr).max() <= 1e-8


def _iou(a, b):
    return (a & b).sum() / max((a | b).sum(), 1)


# Inlier-set IoU with cv2.solvePnPRansac(..., distCoeffs) (same threshold, confidence and budget) on distorted scene
# seed 5, recorded with OpenCV 4.13: 1.0, 1.0 and 1.0 at 0.2, 0.5 and 0.7 outliers; the bound leaves some room.
@pytest.mark.parametrize("o", [0.2, 0.5, 0.7])
def test_inliers_against_opencv(o):
    cv2 = pytest.importorskip("cv2")
    k0, p3, m0, _, K, _, _ = _scene(o, 5)
    iters = 1000 if o > 0.6 else 100
    r = pd.absolute_pose_pair(k0, p3, m0, K, 8.0, iters, 0.99, 0, D)
    rows, pix, wld = pp.compact(k0, p3, m0)
    ok, _, _, idx = cv2.solvePnPRansac(wld.astype(np.float64), pix.astype(np.float64), K, D, iterationsCount=iters,
                                       reprojectionError=8.0, confidence=0.99, flags=cv2.SOLVEPNP_P3P)
    assert ok
    ref = np.zeros(len(m0), dtype=bool)
    ref[rows[idx.ravel()]] = True
    assert _iou(r["inliers"], ref) >= 0.95


@pytest.mark.parametrize("lo", [False, True], ids=["plain", "lo"])
@pytest.mark.parametrize("o,seed", [(0.2, 11), (0.5, 12)])
def test_distorted_scenes_recover_the_pose(lo, o, seed):
    k0, p3, m0, truth, K, Rt, tt = _scene(o, seed, dist=np.array([-0.3, 0.0, 0.0, 0.0]))
    d = np.array([-0.3, 0.0, 0.0, 0.0])
    with_d = (pd.lo_absolute_pose_pair if lo else pd.absolute_pose_pair)(k0, p3, m0, K, 8.0, 1000, 0.99, 0, d)
    without = (lp.lo_absolute_pose_pair if lo else pp.absolute_pose_pair)(k0, p3, m0, K, 8.0, 1000, 0.99, 0)
    assert with_d["success"]
    # 0.011 / 0.028 deg and 1e-3 / 4e-3 in t for the LO estimator; the plain one's single refit also fits the outliers
    # that fall within 8 px, 0.23 deg and 0.024 at 50 % outliers (the tail the LO estimator removes)
    assert lp.rotation_error(with_d["R"], Rt) < 0.5 and np.abs(with_d["t"] - tt).max() < 0.05
    assert (with_d["inliers"] & truth).sum() >= 0.98 * truth.sum()
    # without the coefficients t is 17 to 270 times further off (0.31 to 0.40) and 43 to 60 true inliers are lost
    err_with = np.abs(with_d["t"] - tt).max()
    assert np.abs(without["t"] - tt).max() > 5 * err_with
    assert (without["inliers"] & truth).sum() < (with_d["inliers"] & truth).sum()


@pytest.mark.parametrize("lo", [False, True], ids=["plain", "lo"])
@pytest.mark.parametrize("o,seed", [(0.2, 21), (0.5, 22), (0.7, 23)])
def test_zero_coefficients_agree_with_the_pinhole_estimator(lo, o, seed):
    # With k = 0, D2 returns A2's coordinates exactly, so both draw the same solutions, and AD3's residuals and
    # Jacobian equal A7's bit for bit.  Only the fp32 inlier test differs (x = Xc0 / w through [R | t] and then K,
    # rather than K [R | t] rounded to float), so a point within a rounding of the threshold could flip; these scenes
    # have none.
    k0, p3, m0, _, K, _, _ = pp.localization_scene(M, o, seed)
    a = (lp.lo_absolute_pose_pair if lo else pp.absolute_pose_pair)(k0, p3, m0, K, 8.0, 1000, 0.99, 0)
    b = (pd.lo_absolute_pose_pair if lo else pd.absolute_pose_pair)(k0, p3, m0, K, 8.0, 1000, 0.99, 0, np.zeros(4))
    assert np.array_equal(a["inliers"], b["inliers"])
    assert np.abs(a["R"] - b["R"]).max() <= 1e-8 and np.abs(a["t"] - b["t"]).max() <= 1e-8
