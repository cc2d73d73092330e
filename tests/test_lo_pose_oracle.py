"""The LO-RANSAC relative-pose oracle (oracle/lo_pose_oracle.py) without a GPU: its Sampson Jacobian against central
differences, its Levenberg-Marquardt against scipy's, and its accuracy against the ground truth, the plain RANSAC
oracle and OpenCV's USAC_ACCURATE."""
import math

import numpy as np
import pytest

from oracle import geometry_oracle as go
from oracle import lo_pose_oracle as lo
from oracle import pose_oracle as po


def _rot(rng, deg):
    a = rng.normal(size=3)
    a = a / np.linalg.norm(a) * math.radians(deg)
    K = np.array([[0.0, -a[2], a[1]], [a[2], 0.0, -a[0]], [-a[1], a[0], 0.0]])
    th = np.linalg.norm(a)
    return np.eye(3) + math.sin(th) / th * K + (1.0 - math.cos(th)) / th ** 2 * K @ K


def _points(seed, n, noise=0.5, outliers=0.0):
    k0, k1, m0, _, K0, K1, R, t = po.calibrated_two_view(n, outliers, seed, noise=noise, unmatched=0.0)
    _, px = go.compact(k0, k1, m0)
    pts = np.concatenate([po.calibrate(K0.reshape(9), px[:, :2]), po.calibrate(K1.reshape(9), px[:, 2:])], 1)
    return pts, K0, K1, R, t


def _angle(Ra, Rb):
    return math.acos(min(1.0, max(-1.0, (np.trace(np.asarray(Ra).reshape(3, 3).T @ np.asarray(Rb).reshape(3, 3)) - 1) / 2)))


def _pose_error(r, R, t):
    """The larger of the rotation error and the translation-direction error, in degrees."""
    ct = abs(float(np.asarray(r["t"]).ravel() @ t)) / np.linalg.norm(r["t"])
    return max(math.degrees(_angle(r["R"], R)), math.degrees(math.acos(min(1.0, ct))))


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_sampson_jacobian_equals_central_differences(seed):
    rng = np.random.default_rng(seed)
    pts, _, _, R, t = _points(50 + seed, 64)
    R0 = (_rot(rng, 3.0) @ R).reshape(9).tolist()
    t0 = t + rng.normal(0.0, 0.05, 3)
    t0 = (t0 / np.linalg.norm(t0)).tolist()
    _, _, J = lo.residuals(R0, t0, pts)
    h = 1e-6
    for k in range(5):
        d = [0.0] * 5
        d[k] = h
        rp = lo.residuals(*lo.update(R0, t0, d), pts)[0]
        d[k] = -h
        rm = lo.residuals(*lo.update(R0, t0, d), pts)[0]
        num = (rp - rm) / (2.0 * h)
        assert np.abs(J[k] - num).max() <= 1e-6 * np.abs(num).max(), (k, np.abs(J[k] - num).max())


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_final_refinement_equals_scipy_lm(seed):
    from scipy.optimize import least_squares
    rng = np.random.default_rng(seed)
    pts, K0, K1, R, t = _points(60 + seed, 512)
    # a 50 px threshold keeps every point of this outlier-free scene an inlier: one fixed set, plain least squares
    thr2 = float(po.threshold2(K0, K1, 50.0))
    R0 = (_rot(rng, 1.0) @ R).reshape(9).tolist()
    t0 = t + rng.normal(0.0, 0.02, 3)
    t0 = (t0 / np.linalg.norm(t0)).tolist()
    assert (lo.residuals(R0, t0, pts)[1] < thr2).all()
    Rg, tg = lo.refine(R0, t0, pts, thr2, lo.FINAL_STEPS)
    assert (lo.residuals(Rg, tg, pts)[1] < thr2).all()
    sol = least_squares(lambda x: lo.residuals(*lo.update(R0, t0, list(x)), pts)[0], np.zeros(5), method="lm",
                        xtol=1e-15, ftol=1e-15, gtol=1e-15)
    Rs, ts = lo.update(R0, t0, list(sol.x))
    assert _angle(Rg, Rs) <= 1e-6
    assert np.abs(np.array(tg) - np.array(ts)).max() <= 1e-6


@pytest.mark.parametrize("seed", [0, 1])
def test_refinement_never_raises_the_truncated_cost(seed):
    pts, K0, K1, R, t = _points(70 + seed, 1024, noise=1.5, outliers=0.5)
    thr2 = float(po.threshold2(K0, K1, 1.0))
    rng = np.random.default_rng(seed)
    R0, t0 = (_rot(rng, 0.5) @ R).reshape(9).tolist(), t.tolist()
    before = lo.terms(R0, t0, pts, thr2)[20]
    after = lo.terms(*lo.refine(R0, t0, pts, thr2, lo.STEPS), pts, thr2)[20]
    assert after <= before


def test_score_is_the_quantised_truncated_cost():
    thr2 = np.float32(1e-6)
    err = np.array([[0.0, 0.5e-6, 0.999999e-6, 1e-6, 2e-6, np.inf, np.nan]], dtype=np.float32)
    s, c = lo.score(err, thr2)
    w = np.float32(65536) / thr2
    want = 0 + int(np.float32(0.5e-6) * w) + int(np.float32(0.999999e-6) * w) + 4 * lo.QSCALE
    assert int(s[0]) == want and int(c[0]) == 3


# Median pose error in degrees over seeds 0..15 of calibrated_two_view(1024, outliers, seed, noise), 1 px, 1000
# samples, confidence 0.999 (cv2 4.13 with cv2.setRNGSeed(seed); recorded when this test was written):
#   noise, outliers   plain RANSAC oracle   LO oracle   cv2.findEssentialMat(USAC_ACCURATE) + recoverPose
#   0.5 px, 50 %      0.309                 0.098       0.114
#   1.5 px, 20 %      1.404                 0.432       0.381
#   1.5 px, 50 %      1.533                 0.890       0.855
CONFIGS = [(0.5, 0.5), (1.5, 0.2), (1.5, 0.5)]
SEEDS = range(16)


@pytest.fixture(scope="module")
def errors():
    out = {}
    for noise, outliers in CONFIGS:
        base, lor = [], []
        for seed in SEEDS:
            k0, k1, m0, _, K0, K1, R, t = po.calibrated_two_view(1024, outliers, seed, noise=noise)
            base.append(_pose_error(po.relative_pose_pair(k0, k1, m0, K0, K1, 1.0, 1000, 0.999, 50.0, 0), R, t))
            lor.append(_pose_error(lo.lo_relative_pose_pair(k0, k1, m0, K0, K1, 1.0, 1000, 0.999, 50.0, 0), R, t))
        out[(noise, outliers)] = (float(np.median(base)), float(np.median(lor)))
    return out


@pytest.mark.parametrize("config", CONFIGS)
def test_lo_is_more_accurate_than_plain_ransac(errors, config):
    base, lor = errors[config]
    assert lor < base, (config, base, lor)


def test_lo_accuracy_at_low_noise(errors):
    assert errors[(0.5, 0.5)][1] <= 0.15


def test_lo_is_within_half_again_of_opencv_usac_at_low_noise(errors):
    cv2 = pytest.importorskip("cv2")
    e = []
    for seed in SEEDS:
        k0, k1, m0, _, K0, _, R, t = po.calibrated_two_view(1024, 0.5, seed, noise=0.5)
        v = m0 >= 0
        a, b = k0[v].astype(np.float64), k1[m0[v]].astype(np.float64)
        cv2.setRNGSeed(seed)
        E, mask = cv2.findEssentialMat(a, b, K0, cv2.USAC_ACCURATE, 0.999, 1.0, 1000)
        _, Rc, tc, _ = cv2.recoverPose(E[:3], a, b, K0, mask=mask.copy())
        e.append(_pose_error({"R": Rc, "t": tc.ravel()}, R, t))
    assert errors[(0.5, 0.5)][1] <= 1.5 * float(np.median(e)), (errors[(0.5, 0.5)][1], float(np.median(e)))


def test_failures_are_those_of_plain_ransac():
    k0, k1, m0, *_ = po.calibrated_two_view(256, 0.0, 7, unmatched=0.0)
    m0 = m0.copy()
    m0[4:] = -1
    K = np.array([[500.0, 0.0, 320.0], [0.0, 500.0, 240.0], [0.0, 0.0, 1.0]])
    r = lo.lo_relative_pose_pair(k0, k1, m0, K, K, 1.0, 1000, 0.999, 50.0, 0)
    assert not r["success"] and r["cost"] == 0 and r["num_local_optimizations"] == 0 and r["best_hypothesis"] == -1
