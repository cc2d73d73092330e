"""The relative-pose oracle (oracle/pose_oracle.py, the numpy statement of geo_relative_pose in include/geometry_b200.h)
against the ground truth of seeded calibrated scenes, and against OpenCV's five-point solver and recoverPose."""
import numpy as np
import pytest

from oracle import geometry_oracle as go
from oracle import pose_oracle as po

M = 2048


def _angle_errors(r, R, t):
    cos = (np.trace(r["R"].T @ R) - 1.0) / 2.0
    return np.degrees(np.arccos(min(1.0, cos))), np.degrees(np.arccos(min(1.0, float(r["t"] @ t))))


# Measured here (rotation error, translation-direction error, inlier recall) at seeds 1-3:
#   20 %: 0.013-0.023 deg, 0.016-0.080 deg, 0.992-0.996
#   50 %: 0.047-0.161 deg, 0.363-1.228 deg, 0.958-0.994
#   70 % (max_iters 5000): 0.057-0.075 deg, 0.351-0.514 deg, 0.987-0.993
@pytest.mark.parametrize("o,iters", [(0.2, 1000), (0.5, 1000), (0.7, 5000)])
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_recovers_the_truth(o, iters, seed):
    k0, k1, m0, truth, K0, K1, R, t = po.calibrated_two_view(M, o, seed)
    r = po.relative_pose_pair(k0, k1, m0, K0, K1, 1.0, iters, 0.999, 50.0, 0)
    assert r["success"]
    rot, tra = _angle_errors(r, R, t)
    assert rot <= 0.3 and tra <= 2.0
    assert (r["inliers"] & truth).sum() / truth.sum() >= 0.95
    assert r["num_inliers"] == r["inliers"].sum() and r["num_pose_inliers"] == r["pose_inliers"].sum()
    assert not (r["pose_inliers"] & ~r["inliers"]).any() and not r["inliers"][m0 < 0].any()
    assert abs(np.linalg.norm(r["E"]) - 1.0) < 1e-12 and abs(np.linalg.norm(r["t"]) - 1.0) < 1e-12
    assert np.abs(r["R"] @ r["R"].T - np.eye(3)).max() < 1e-12 and abs(np.linalg.det(r["R"]) - 1.0) < 1e-12


def test_different_intrinsics_per_image():
    K0 = np.array([[620.0, 0.5, 300.0], [0.0, 580.0, 250.0], [0.0, 0.0, 1.0]])
    K1 = np.array([[450.0, 0.0, 330.0], [0.0, 470.0, 230.0], [0.0, 0.0, 1.0]])
    k0, k1, m0, truth, K0, K1, R, t = po.calibrated_two_view(M, 0.3, 4, K0=K0, K1=K1)
    r = po.relative_pose_pair(k0, k1, m0, K0, K1, 1.0, 1000, 0.999, 50.0, 0)
    rot, tra = _angle_errors(r, R, t)
    assert r["success"] and rot <= 0.3 and tra <= 2.0
    assert (r["inliers"] & truth).sum() / truth.sum() >= 0.95


def test_failures():
    k0, k1, m0, *_ = po.calibrated_two_view(64, 0.0, 1, unmatched=0.0)
    K = np.array([[500.0, 0.0, 320.0], [0.0, 500.0, 240.0], [0.0, 0.0, 1.0]])
    m = np.full(64, -1)
    m[:4] = m0[:4]
    r = po.relative_pose_pair(k0, k1, m, K, K, 1.0, 1000, 0.999, 50.0, 0)
    assert not r["success"] and r["best_hypothesis"] == r["best_solution"] == -1 and r["num_hypotheses"] == 0
    bad = K.copy()
    bad[2, 2] = 0.5
    r = po.relative_pose_pair(k0, k1, m0, K, bad, 1.0, 1000, 0.999, 50.0, 0)
    assert not r["success"] and not r["inliers"].any() and not r["E"].any()
    p = np.full((64, 2), 10.0, dtype=np.float32)
    r = po.relative_pose_pair(p, p, np.arange(64), K, K, 1.0, 300, 0.999, 50.0, 0)
    assert not r["success"] and r["num_hypotheses"] == 300


def _normalise(E):
    E = E.reshape(9) / np.linalg.norm(E)
    return E * np.sign(E[np.argmax(np.abs(E))])


def _samples(n):
    rng = np.random.default_rng(0)
    out = []
    for i in range(n):
        k0, k1, m0, _, K0, K1, _, _ = po.calibrated_two_view(64, 0.0, 1000 + i, noise=0.0 if i % 2 else 0.5,
                                                           unmatched=0.0)
        _, px = go.compact(k0, k1, m0)
        pts = np.concatenate([po.calibrate(K0, px[:, :2]), po.calibrate(K1, px[:, 2:])], 1)
        out.append(pts[rng.choice(len(pts), 5, replace=False)])
    return np.stack(out)


# 600 samples, half noise-free: cv2 returns 2, 4, 6 or 8 solutions (51, 312, 235 and 2 samples) and this solver the
# same number in every sample.  Each solution agrees within 1e-6 in 586 samples (97.7 %), recorded with OpenCV 4.13.
# In the other 14 one to three solutions differ by 1.3e-6 .. 8.6e-1 (samples 52, 73, 135, 161, 191, 205, 371, 391,
# 473, 545, 549, 557, 580, 590): near-coincident roots of the degree-10 polynomial, where either solver's root is only
# as good as the polynomial's conditioning.
def test_minimal_solver_agrees_with_opencv():
    cv2 = pytest.importorskip("cv2")
    sp = _samples(600)
    E, found = po.five_point(sp)
    agree = 0
    for i in range(len(sp)):
        p = sp[i].astype(np.float64)
        Ecv, _ = cv2.findEssentialMat(p[:, :2], p[:, 2:], np.eye(3), cv2.RANSAC, 0.999, 1e-3)
        ref = [] if Ecv is None else [_normalise(Ecv[3 * j:3 * j + 3]) for j in range(Ecv.shape[0] // 3)]
        got = [E[i, j] for j in range(10) if found[i, j]]
        agree += len(ref) == len(got) and all(min(np.abs(g - r).max() for r in ref) <= 1e-6 for g in got)
    assert agree >= 0.97 * len(sp), agree


def test_pose_recovery_agrees_with_opencv():
    cv2 = pytest.importorskip("cv2")
    for seed, o in ((11, 0.2), (12, 0.5), (13, 0.3)):
        k0, k1, m0, _, K0, K1, _, _ = po.calibrated_two_view(M, o, seed)
        r = po.relative_pose_pair(k0, k1, m0, K0, K1, 1.0, 1000, 0.999, 50.0, 0)
        rows, px = go.compact(k0, k1, m0)
        pts = np.concatenate([po.calibrate(K0, px[:, :2]), po.calibrate(K1, px[:, 2:])], 1).astype(np.float64)
        mask = r["inliers"][rows].astype(np.uint8)[:, None] * 255
        n, R, t, pmask = cv2.recoverPose(r["E"], pts[:, :2], pts[:, 2:], np.eye(3), 50.0, mask=mask.copy())[:4]
        assert np.abs(R - r["R"]).max() <= 1e-6 and np.abs(t.ravel() - r["t"]).max() <= 1e-6
        assert abs(int(n) - r["num_pose_inliers"]) <= 0.005 * r["num_pose_inliers"]


def _iou(a, b):
    return (a & b).sum() / max((a | b).sum(), 1)


# Inlier-set IoU with cv2.findEssentialMat(RANSAC, 1 px, 0.999, 1000) on scene seed 5, recorded with OpenCV 4.13:
# 0.902, 0.885 and 0.654 at 0.2, 0.5 and 0.7 outliers (this side with 5000 samples at 0.7).  OpenCV keeps its minimal
# model's inliers where this side refits, and at 0.7 its 1000 samples end on a weaker model.  The bounds sit under the
# recorded values and leave room for OpenCV's own sampling.
IOU = {0.2: 0.88, 0.5: 0.86, 0.7: 0.60}


@pytest.mark.parametrize("o", [0.2, 0.5, 0.7])
def test_inliers_against_opencv(o):
    cv2 = pytest.importorskip("cv2")
    k0, k1, m0, _, K0, K1, _, _ = po.calibrated_two_view(M, o, 5)
    r = po.relative_pose_pair(k0, k1, m0, K0, K1, 1.0, 5000 if o > 0.6 else 1000, 0.999, 50.0, 0)
    v = m0 >= 0
    _, mask = cv2.findEssentialMat(k0[v].astype(np.float64), k1[m0[v]].astype(np.float64), K0, cv2.RANSAC, 0.999, 1.0,
                                   maxIters=1000)
    ref = np.zeros(M, dtype=bool)
    ref[np.nonzero(v)[0]] = mask.ravel() > 0
    assert _iou(r["inliers"], ref) >= IOU[o]
