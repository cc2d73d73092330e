"""oracle/camera_oracle.py (header steps D1-D3) against OpenCV: cv2.undistortPoints, cv2.undistortPointsIter and
cv2.projectPoints at 4, 5, 8 and 12 coefficients, the icdist < 0 branch, NaN pass-through, and convergence with
max_iters."""
import numpy as np
import pytest

from oracle import camera_oracle as co

cv2 = pytest.importorskip("cv2")

K = np.array([[500.0, 0.0, 320.0], [0.0, 480.0, 240.0], [0.0, 0.0, 1.0]])
DIST = {4: [-0.3, 0.09, 1e-3, -5e-4], 5: [-0.28, 0.07, 8e-4, -6e-4, -0.01],
        8: [-0.25, 0.05, 5e-4, -3e-4, 0.002, 0.02, 0.004, 0.001],
        12: [-0.25, 0.06, 6e-4, -4e-4, 0.003, 0.01, 0.002, 0.0005, 1e-3, -2e-4, -8e-4, 3e-4]}


def _pixels(n=2000, seed=0):
    rng = np.random.default_rng(seed)
    return np.stack([rng.uniform(0, 640, n), rng.uniform(0, 480, n)], 1)


@pytest.mark.parametrize("nd", [4, 5, 8, 12])
def test_undistort_matches_opencv(nd):
    d = np.array(DIST[nd])
    px = _pixels()
    ref = cv2.undistortPoints(px[:, None], K, d, P=K)[:, 0]
    got = co.undistort_points(px[None], K, d)[0]
    assert np.abs(got - ref).max() <= 1e-9


@pytest.mark.parametrize("nd", [4, 5, 8, 12])
@pytest.mark.parametrize("crit", ["count", "count+eps"])
def test_undistort_iter_matches_opencv(nd, crit):
    d = np.array(DIST[nd])
    px = _pixels(seed=1)
    if crit == "count":
        c, eps = (cv2.TERM_CRITERIA_COUNT, 40, 0.0), 0.0
    else:
        c, eps = (cv2.TERM_CRITERIA_COUNT | cv2.TERM_CRITERIA_EPS, 40, 1e-3), 1e-3
    ref = cv2.undistortPointsIter(px[:, None], K, d, None, K, c)[:, 0]
    got = co.undistort_points(px[None], K, d, max_iters=40, eps=eps)[0]
    assert np.abs(got - ref).max() <= 1e-9


@pytest.mark.parametrize("nd", [4, 5, 8, 12])
def test_distort_matches_project_points(nd):
    d = np.array(DIST[nd])
    px = _pixels(seed=2)
    xn = np.stack([(px[:, 0] - K[0, 2]) / K[0, 0], (px[:, 1] - K[1, 2]) / K[1, 1], np.ones(len(px))], 1)
    ref = cv2.projectPoints(xn, np.zeros(3), np.zeros(3), K, d)[0][:, 0]
    got = co.distort_points(px[None], K, d)[0]
    assert np.abs(got - ref).max() <= 1e-9


def test_negative_icdist_returns_the_pinhole_estimate():
    # k1 = -2: at the image corners 1 + k1*r2 < 0, so OpenCV returns the undistorted pinhole estimate there
    d = np.array([-2.0, 0.0, 0.0, 0.0])
    px = np.array([[0.0, 0.0], [639.0, 479.0], [320.0, 240.0]])
    ref = cv2.undistortPoints(px[:, None], K, d, P=K)[:, 0]
    got = co.undistort_points(px[None], K, d)[0]
    assert np.abs(got - ref).max() <= 1e-9
    assert np.abs(got[:2] - px[:2]).max() <= 1e-9  # the pinhole estimate, mapped back through K, is the input


def test_nan_pass_through():
    d = np.array(DIST[5])
    px = _pixels(10)
    px[3, 0] = np.nan
    px[5, 1] = np.inf
    for f in (lambda p: co.undistort_points(p, K, d), lambda p: co.distort_points(p, K, d)):
        got = f(px[None])[0]
        assert np.isnan(got[[3, 5]]).all() and np.isfinite(np.delete(got, [3, 5], 0)).all()
    bad = d.copy()
    bad[2] = np.nan
    assert np.isnan(co.undistort_points(px[None], K, bad)).all()
    Kb = K.copy()
    Kb[2, 2] = 2.0
    assert np.isnan(co.distort_points(px[None], Kb, d)).all()


def test_round_trip_error_falls_with_max_iters():
    # f = 500, 640x480, k1 = -0.3: the image of a grid of undistorted points over the frame, undistorted again.
    # OpenCV's default 5 iterations leave errors of about a pixel at the corners.
    Kc = np.array([[500.0, 0.0, 320.0], [0.0, 500.0, 240.0], [0.0, 0.0, 1.0]])
    d = np.array([-0.3, 0.0, 0.0, 0.0])
    g = np.stack(np.meshgrid(np.linspace(0, 639, 33), np.linspace(0, 479, 25)), -1).reshape(-1, 2)
    seen = co.distort_points(g[None], Kc, d)
    errs = [np.abs(co.undistort_points(seen, Kc, d, max_iters=it)[0] - g).max() for it in (1, 2, 5, 20, 100)]
    assert all(a > b for a, b in zip(errs, errs[1:])), errs
    assert 0.1 < errs[2] < 5.0 and errs[-1] < 1e-6, errs
