"""The LO-RANSAC homography oracle (oracle/lo_homography_oracle.py) without a GPU: its tangent basis and transfer
Jacobian against central differences, its Levenberg-Marquardt against scipy's, its score, and its accuracy against the
ground truth, the plain RANSAC oracle and OpenCV's USAC_ACCURATE."""
import numpy as np
import pytest

from oracle import geometry_oracle as go
from oracle import geometry_synth as gs
from oracle import lo_homography_oracle as lh
from oracle import lo_pose_oracle as lpo


def _scene(seed, n, noise=0.5, outliers=0.0):
    k0, k1, m0, truth, Hm = gs.planar(n, outliers, seed, noise=noise, unmatched=0.0)
    _, pts = go.compact(k0, k1, m0)
    return pts, go.normalisation(pts), Hm


def _perturbed(rng, Hm, norm, scale=1e-3):
    Hn = np.array(lh.normalised_model(norm, Hm)) + rng.normal(0.0, scale, 9)
    return (Hn / np.linalg.norm(Hn)).tolist()


def _corner_error(H, Hm):
    return float(np.linalg.norm(gs.apply_h(H, gs.CORNERS) - gs.apply_h(Hm, gs.CORNERS), axis=1).mean())


def test_basis_is_an_orthonormal_tangent_basis():
    rng = np.random.default_rng(0)
    for _ in range(20):
        Hn = rng.normal(size=9)
        Hn = (Hn / np.linalg.norm(Hn)).tolist()
        B = np.array(lh.basis(Hn))
        assert np.abs(B @ B.T - np.eye(8)).max() <= 1e-14
        assert np.abs(B @ np.array(Hn)).max() <= 1e-14


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_transfer_jacobian_equals_central_differences(seed):
    rng = np.random.default_rng(seed)
    pts, norm, Hm = _scene(50 + seed, 64)
    Hn = _perturbed(rng, Hm, norm)
    _, _, _, jx, jy = lh.residuals(norm, Hn, pts)
    h = 1e-6
    for k in range(lh.DOF):
        d = [0.0] * lh.DOF
        d[k] = h
        xp, yp = lh.residuals(norm, lh.update(Hn, d), pts)[:2]
        d[k] = -h
        xm, ym = lh.residuals(norm, lh.update(Hn, d), pts)[:2]
        # one tolerance per direction: a direction that moves one row of H moves dx or dy alone
        num = np.concatenate([(xp - xm) / (2.0 * h), (yp - ym) / (2.0 * h)])
        j = np.concatenate([jx[k], jy[k]])
        assert np.abs(j - num).max() <= 1e-6 * np.abs(num).max(), (k, np.abs(j - num).max())


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_final_refinement_equals_scipy_lm(seed):
    from scipy.optimize import least_squares
    rng = np.random.default_rng(seed)
    pts, norm, Hm = _scene(60 + seed, 512)
    # a 50 px threshold keeps every point of this outlier-free scene an inlier: one fixed set, plain least squares
    thr2 = 2500.0
    H0 = _perturbed(rng, Hm, norm)
    assert (lh.residuals(norm, H0, pts)[2] < thr2).all()
    Hg = lh.refine(norm, H0, pts, thr2, lh.FINAL_STEPS)
    assert (lh.residuals(norm, Hg, pts)[2] < thr2).all()

    def fun(x):
        dx, dy = lh.residuals(norm, lh.update(H0, list(x)), pts)[:2]
        return np.concatenate([dx, dy])

    sol = least_squares(fun, np.zeros(lh.DOF), method="lm", xtol=1e-15, ftol=1e-15, gtol=1e-15)
    Hs = lh.update(H0, list(sol.x))
    sign = 1.0 if np.dot(Hg, Hs) >= 0.0 else -1.0
    assert np.abs(np.array(Hg) - sign * np.array(Hs)).max() <= 1e-6
    assert _corner_error(go.denormalise(go.HOMOGRAPHY, norm, np.array([Hg]))[0].reshape(3, 3),
                         go.denormalise(go.HOMOGRAPHY, norm, np.array([Hs]))[0].reshape(3, 3)) <= 1e-6


@pytest.mark.parametrize("seed", [0, 1])
def test_refinement_never_raises_the_truncated_cost(seed):
    rng = np.random.default_rng(seed)
    pts, norm, Hm = _scene(70 + seed, 1024, noise=1.5, outliers=0.5)
    thr2 = 9.0
    H0 = _perturbed(rng, Hm, norm, 3e-3)
    before = lh.terms(norm, H0, pts, thr2)[-1]
    after = lh.terms(norm, lh.refine(norm, H0, pts, thr2, lh.STEPS), pts, thr2)[-1]
    assert after <= before


def test_score_is_the_quantised_truncated_cost():
    # LH3 through the model: the score of a model is the sum of floor(err / thr2 * QSCALE) over its inliers plus QSCALE
    # per other point, a point mapped to infinity (w = 1/0) included
    pts, norm, Hm = _scene(80, 256, noise=1.5, outliers=0.3)
    pts = np.concatenate([pts, np.array([[0.0, 0.0, 1.0, 1.0]], dtype=np.float32)])
    H = Hm.reshape(9).copy()
    H[6:] = [0.0, 0.0, 0.0]  # w = 1/0 at every point: all outliers
    thr2 = np.float32(9.0)
    for model in (Hm.reshape(9), H):
        err = go.errors(go.HOMOGRAPHY, model[None], pts)[0]
        s, c = lpo.score(err, thr2)
        w = np.float32(lh.QSCALE) / thr2
        inl = err < thr2
        want = sum(int(np.float32(e) * w) for e in err[inl]) + lh.QSCALE * int((~inl).sum())
        assert int(s) == want and int(c) == int(inl.sum())
    assert int(lpo.score(go.errors(go.HOMOGRAPHY, H[None], pts)[0], thr2)[0]) == lh.QSCALE * len(pts)


# Median mean-corner error in px of the 640x480 frame over seeds 0..15 of geometry_synth.planar(1024, outliers, seed,
# noise), 3 px, 2000 samples, confidence 0.995 (cv2 4.13 with cv2.setRNGSeed(seed); recorded when this test was written):
#   noise, outliers   plain RANSAC oracle   LO oracle   cv2.findHomography(USAC_ACCURATE)
#   0.5 px, 50 %      0.122                 0.100       0.103
#   1.5 px, 20 %      0.993                 0.329       0.305
#   1.5 px, 50 %      1.413                 0.392       0.359
CONFIGS = [(0.5, 0.5), (1.5, 0.2), (1.5, 0.5)]
SEEDS = range(16)


@pytest.fixture(scope="module")
def errors():
    out = {}
    for noise, outliers in CONFIGS:
        base, lor = [], []
        for seed in SEEDS:
            k0, k1, m0, _, Hm = gs.planar(1024, outliers, seed, noise=noise)
            base.append(_corner_error(go.estimate_pair(go.HOMOGRAPHY, k0, k1, m0, 3.0, 2000, 0.995, 0)["model"], Hm))
            lor.append(_corner_error(lh.lo_homography_pair(k0, k1, m0, 3.0, 2000, 0.995, 0)["H"], Hm))
        out[(noise, outliers)] = (float(np.median(base)), float(np.median(lor)))
    return out


@pytest.mark.parametrize("config", CONFIGS)
def test_lo_is_more_accurate_than_plain_ransac(errors, config):
    base, lor = errors[config]
    assert lor < base, (config, base, lor)


def test_lo_is_within_half_again_of_opencv_usac_at_low_noise(errors):
    cv2 = pytest.importorskip("cv2")
    e = []
    for seed in SEEDS:
        k0, k1, m0, _, Hm = gs.planar(1024, 0.5, seed, noise=0.5)
        v = m0 >= 0
        cv2.setRNGSeed(seed)
        H, _ = cv2.findHomography(k0[v].astype(np.float64), k1[m0[v]].astype(np.float64), cv2.USAC_ACCURATE, 3.0,
                                  maxIters=2000, confidence=0.995)
        e.append(_corner_error(H, Hm))
    assert errors[(0.5, 0.5)][1] <= 1.5 * float(np.median(e)), (errors[(0.5, 0.5)][1], float(np.median(e)))


@pytest.mark.parametrize("case", ["few", "coincident", "collinear"])
def test_failures_are_those_of_plain_ransac(case):
    k0, k1, m0, _, _ = gs.planar(256, 0.0, 7, unmatched=0.0)
    m0 = m0.copy()
    if case == "few":
        m0[3:] = -1
    elif case == "coincident":
        k0 = np.full_like(k0, 100.0)
        k1 = k0.copy()
        m0 = np.arange(256)
    else:
        k0 = np.stack([np.linspace(0, 600, 256), np.linspace(10, 400, 256)], 1).astype(np.float32)
        k1 = k0.copy()
        m0 = np.arange(256)
    p = go.estimate_pair(go.HOMOGRAPHY, k0, k1, m0, 3.0, 512, 0.995, 0)
    r = lh.lo_homography_pair(k0, k1, m0, 3.0, 512, 0.995, 0)
    assert not p["success"] and not r["success"]
    assert r["num_hypotheses"] == p["num_hypotheses"] and r["best_hypothesis"] == -1
    assert r["cost"] == 0 and r["num_local_optimizations"] == 0 and not r["H"].any() and not r["inliers"].any()
