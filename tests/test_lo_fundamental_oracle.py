"""The LO-RANSAC fundamental-matrix oracle (oracle/lo_fundamental_oracle.py) without a GPU: its factorisation and
Sampson Jacobian against central differences, its Levenberg-Marquardt against scipy's, its score, its failures, and its
accuracy against the ground truth, the plain RANSAC oracle and OpenCV's USAC_ACCURATE."""
import numpy as np
import pytest

from oracle import geometry_oracle as go
from oracle import geometry_synth as gs
from oracle import lo_common as lc
from oracle import lo_fundamental_oracle as lf


def _scene(seed, n, noise=0.5, outliers=0.0):
    k0, k1, m0, truth, Ft = gs.two_view(n, outliers, seed, noise=noise, unmatched=0.0)
    _, pts = go.compact(k0, k1, m0)
    return pts, go.normalisation(pts), Ft


def _perturbed(rng, Ft, norm, scale=1e-3):
    U, V, sig = lf.factorise(lf.normalised_model(norm, Ft))
    return lf.update(U, V, sig, rng.normal(0.0, scale, lf.DOF).tolist())


def _unit(F):
    F = np.asarray(F, dtype=np.float64).reshape(9)
    F = F / np.linalg.norm(F)
    return F if F[np.argmax(np.abs(F))] >= 0.0 else -F


def _rotation(rng):
    q = rng.normal(size=4)
    q = q / np.linalg.norm(q)
    return np.array(lc.quat_rotation((q[1:] / q[0] * 2.0).tolist())).reshape(3, 3)


def test_factorise_then_compose_returns_the_model():
    rng = np.random.default_rng(0)
    for _ in range(50):
        Fn = _rotation(rng) @ np.diag([rng.uniform(0.5, 2.0), rng.uniform(0.01, 0.5), 0.0]) @ _rotation(rng).T
        U, V, sig = lf.factorise(Fn.reshape(9).tolist())
        C = np.array(lf.compose(U, V, sig))
        assert np.abs(_unit(C) - _unit(Fn)).max() <= 1e-14
        assert np.linalg.svd(C.reshape(3, 3), compute_uv=False)[2] <= 1e-14 * np.linalg.norm(C)
        assert 0.0 < sig <= 1.0
        for R in (np.array(U).reshape(3, 3), np.array(V).reshape(3, 3)):
            assert np.abs(R.T @ R - np.eye(3)).max() <= 1e-14 and abs(np.linalg.det(R) - 1.0) <= 1e-14


def test_update_keeps_rotations_and_rank_two():
    rng = np.random.default_rng(1)
    pts, norm, Ft = _scene(40, 64)
    U, V, sig = _perturbed(rng, Ft, norm, 0.1)
    for R in (np.array(U).reshape(3, 3), np.array(V).reshape(3, 3)):
        assert np.abs(R.T @ R - np.eye(3)).max() <= 1e-14 and abs(np.linalg.det(R) - 1.0) <= 1e-14
    C = np.array(lf.compose(U, V, sig)).reshape(3, 3)
    assert np.linalg.svd(C, compute_uv=False)[2] <= 1e-14 * np.linalg.norm(C)


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_sampson_jacobian_equals_central_differences(seed):
    rng = np.random.default_rng(seed)
    pts, norm, Ft = _scene(50 + seed, 64)
    model = _perturbed(rng, Ft, norm)
    J = lf.residuals(norm, *model, pts)[2]
    h = 1e-6
    for k in range(lf.DOF):
        d = [0.0] * lf.DOF
        d[k] = h
        rp = lf.residuals(norm, *lf.update(*model, d), pts)[0]
        d[k] = -h
        rm = lf.residuals(norm, *lf.update(*model, d), pts)[0]
        num = (rp - rm) / (2.0 * h)
        assert np.abs(J[k] - num).max() <= 1e-6 * np.abs(num).max(), (k, np.abs(J[k] - num).max())


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_final_refinement_equals_scipy_lm(seed):
    from scipy.optimize import least_squares
    rng = np.random.default_rng(seed)
    pts, norm, Ft = _scene(60 + seed, 512)
    # a 50 px threshold keeps every point of this outlier-free scene an inlier: one fixed set, plain least squares
    thr2 = 2500.0
    m0 = _perturbed(rng, Ft, norm)
    assert (lf.residuals(norm, *m0, pts)[1] < thr2).all()
    mg = lf.refine(norm, m0, pts, thr2, lf.FINAL_STEPS)
    assert (lf.residuals(norm, *mg, pts)[1] < thr2).all()

    def fun(x):
        return lf.residuals(norm, *lf.update(*m0, list(x)), pts)[0]

    sol = least_squares(fun, np.zeros(lf.DOF), method="lm", xtol=1e-15, ftol=1e-15, gtol=1e-15)
    Fg, Fs = _unit(lf.compose(*mg)), _unit(lf.compose(*lf.update(*m0, list(sol.x))))
    assert np.abs(Fg - Fs).max() <= 1e-6, np.abs(Fg - Fs).max()


@pytest.mark.parametrize("seed", [0, 1])
def test_refinement_never_raises_the_truncated_cost(seed):
    rng = np.random.default_rng(seed)
    pts, norm, Ft = _scene(70 + seed, 1024, noise=1.5, outliers=0.5)
    thr2 = 9.0
    m0 = _perturbed(rng, Ft, norm, 3e-3)
    before = lf.terms(norm, *m0, pts, thr2)[-1]
    after = lf.terms(norm, *lf.refine(norm, m0, pts, thr2, lf.STEPS), pts, thr2)[-1]
    assert after <= before


def test_score_is_the_quantised_truncated_cost():
    # LF3 through the model: the score of a model is the sum of floor(err / thr2 * QSCALE) over its inliers plus QSCALE
    # per other point, a point with a non-finite error (no epipolar line: a = b = 0) included
    pts, norm, Ft = _scene(80, 256, noise=1.5, outliers=0.3)
    flat = np.zeros(9)
    flat[8] = 1.0  # F x0 = (0, 0, 1) at every point: s2 = 1/0, every error non-finite
    thr2 = np.float32(9.0)
    for model in (Ft.reshape(9), flat):
        err = go.errors(go.FUNDAMENTAL, model[None], pts)[0]
        s, c = lf.lpo.score(err, thr2)
        w = np.float32(lf.QSCALE) / thr2
        inl = err < thr2
        want = sum(int(np.float32(e) * w) for e in err[inl]) + lf.QSCALE * int((~inl).sum())
        assert int(s) == want and int(c) == int(inl.sum())
    assert int(lf.lpo.score(go.errors(go.FUNDAMENTAL, flat[None], pts)[0], thr2)[0]) == lf.QSCALE * len(pts)


@pytest.mark.parametrize("case", ["few", "coincident", "collinear"])
def test_failures_are_those_of_plain_ransac(case):
    k0, k1, m0, _, _ = gs.two_view(256, 0.0, 7, unmatched=0.0)
    m0 = m0.copy()
    if case == "few":
        m0[7:] = -1
    elif case == "coincident":
        k0 = np.full_like(k0, 100.0)
        k1 = k0.copy()
        m0 = np.arange(256)
    else:  # every eight-point system on one line in both images is rank-deficient: every sample is degenerate
        k0 = np.stack([np.linspace(0, 600, 256), np.linspace(10, 400, 256)], 1).astype(np.float32)
        k1 = k0.copy()
        m0 = np.arange(256)
    p = go.estimate_pair(go.FUNDAMENTAL, k0, k1, m0, 3.0, 512, 0.99, 0)
    r = lf.lo_fundamental_pair(k0, k1, m0, 3.0, 512, 0.99, 0)
    assert not p["success"] and not r["success"]
    assert r["num_hypotheses"] == p["num_hypotheses"] and r["best_hypothesis"] == -1
    assert r["num_hypotheses"] == (512 if case == "collinear" else 0)
    assert r["cost"] == 0 and r["num_local_optimizations"] == 0 and not r["F"].any() and not r["inliers"].any()


def test_outputs_are_a_scaled_rank_two_f():
    k0, k1, m0, truth, Ft = gs.two_view(1024, 0.3, 11)
    r = lf.lo_fundamental_pair(k0, k1, m0)
    F = r["F"].reshape(9)
    assert r["success"] and r["num_local_optimizations"] >= 1
    assert abs(np.linalg.norm(F) - 1.0) <= 1e-14 and F[np.argmax(np.abs(F))] > 0.0
    assert np.linalg.svd(F.reshape(3, 3), compute_uv=False)[2] <= 1e-12
    _, pts = go.compact(k0, k1, m0)
    sc, cnt = lf.lpo.score(go.errors(go.FUNDAMENTAL, F[None], pts)[0], np.float32(9.0))
    assert r["cost"] == int(sc) and r["num_inliers"] == int(cnt) == r["inliers"].sum()


def test_fundamental_error_is_zero_at_the_truth_and_scale_free():
    _, _, _, _, Ft = gs.two_view(64, 0.0, 3)
    assert lf.fundamental_error(Ft, Ft) <= 1e-9
    assert lf.fundamental_error(-3.0 * Ft, Ft) <= 1e-9
    assert lf.fundamental_error(Ft + 1e-4 * np.eye(3), Ft) > 0.1


# Median error in px of lo_fundamental_oracle.fundamental_error over seeds 0..15 of geometry_synth.two_view(1024,
# outliers, seed, noise) with 10 % unmatched rows, 3 px, 1000 samples, confidence 0.99 (cv2 4.13 with
# cv2.setRNGSeed(seed); recorded when this test was written):
#   noise, outliers   plain RANSAC oracle   LO oracle   cv2.findFundamentalMat(USAC_ACCURATE)
#   0.5 px, 50 %      3.00                  1.12        1.47
#   1.5 px, 20 %      2.73                  0.90        0.95
#   1.5 px, 50 %      17.4                  2.47        2.23
CONFIGS = [(0.5, 0.5), (1.5, 0.2), (1.5, 0.5)]
SEEDS = range(16)


@pytest.fixture(scope="module")
def errors():
    out = {}
    for noise, outliers in CONFIGS:
        base, lor = [], []
        for seed in SEEDS:
            k0, k1, m0, _, Ft = gs.two_view(1024, outliers, seed, noise=noise)
            base.append(lf.fundamental_error(go.estimate_pair(go.FUNDAMENTAL, k0, k1, m0, 3.0, 1000, 0.99, 0)["model"],
                                             Ft))
            lor.append(lf.fundamental_error(lf.lo_fundamental_pair(k0, k1, m0, 3.0, 1000, 0.99, 0)["F"], Ft))
        out[(noise, outliers)] = (float(np.median(base)), float(np.median(lor)))
    return out


@pytest.mark.parametrize("config", CONFIGS)
def test_lo_is_more_accurate_than_plain_ransac(errors, config):
    base, lor = errors[config]
    assert lor < base, (config, base, lor)


@pytest.mark.parametrize("config", CONFIGS)
def test_lo_is_within_twice_opencv_usac(errors, config):
    cv2 = pytest.importorskip("cv2")
    noise, outliers = config
    e = []
    for seed in SEEDS:
        k0, k1, m0, _, Ft = gs.two_view(1024, outliers, seed, noise=noise)
        v = m0 >= 0
        cv2.setRNGSeed(seed)
        F, _ = cv2.findFundamentalMat(k0[v].astype(np.float64), k1[m0[v]].astype(np.float64), cv2.USAC_ACCURATE, 3.0,
                                      0.99, 1000)
        e.append(lf.fundamental_error(F[:3], Ft))
    assert errors[config][1] <= 2.0 * float(np.median(e)), (config, errors[config][1], float(np.median(e)))
