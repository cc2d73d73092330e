"""The LO-RANSAC absolute-pose oracle (oracle/lo_pnp_oracle.py) without a GPU: its reprojection Jacobian against
central differences, its Levenberg-Marquardt against scipy's, its score, its failures, and its rotation accuracy against
the ground truth, the plain RANSAC oracle and OpenCV's USAC."""
import numpy as np
import pytest

from oracle import lo_common as lc
from oracle import lo_pnp_oracle as la
from oracle import pnp_oracle as pp


def _scene(seed, n, noise=0.5, outliers=0.0):
    k0, p3, m0, truth, K, R, t = pp.localization_scene(n, outliers, seed, noise=noise, unmatched=0.0, missing3d=0.0)
    _, pix, wld = pp.compact(k0, p3, m0)
    return pix, wld, K.reshape(9), R, t


def _perturbed(rng, R, t, scale=1e-3):
    return la.update(R.reshape(9).tolist() + t.tolist(), rng.normal(0.0, scale, la.DOF).tolist())


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_reprojection_jacobian_equals_central_differences(seed):
    rng = np.random.default_rng(seed)
    pix, wld, K, R, t = _scene(50 + seed, 64)
    x = _perturbed(rng, R, t)
    _, _, _, z, ju, jv = la.residuals(x, K, pix, wld)
    assert (z > 0.0).all()
    h = 1e-6
    for k in range(la.DOF):
        d = [0.0] * la.DOF
        d[k] = h
        up, vp = la.residuals(la.update(x, d), K, pix, wld)[:2]
        d[k] = -h
        um, vm = la.residuals(la.update(x, d), K, pix, wld)[:2]
        for J, num in ((ju[k], (up - um) / (2.0 * h)), (jv[k], (vp - vm) / (2.0 * h))):
            assert np.abs(J - num).max() <= 1e-6 * max(np.abs(num).max(), 1.0), (k, np.abs(J - num).max())


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_final_refinement_equals_scipy_lm(seed):
    from scipy.optimize import least_squares
    rng = np.random.default_rng(seed)
    pix, wld, K, R, t = _scene(60 + seed, 512)
    # a 50 px threshold keeps every point of this outlier-free scene an inlier: one fixed set, plain least squares
    thr2 = 2500.0
    x0 = _perturbed(rng, R, t)
    assert (la.residuals(x0, K, pix, wld)[2] < thr2).all()
    xg = la.refine(x0, K, pix, wld, thr2, la.FINAL_STEPS)
    assert (la.residuals(xg, K, pix, wld)[2] < thr2).all()

    def fun(d):
        ru, rv = la.residuals(la.update(x0, list(d)), K, pix, wld)[:2]
        return np.concatenate([ru, rv])

    sol = least_squares(fun, np.zeros(la.DOF), method="lm", xtol=1e-15, ftol=1e-15, gtol=1e-15)
    xs = la.update(x0, list(sol.x))
    assert np.abs(np.array(xg[:9]) - np.array(xs[:9])).max() <= 1e-9, np.abs(np.array(xg) - np.array(xs)).max()
    assert np.abs(np.array(xg[9:]) - np.array(xs[9:])).max() <= 1e-8, np.abs(np.array(xg) - np.array(xs)).max()


@pytest.mark.parametrize("seed", [0, 1])
def test_refinement_never_raises_the_truncated_cost(seed):
    rng = np.random.default_rng(seed)
    pix, wld, K, R, t = _scene(70 + seed, 1024, noise=1.5, outliers=0.5)
    thr2 = 64.0
    for scale in (1e-3, 3e-3, 1e-2):
        x0 = _perturbed(rng, R, t, scale)
        costs = [la.terms(x0, K, pix, wld, thr2)[-1]]
        for steps in (1, 2, la.STEPS, la.FINAL_STEPS):
            costs.append(la.terms(la.refine(x0, K, pix, wld, thr2, steps), K, pix, wld, thr2)[-1])
        assert all(b <= a for a, b in zip(costs, costs[1:])), costs


def test_truncated_cost_counts_points_behind_the_camera_at_thr2():
    pix, wld, K, R, t = _scene(75, 256)
    x = R.reshape(9).tolist() + t.tolist()
    thr2 = 64.0
    base = la.terms(x, K, pix, wld, thr2)
    # the same pixels seen with the world points mirrored behind the camera: each adds thr2 and nothing to J
    behind = ((-(wld.astype(np.float64) @ R.T + t) - t) @ R).astype(np.float32)
    both = la.terms(x, K, np.concatenate([pix, pix]), np.concatenate([wld, behind]), thr2)
    assert la.residuals(x, K, pix, behind)[3].max() < 0.0
    assert both[-1] == pytest.approx(base[-1] + 256 * thr2, rel=1e-12)
    assert np.abs(both[:-1] - base[:-1]).max() <= 1e-9 * np.abs(base[:-1]).max()


def test_score_is_the_quantised_truncated_cost():
    # LA3 through the model: the score is the sum of floor(err * QSCALE / thr2) over its inliers plus QSCALE per other
    # point, a point behind the camera included whatever its pixel error
    pix, wld, K, R, t = _scene(80, 256, noise=1.5, outliers=0.3)
    thr2 = np.float32(64.0)
    behind = ((-(wld.astype(np.float64) @ R.T + t) - t) @ R).astype(np.float32)
    wld2 = np.concatenate([wld, behind[:32]])
    pix2 = np.concatenate([pix, pix[:32]])
    P = pp.projection(R.reshape(9), t, K)[None]
    err = la.errors(P, pix2, wld2)[0]
    assert np.isinf(err[256:]).all()
    s, c = la.lpo.score(err, thr2)
    w = np.float32(la.QSCALE) / thr2
    inl = pp.reproj_inliers(P, pix2, wld2, thr2)[0]
    assert np.array_equal(inl, err < thr2)
    want = sum(int(np.float32(e) * w) for e in err[inl]) + la.QSCALE * int((~inl).sum())
    assert int(s) == want and int(c) == int(inl.sum())
    assert la.rescore(R.reshape(9).tolist() + t.tolist(), K, pix2, wld2, thr2) == (want, int(inl.sum()))


@pytest.mark.parametrize("case", ["few", "nan", "collinear", "k"])
def test_failures_are_those_of_plain_ransac(case):
    k0, p3, m0, _, K, _, _ = pp.localization_scene(256, 0.0, 7, unmatched=0.0, missing3d=0.0)
    m0, p3 = m0.copy(), p3.copy()
    if case == "few":
        m0[2:] = -1
    elif case == "nan":
        p3[m0[2:], 2] = np.nan
    elif case == "collinear":
        s = np.random.default_rng(4).integers(-96, 97, 256) / 32.0
        p3 = np.stack([s, 0.5 * s, 8.0 + 0.25 * s], 1).astype(np.float32)
        q = p3.astype(np.float64) @ K.T
        k0 = (q[:, :2] / q[:, 2:]).astype(np.float32)
        m0 = np.arange(256, dtype=np.int64)
    else:
        K = K.copy()
        K[2, 2] = 2.0
    p = pp.absolute_pose_pair(k0, p3, m0, K, 8.0, 512, 0.99, 0)
    r = la.lo_absolute_pose_pair(k0, p3, m0, K, 8.0, 512, 0.99, 0)
    assert not p["success"] and not r["success"]
    for k in p:
        assert np.array_equal(np.asarray(p[k]), np.asarray(r[k])), k
    assert r["num_hypotheses"] == (512 if case == "collinear" else 0)
    assert r["cost"] == 0 and r["num_local_optimizations"] == 0


def test_outputs_are_the_final_pose_and_its_score():
    k0, p3, m0, truth, K, R, t = pp.localization_scene(1024, 0.4, 11)
    r = la.lo_absolute_pose_pair(k0, p3, m0, K)
    assert r["success"] and r["num_local_optimizations"] >= 1
    Rf = r["R"]
    assert np.abs(Rf @ Rf.T - np.eye(3)).max() <= 1e-12 and abs(np.linalg.det(Rf) - 1.0) <= 1e-12
    idx, pix, wld = pp.compact(k0, p3, m0)
    x = Rf.reshape(9).tolist() + r["t"].tolist()
    assert la.rescore(x, K.reshape(9), pix, wld, np.float32(64.0)) == (r["cost"], r["num_inliers"])
    assert r["num_inliers"] == r["inliers"].sum() and (r["inliers"] & truth).sum() >= 0.98 * truth.sum()


def test_quaternion_update_keeps_a_rotation():
    rng = np.random.default_rng(3)
    pix, wld, K, R, t = _scene(90, 16)
    x = _perturbed(rng, R, t, 0.3)
    Rn = np.array(x[:9]).reshape(3, 3)
    assert np.abs(Rn @ Rn.T - np.eye(3)).max() <= 1e-14 and abs(np.linalg.det(Rn) - 1.0) <= 1e-14
    assert lc.quat_rotation([0.0, 0.0, 0.0]) == [1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0]


# Rotation error in degrees, median / p90 / max, over seeds 0..63 of pnp_oracle.localization_scene(1024, outliers,
# seed, noise) with 10 % unmatched rows and 5 % NaN 3D points, confidence 0.99 (cv2 4.13 solvePnPRansac with
# UsacParams: MSAC, inner + iterative LO, the LSQ polisher, randomGeneratorState = seed; recorded when this test was
# written):
#   noise, outliers, threshold, budget   plain RANSAC oracle     LO oracle               cv2 USAC
#   0.5 px, 50 %, 8 px, 100              0.0125 / 0.129 / 0.476  0.0121 / 0.019 / 0.029  0.0145 / 0.024 / 0.033
#   1.5 px, 70 %, 8 px, 1000             0.0505 / 0.083 / 1.047  0.0484 / 0.073 / 0.105  0.0544 / 0.092 / 0.113
#   3.0 px, 50 %, 12 px, 1000            0.0763 / 0.141 / 0.754  0.0688 / 0.115 / 0.188  0.0842 / 0.135 / 0.200
CONFIGS = [(0.5, 0.5, 8.0, 100), (1.5, 0.7, 8.0, 1000), (3.0, 0.5, 12.0, 1000)]
SEEDS = range(64)


def _stats(e):
    return float(np.median(e)), float(np.percentile(e, 90)), float(np.max(e))


@pytest.fixture(scope="module")
def errors():
    out = {}
    for noise, outliers, thr, budget in CONFIGS:
        base, lor = [], []
        for seed in SEEDS:
            k0, p3, m0, _, K, R, _ = pp.localization_scene(1024, outliers, seed, noise=noise)
            base.append(la.rotation_error(pp.absolute_pose_pair(k0, p3, m0, K, thr, budget, 0.99, 0)["R"], R))
            lor.append(la.rotation_error(la.lo_absolute_pose_pair(k0, p3, m0, K, thr, budget, 0.99, 0)["R"], R))
        out[(noise, outliers, thr, budget)] = (_stats(base), _stats(lor))
    return out


@pytest.mark.parametrize("config", CONFIGS)
def test_lo_median_is_no_worse_than_plain_ransac(errors, config):
    base, lor = errors[config]
    assert lor[0] <= 1.1 * base[0], (config, base, lor)


@pytest.mark.parametrize("config", CONFIGS)
def test_lo_tail_is_close_to_opencv_usac(errors, config):
    cv2 = pytest.importorskip("cv2")
    noise, outliers, thr, budget = config
    e = []
    for seed in SEEDS:
        k0, p3, m0, _, K, R, _ = pp.localization_scene(1024, outliers, seed, noise=noise)
        v = m0 >= 0
        obj, img = p3[m0[v]].astype(np.float64), k0[v].astype(np.float64)
        f = np.isfinite(obj).all(1)
        p = cv2.UsacParams()
        p.confidence, p.maxIterations, p.threshold, p.randomGeneratorState = 0.99, budget, thr, seed
        p.score, p.loMethod = cv2.SCORE_METHOD_MSAC, cv2.LOCAL_OPTIM_INNER_AND_ITER_LO
        p.final_polisher = cv2.LSQ_POLISHER
        _, _, rvec, _, _ = cv2.solvePnPRansac(obj[f], img[f], K, None, params=p)
        e.append(la.rotation_error(cv2.Rodrigues(rvec)[0], R))
    usac = _stats(e)
    lor = errors[config][1]
    assert lor[1] <= 1.5 * usac[1] and lor[2] <= 2.0 * usac[2], (config, lor, usac)
