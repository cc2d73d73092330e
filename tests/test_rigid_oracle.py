"""The 3D rigid and similarity oracle (oracle/rigid_oracle.py, header steps RG1-RG7) without a GPU: exact recovery on
noise-free scenes, RG6's closed form against OpenCV's and a numpy SVD Umeyama fit on fixed inlier sets, proper
rotations even on mirrored data, degenerate samples and failing pairs, and the accuracy table of INTEGRATION.md."""
import itertools

import numpy as np
import pytest

from oracle import rigid_oracle as ro

KINDS = [ro.RIGID, ro.SIMILARITY]


def umeyama(src, dst, with_scale):
    """Umeyama's least-squares (R, t, scale) of dst = scale R src + t, by numpy's SVD (Kabsch when not with_scale)."""
    ms, md = src.mean(0), dst.mean(0)
    a, b = src - ms, dst - md
    U, D, Vt = np.linalg.svd(b.T @ a / len(src))
    E = np.diag([1.0, 1.0, np.sign(np.linalg.det(U @ Vt))])
    R = U @ E @ Vt
    sc = np.trace(np.diag(D) @ E) / (a * a).sum(1).mean() if with_scale else 1.0
    return R, md - sc * R @ ms, sc


def _cube_rotations():
    """The 24 proper rotations that permute and negate the axes: they map float32 grid points to float32 exactly."""
    out = []
    for perm in itertools.permutations(range(3)):
        for signs in itertools.product((1.0, -1.0), repeat=3):
            R = np.zeros((3, 3))
            R[range(3), perm] = signs
            if np.linalg.det(R) > 0:
                out.append(R)
    return out


def _exact_scene(kind, R, seed, m=400, outliers=0.4):
    """Points on a 1/64 grid and a transform with a dyadic scale and translation, so points1 = scale R points0 + t
    holds exactly in float32; outliers are random grid points."""
    g = np.random.default_rng(seed)
    p0 = g.integers(-256, 256, (m, 3)) / 64.0
    sc = 1.0 if kind == ro.RIGID else [0.5, 1.5, 2.0, 0.75][seed % 4]
    t = g.integers(-64, 64, 3) / 16.0
    p1 = sc * p0 @ R.T + t
    out = g.random(m) < outliers
    p1[out] = g.integers(-256, 256, (int(out.sum()), 3)) / 64.0
    return p0.astype(np.float32), p1.astype(np.float32), np.arange(m), sc, t


@pytest.mark.parametrize("kind", KINDS)
def test_noise_free_scenes_recover_the_transform(kind):
    for i, R in enumerate(_cube_rotations()[::3]):
        p0, p1, m0, sc, t = _exact_scene(kind, R, i)
        r = ro.estimate_pair(kind, p0, p1, m0, 1e-3)
        assert r["success"], i
        assert np.abs(r["R"] - R).max() <= 1e-9 and np.abs(r["t"] - t).max() <= 1e-9, (i, r["R"], r["t"])
        assert abs(r["scale"] - sc) <= 1e-9, (i, r["scale"], sc)


@pytest.mark.parametrize("kind", KINDS)
def test_random_noise_free_scenes_recover_the_transform_to_float32_rounding(kind):
    for seed in range(4):
        p0, p1, m0, (R, t, sc), inl = ro.scene(kind, 2048, 0.5, seed, noise=0.0)
        r = ro.estimate_pair(kind, p0, p1, m0, 0.01)
        assert r["success"] and r["num_inliers"] == inl.sum() and np.array_equal(r["inliers"], inl)
        assert np.abs(r["R"] - R).max() < 1e-7 and np.abs(r["t"] - t).max() < 1e-7 and abs(r["scale"] - sc) < 1e-7


def _fixed_set(seed, n=300, mirror=False):
    g = np.random.default_rng(seed)
    src = ro.depth_points(g, n).astype(np.float32).astype(np.float64)
    R, sc, t = ro.random_rotation(g), g.uniform(0.5, 2.0), g.uniform(-1, 1, 3)
    dst = sc * src @ R.T + t + g.normal(0, 0.02, (n, 3))
    if mirror:
        dst[:, 0] = -dst[:, 0]
    return src, dst.astype(np.float32).astype(np.float64)


@pytest.mark.parametrize("seed", range(6))
def test_refit_equals_opencv_and_umeyama(seed):
    cv2 = pytest.importorskip("cv2")
    src, dst = _fixed_set(seed)
    inl = np.ones(len(src), dtype=bool)
    inl[::7] = False  # the refit sums over the inlier set only
    p, q = src.astype(np.float32), dst.astype(np.float32)
    sim = ro.refit(ro.SIMILARITY, p, q, inl)
    out, scale = cv2.estimateAffine3D(src[inl], dst[inl], force_rotation=True)
    np.testing.assert_allclose(sim[:9].reshape(3, 3), out[:, :3], rtol=0, atol=1e-9)
    np.testing.assert_allclose(sim[9:12], out[:, 3], rtol=0, atol=1e-9)
    assert abs(sim[12] - scale) <= 1e-9 * scale
    for kind, with_scale in ((ro.SIMILARITY, True), (ro.RIGID, False)):
        x = ro.refit(kind, p, q, inl)
        R, t, sc = umeyama(src[inl], dst[inl], with_scale)
        np.testing.assert_allclose(x[:9].reshape(3, 3), R, rtol=0, atol=1e-9)
        np.testing.assert_allclose(x[9:12], t, rtol=0, atol=1e-9)
        assert abs(x[12] - sc) <= 1e-9 * sc
        assert kind == ro.SIMILARITY or x[12] == 1.0


@pytest.mark.parametrize("kind", KINDS)
def test_rotations_are_proper_even_on_mirrored_data(kind):
    for seed in range(4):
        src, dst = _fixed_set(seed, mirror=True)
        x = ro.refit(kind, src.astype(np.float32), dst.astype(np.float32), np.ones(len(src), dtype=bool))
        R = x[:9].reshape(3, 3)
        assert np.abs(R @ R.T - np.eye(3)).max() < 1e-14 and abs(np.linalg.det(R) - 1.0) < 1e-14
        assert np.isfinite(x).all() and x[12] > 0
        r = ro.estimate_pair(kind, src, dst, np.arange(len(src)), 0.5)
        assert r["success"] and abs(np.linalg.det(r["R"]) - 1.0) < 1e-14


def test_rigid_scale_is_exactly_one():
    for seed in range(4):
        p0, p1, m0, _, _ = ro.scene(ro.SIMILARITY, 500, 0.3, seed, noise=0.01)
        r = ro.estimate_pair(ro.RIGID, p0, p1, m0, 0.05)
        assert r["success"] and r["scale"] == 1.0


def test_degenerate_samples_are_rejected():
    g = np.random.default_rng(3)
    good = g.normal(size=(3, 3))
    line = np.outer([0.0, 1.0, 2.5], g.normal(size=3)) + g.normal(size=3)
    coincident = np.repeat(g.normal(size=(1, 3)), 3, 0)
    two = np.concatenate([good[:2], good[1:2]])
    for bad in (line, coincident, two):
        assert ro.collinear(bad[None])[0]
    assert not ro.collinear(good[None])[0]
    # through the solver, in either set: a degenerate triangle gives no hypothesis
    for kind in KINDS:
        for p, q in ((line, good), (good, line), (coincident, good), (good, two)):
            pts0, pts1 = p.astype(np.float32), q.astype(np.float32)
            x, ok = ro.hypotheses(kind, 0, np.arange(64), pts0, pts1)
            assert not ok.any()
        x, ok = ro.hypotheses(kind, 0, np.arange(64), good.astype(np.float32), (good @ np.eye(3) + 1).astype(np.float32))
        assert ok.all()


@pytest.mark.parametrize("kind", KINDS)
def test_failures_and_nan_rows(kind):
    p0, p1, m0, _, _ = ro.scene(kind, 200, 0.2, 11, unmatched=0.0)
    two = m0.copy()
    two[2:] = -1
    r = ro.estimate_pair(kind, p0, p1, two, 0.05)
    assert not r["success"] and r["best_hypothesis"] == -1 and r["num_hypotheses"] == 0
    assert r["num_inliers"] == 0 and not r["inliers"].any() and r["scale"] == 0.0 and not r["R"].any()
    flat = p0.copy()
    flat[:] = np.outer(np.linspace(0, 1, len(p0)), [1.0, 2.0, 3.0])  # every sample collinear in set 0
    r = ro.estimate_pair(kind, flat, p1, m0, 0.05, max_iters=300)
    assert not r["success"] and r["best_hypothesis"] == -1 and r["num_hypotheses"] == 300
    nan = p0.copy()
    nan[:, 2] = np.nan
    r = ro.estimate_pair(kind, nan, p1, m0, 0.05)
    assert not r["success"] and r["num_hypotheses"] == 0
    # NaN rows are dropped: the same pair with some rows NaN in either set equals the pair without those matches
    drop = m0.copy()
    drop[::5] = -1
    holes0, holes1 = p0.copy(), p1.copy()
    holes0[::10, 0] = np.nan
    holes1[m0[5::10], 1] = np.inf
    a = ro.estimate_pair(kind, holes0, holes1, m0, 0.05)
    b = ro.estimate_pair(kind, p0, p1, drop, 0.05)
    for k in a:
        assert np.array_equal(a[k], b[k]), k
    assert not a["inliers"][::5].any()


def _rot_err_deg(R, Rt):
    return np.degrees(np.arccos(np.clip((np.trace(R.T @ Rt) - 1) / 2, -1, 1)))


def accuracy_table(kind, m=1000, scenes=30, noises=(0.005, 0.02), outliers=(0.2, 0.5, 0.7)):
    """Per (outliers, noise): median and p90 of the rotation error (degrees), the translation error relative to |t|
    and the relative scale error, for the oracle (bit for bit the GPU) and for Umeyama on the true inliers."""
    rows = []
    for o, s in itertools.product(outliers, noises):
        errs = {"ransac": [], "oracle_inliers": []}
        for seed in range(scenes):
            p0, p1, m0, (R, t, sc), inl = ro.scene(kind, m, o, 7000 + seed, noise=s)
            r = ro.estimate_pair(kind, p0, p1, m0, 3 * s)
            assert r["success"]
            v = np.flatnonzero(inl)
            Ru, tu, su = umeyama(p0[v].astype(np.float64), p1[m0[v]].astype(np.float64), kind == ro.SIMILARITY)
            for key, (Re, te, se) in (("ransac", (r["R"], r["t"], r["scale"])), ("oracle_inliers", (Ru, tu, su))):
                errs[key].append((_rot_err_deg(Re, R), np.linalg.norm(te - t) / np.linalg.norm(t), abs(se / sc - 1)))
        row = {"outliers": o, "noise": s}
        for key, e in errs.items():
            e = np.array(e)
            row[key] = np.concatenate([np.median(e, 0), np.percentile(e, 90, 0)])
        rows.append(row)
    return rows


@pytest.mark.parametrize("kind", KINDS)
def test_accuracy_table(kind):
    rows = accuracy_table(kind, scenes=12)
    for r in rows:
        print(kind, r["outliers"], r["noise"], np.array2string(r["ransac"], precision=5),
              np.array2string(r["oracle_inliers"], precision=5))
        # within a small factor of the fit on the true inliers, at every outlier fraction and noise level
        med, ref = r["ransac"][:3], r["oracle_inliers"][:3]
        assert (med <= 3.0 * ref + 1e-6).all(), (r["outliers"], r["noise"], med, ref)
        assert r["ransac"][0] < 0.5  # median rotation error below half a degree

