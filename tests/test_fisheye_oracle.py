"""The fisheye camera model and absolute pose of oracle/fisheye_oracle.py (include/geometry_b200.h steps FE1-FE4,
AE1-AE4) against numpy, OpenCV and scipy, without a GPU: FE1's stated atan and tan against numpy's; FE3 and FE2
against cv2.fisheye under every criterion, with the clamp, the principal point and failing points; round trips; the
refit against scipy.optimize.least_squares; and the accuracy of the estimator on wide-angle localization scenes next
to cv2.fisheye.solvePnPRansac and the undistort-then-pinhole composition."""
import numpy as np
import pytest

from oracle import fisheye_oracle as fo
from oracle import make_fisheye_poly as mk
from oracle import pnp_oracle as pp

cv2 = pytest.importorskip("cv2")

K = np.array([[280.0, 0.0, 512.0], [0.0, 285.0, 500.0], [0.0, 0.0, 1.0]])
D0 = np.array([0.03, -0.012, 0.004, -0.0006])
D_FAIL = np.array([-0.3, 0.1, -0.05, 0.01])
CRITERIA = [(10, 1e-8), (10, 0.0), (3, 1e-3), (20, 1e-12), (1, 0.0), (0, 1e-8)]


def _ulp(got, ref):
    return float(np.max(np.abs(got.astype(np.float64) - ref.astype(np.float64)) / np.spacing(np.abs(ref))))


def test_header_is_reproducible():
    pytest.importorskip("mpmath")
    assert open(fo.HEADER).read() == mk.render()


def test_atan_and_tan_against_numpy():
    # measured: 2 ulp (double atan), 1 ulp (float atan), 2 ulp (double tan); numpy's own results are within 1 ulp
    rng = np.random.default_rng(0)
    r = np.concatenate([rng.uniform(0, 1, 400_000), rng.uniform(0, 10, 400_000),
                        np.exp(rng.uniform(-40, np.log(1e6), 400_000)), np.linspace(0.41, 0.42, 20_000),
                        np.linspace(2.41, 2.42, 20_000), [0.0, 1e6]])
    assert _ulp(fo.atan(r), np.arctan(r)) <= 2.0
    assert np.array_equal(fo.atan(-r), -fo.atan(r))
    rf = r.astype(np.float32)
    assert _ulp(fo.atan(rf), np.arctan(rf.astype(np.float64)).astype(np.float32)) <= 1.0
    x = np.concatenate([rng.uniform(0, np.pi / 2, 800_000), np.pi / 2 - np.exp(rng.uniform(-35, 0, 50_000))])
    x = x[x < np.pi / 2]
    assert _ulp(fo.tan(x), np.tan(x)) <= 2.0


def _pixels(n, seed):
    rng = np.random.default_rng(seed)
    px = rng.uniform(-400, 1400, (n, 2))  # beyond the 180 degree circle (clamp) on every side
    px[:3] = [[512, 500], [512 + 1e-7, 500], [512, 500 + 3e-6]]  # the principal point and a hair off it
    return px


@pytest.mark.parametrize("D", [D0, D_FAIL], ids=["mild", "failing"])
@pytest.mark.parametrize("crit", CRITERIA, ids=[f"{i}-{e:g}" for i, e in CRITERIA])
def test_undistort_matches_opencv(D, crit):
    it, eps = crit
    px = _pixels(20_000, 1)
    cv_crit = (cv2.TERM_CRITERIA_COUNT + (cv2.TERM_CRITERIA_EPS if eps > 0 else 0), it, eps)
    ref = cv2.fisheye.undistortPoints(px[:, None], K, D, P=K, criteria=cv_crit)[:, 0]
    got = fo.undistort_points(px[None], K, D, it, eps)[0]
    failed = (ref == -1e6).all(1) | np.isnan(ref).any(1)  # OpenCV's sentinel (and its 0/0) is NaN here
    assert np.array_equal(np.isnan(got).any(1), failed)
    assert np.abs(got[~failed] - ref[~failed]).max() <= 1e-9
    if D is D_FAIL and it > 0:
        assert 0 < failed.sum() < len(px)
    if eps == 0.0 and it > 0:
        assert np.isnan(got[0]).all()  # the principal point is 0 / 0 without the EPS criterion


def test_distort_matches_opencv():
    rng = np.random.default_rng(2)
    x = rng.uniform(-4, 4, (20_000, 2))
    x[0] = 0.0
    x[1] = [1e-9, 0.0]
    Ks = K.copy()
    Ks[0, 1] = 1.5
    ref = cv2.fisheye.distortPoints(x[:, None], Ks, D0, alpha=Ks[0, 1] / Ks[0, 0])[:, 0]
    pin = np.stack([Ks[0, 0] * x[:, 0] + Ks[0, 1] * x[:, 1] + Ks[0, 2], Ks[1, 1] * x[:, 1] + Ks[1, 2]], 1)
    assert np.abs(fo.distort_points(pin[None], Ks, D0)[0] - ref).max() <= 1e-9
    X = np.concatenate([x, np.ones((len(x), 1))], 1)
    proj = cv2.fisheye.projectPoints(X[:, None], np.zeros(3), np.zeros(3), K, D0)[0][:, 0]
    pin = x * np.diag(K)[:2] + K[:2, 2]
    assert np.abs(fo.distort_points(pin[None], K, D0)[0] - proj).max() <= 1e-9


def test_round_trips_away_from_the_clamp():
    rng = np.random.default_rng(3)
    th = rng.uniform(0, np.radians(80), 20_000)  # theta_d reaches pi/2, the clamp, near 86 degrees with D0
    ph = rng.uniform(0, 2 * np.pi, 20_000)
    pin = np.stack([np.tan(th) * np.cos(ph), np.tan(th) * np.sin(ph)], 1) * np.diag(K)[:2] + K[:2, 2]
    fish = fo.distort_points(pin[None], K, D0)
    back = fo.undistort_points(fish, K, D0)[0]
    assert (np.abs(back - pin).max(1) / np.abs(pin - K[:2, 2]).max(1)).max() <= 1e-12
    near = th < np.radians(70)
    assert np.abs(back[near] - pin[near]).max() <= 1e-9
    again = fo.distort_points(back[None], K, D0)[0]
    assert np.abs(again - fish[0]).max() <= 1e-9


def test_refit_lands_where_scipy_does():
    from scipy.optimize import least_squares
    from scipy.spatial.transform import Rotation
    k0, p3, m0, truth, Kc, R, t, _ = fo.scene(400, 0.0, 7, noise=1.0, unmatched=0.0, missing3d=0.0)
    idx, pix, wld = pp.compact(k0, p3, m0)
    inl = np.ones(len(pix), dtype=bool)
    R0 = Rotation.from_rotvec([0.01, -0.02, 0.015]).as_matrix() @ R
    Rr, tr = R0.reshape(9), t + 0.02
    for _ in range(3):  # A7 runs GEO_PNP_LM_STEPS steps per call; three calls converge from this start
        Rr, tr = fo.refine_lm(Rr, tr, Kc, pix, wld, inl, fo.D_SCENE)

    def res(v):
        Rm = Rotation.from_rotvec(v[:3]).as_matrix()
        Xc = wld.astype(np.float64) @ Rm.T + v[3:]
        pxs = fo.distort_points(((Xc[:, :2] / Xc[:, 2:]) * np.diag(Kc)[:2] + Kc[:2, 2])[None], Kc, fo.D_SCENE)[0]
        return (pxs - pix).ravel()
    ls = least_squares(res, np.concatenate([Rotation.from_matrix(R0).as_rotvec(), t + 0.02]), xtol=1e-15,
                       ftol=1e-15, gtol=1e-15)
    assert np.abs(Rotation.from_rotvec(ls.x[:3]).as_matrix().reshape(9) - Rr).max() <= 1e-8
    assert np.abs(ls.x[3:] - tr).max() <= 1e-8


# ---- accuracy on wide-angle localization scenes ----

BANDS = ((0, 30), (30, 60), (60, 85))


def _study(seeds=3, m=1000):
    """Per estimator and outlier share: rotation and translation errors, and true-inlier recall per field-angle band."""
    rows = {}
    for out in (0.2, 0.5, 0.7):
        for s in range(seeds):
            noise = (0.5, 1.0, 2.0)[s % 3]
            k0, p3, m0, truth, Kc, R, t, ang = fo.scene(m, out, 100 + s, noise=noise)
            idx, pix, wld = pp.compact(k0, p3, m0)
            res = {"fisheye": fo.absolute_pose_pair(k0, p3, m0, Kc, 3.0, 1000, 0.999, 0, fo.D_SCENE),
                   "fisheye_lo": fo.lo_absolute_pose_pair(k0, p3, m0, Kc, 3.0, 1000, 0.999, 0, fo.D_SCENE)}
            und = fo.undistort_points(k0[None].astype(np.float64), Kc, fo.D_SCENE)[0].astype(np.float32)
            res["undistort_then_pinhole"] = pp.absolute_pose_pair(und, p3, m0, Kc, 3.0, 1000, 0.999, 0)
            ok, rv, tv, inl = cv2.fisheye.solvePnPRansac(wld[:, None].astype(np.float64),
                                                        pix[:, None].astype(np.float64), Kc, fo.D_SCENE,
                                                        iterationsCount=1000, reprojectionError=3.0,
                                                        confidence=0.999)
            mask = np.zeros(m, dtype=bool)
            if ok and inl is not None:
                mask[idx[inl[:, 0]]] = True
            res["cv2_fisheye"] = {"R": cv2.Rodrigues(rv)[0] if ok else np.eye(3), "t": tv.reshape(3) if ok else
                                  np.zeros(3), "inliers": mask}
            for name, o in res.items():
                r = rows.setdefault((name, out), {"rot": [], "trans": [], "recall": {b: [] for b in BANDS}})
                Rm = np.asarray(o["R"]).reshape(3, 3)
                r["rot"].append(np.degrees(np.arccos(np.clip((np.trace(Rm @ R.T) - 1) / 2, -1, 1))))
                r["trans"].append(float(np.linalg.norm(np.asarray(o["t"]).reshape(3) - t)))
                for lo, hi in BANDS:
                    sel = truth & (ang >= lo) & (ang < hi)
                    r["recall"][(lo, hi)].append(float((o["inliers"] & sel).sum() / max(sel.sum(), 1)))
    return rows


@pytest.fixture(scope="module")
def study():
    return _study()


def test_accuracy_table(study):
    """3 seeds per outlier share, 1000 matches, 3 px threshold, 0.5 / 1 / 2 px noise, field angles to 85 degrees.
    Recorded true-inlier recall at 60-85 degrees for 20 / 50 / 70 % outliers: this estimator 0.89 / 0.90 / 0.83, LO
    0.90 / 0.91 / 0.88, cv2.fisheye.solvePnPRansac 0.22 / 0.21 / 0.10, the undistort-then-pinhole composition
    0.23 / 0.25 / 0.22 (at 0-30 degrees all four keep 0.75-0.90).  Median rotation error: 0.02-0.05 degrees here, 0.10-0.17
    for OpenCV.  The estimator keeps the true inliers at the edge of the lens that a pinhole-pixel threshold throws
    away; the composition behaves as OpenCV does (within 0.12 of its wide-angle recall)."""
    lines = []
    for (name, out), r in sorted(study.items()):
        rec = " ".join(f"{np.mean(v):.3f}" for v in r["recall"].values())
        lines.append(f"{name:24s} {out:.1f}  rot med {np.median(r['rot']):.4f} p90 {np.percentile(r['rot'], 90):.4f}"
                     f"  t med {np.median(r['trans']):.4f} p90 {np.percentile(r['trans'], 90):.4f}  recall {rec}")
    print("\n" + "\n".join(lines))
    for out in (0.2, 0.5, 0.7):
        wide = {n: np.mean(study[(n, out)]["recall"][(60, 85)]) for n in
                ("fisheye", "fisheye_lo", "cv2_fisheye", "undistort_then_pinhole")}
        assert wide["fisheye"] >= wide["cv2_fisheye"] + 0.1, (out, wide)
        assert wide["fisheye_lo"] >= wide["cv2_fisheye"] + 0.1, (out, wide)
        assert wide["fisheye_lo"] >= 0.8, (out, wide)
        assert abs(wide["undistort_then_pinhole"] - wide["cv2_fisheye"]) <= 0.15, (out, wide)
        for n in ("fisheye", "fisheye_lo"):
            assert np.median(study[(n, out)]["rot"]) <= 0.1, (n, out)
