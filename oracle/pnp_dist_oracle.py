"""numpy restatement of the distortion-aware absolute pose of include/geometry_b200.h (steps AD1-AD4 on A1-A8 and
LA1-LA8; geo_absolute_pose_dist in csrc/pnp_api.cu and geo_absolute_pose_lo_dist in csrc/lo_pnp_api.cu).

The compaction, samples, Lambda Twist solver, normal sums, pose update, sampler loop and LO schedule are pnp_oracle's,
lo_pnp_oracle's, geometry_oracle's and lo_common's, unchanged; D1 and D2 are camera_oracle's.  What is new here: the
calibrated coordinates of D2 (AD1), the fp32 test in distorted pixels on [R | t] (AD2), and the double residuals and
Jacobian through D1 (AD3).  Elementwise operations only, so the CUDA build compiled with -fmad=false agrees bit for bit.

``scene`` draws pnp_oracle's localization scenes seen through a distorting lens.
"""
from __future__ import annotations

import numpy as np

from oracle import camera_oracle as co
from oracle import geometry_oracle as go
from oracle import lo_common as lc
from oracle import lo_pnp_oracle as lp
from oracle import lo_pose_oracle as lpo
from oracle import pnp_oracle as pp

S = pp.S
UNDISTORT_ITERS = 5  # AD1: cv2.solvePnP's undistortion


def scene(m: int, outliers: float, seed: int, dist, **kw):
    """pnp_oracle.localization_scene(m, outliers, seed, **kw) with every query pixel moved through the lens: K^-1,
    D1 with the coefficients dist, then K.  Returns the same tuple."""
    kpts0, pts3d, matches0, truth, K, R, t = pp.localization_scene(m, outliers, seed, **kw)
    kpts0 = co.distort_points(kpts0[None].astype(np.float64), K, dist)[0].astype(kpts0.dtype)
    return kpts0, pts3d, matches0, truth, K, R, t


def camera_valid(K, dist) -> bool:
    """A8 and AD1: K0 valid, and the coefficients all finite."""
    return pp.k_valid(K) and bool(np.isfinite(np.asarray(dist, dtype=np.float64)).all())


def bearings(K, pix: np.ndarray, dist) -> np.ndarray:
    """AD1: the fp32 calibrated coordinates P3P reads, D2's with 5 iterations and no EPS stop."""
    x, y = co.undistort_normalised(K, [np.float64(c) for c in co.pad(dist)], pix[:, 0].astype(np.float64),
                                   pix[:, 1].astype(np.float64), UNDISTORT_ITERS, 0.0)
    return np.stack([x, y], 1).astype(np.float32)


def model(R: np.ndarray, t: np.ndarray) -> np.ndarray:
    """M = [R | t] [..., 12] row-major: the model AD2 rounds to float."""
    return np.stack([R[..., 3 * i + j] if j < 3 else t[..., i] for i in range(3) for j in range(4)], -1)


def errors(M: np.ndarray, pix: np.ndarray, wld: np.ndarray, K, dist) -> np.ndarray:
    """AD2's fp32 errors [H, n] of models M [H, 12] (cast to fp32): du*du + dv*dv in distorted pixels in front of the
    camera, +inf behind it."""
    g = [M.astype(np.float32)[:, i:i + 1] for i in range(12)]
    Kf = np.asarray(K, dtype=np.float64).reshape(9).astype(np.float32)
    fx, s, cx, fy, cy = Kf[0], Kf[1], Kf[2], Kf[4], Kf[5]
    d = [np.float32(c) for c in co.pad(dist)]
    u, v = pix[None, :, 0], pix[None, :, 1]
    X, Y, Z = wld[None, :, 0], wld[None, :, 1], wld[None, :, 2]
    with np.errstate(all="ignore"):
        X0 = g[0] * X + g[1] * Y + g[2] * Z + g[3]
        X1 = g[4] * X + g[5] * Y + g[6] * Z + g[7]
        w = g[8] * X + g[9] * Y + g[10] * Z + g[11]
        xd, yd = co.distort(d, X0 / w, X1 / w)
        du = u - (fx * xd + s * yd + cx)
        dv = v - (fy * yd + cy)
        return np.where(w > 0.0, du * du + dv * dv, np.float32(np.inf))


def inliers(M: np.ndarray, pix: np.ndarray, wld: np.ndarray, thr2: np.float32, K, dist) -> np.ndarray:
    """AD2's inlier masks [H, n]: w > 0 and err < thr2."""
    with np.errstate(invalid="ignore"):
        return errors(M, pix, wld, K, dist) < thr2


def residuals(x, K, pix: np.ndarray, wld: np.ndarray, dist):
    """AD3 at x = R (9, row-major) + t (3): double residuals (ru, rv) in distorted pixels, errors ru*ru + rv*rv, depths
    Xc2 and the Jacobian rows ju, jv [6, n] (pnp_oracle.residuals' layout)."""
    R, t = x[:9], x[9:]
    K = np.asarray(K, dtype=np.float64).reshape(9)
    fx, s, cx, fy, cy = (float(K[i]) for i in (0, 1, 2, 4, 5))
    d = [np.float64(c) for c in co.pad(dist)]
    u, v = pix[:, 0].astype(np.float64), pix[:, 1].astype(np.float64)
    W = [wld[:, i].astype(np.float64) for i in range(3)]
    with np.errstate(all="ignore"):
        Xc = [R[3 * i] * W[0] + R[3 * i + 1] * W[1] + R[3 * i + 2] * W[2] + t[i] for i in range(3)]
        iz = 1.0 / Xc[2]
        a, b = Xc[0] * iz, Xc[1] * iz
        xd, yd = co.distort(d, a, b)
        ru, rv = fx * xd + s * yd + cx - u, fy * yd + cy - v
        J = co.distort_jacobian(d, a, b)
        ua, ub, va, vb = fx * J[0] + s * J[2], fx * J[1] + s * J[3], fy * J[2], fy * J[3]
        gu = [ua * iz, ub * iz, -((ua * a + ub * b) * iz)]
        gv = [va * iz, vb * iz, -((va * a + vb * b) * iz)]

        def jrow(g):
            return [g[2] * Xc[1] - g[1] * Xc[2], g[0] * Xc[2] - g[2] * Xc[0], g[1] * Xc[0] - g[0] * Xc[1],
                    g[0], g[1], g[2]]
        ju, jv = np.stack(jrow(gu)), np.stack(jrow(gv))
        err = ru * ru + rv * rv
    return ru, rv, err, Xc[2], ju, jv


def refine_lm(R, t, K, pix, wld, inl, dist):
    """A7's GEO_PNP_LM_STEPS Levenberg-Marquardt steps on AD3's squared error of the fixed inliers inl, from (R, t)."""
    def terms(x):
        ru, rv, err, _, ju, jv = residuals(x, K, pix, wld, dist)
        return go.fixed_sum(np.stack(pp.normal_sums(ru, rv, ju, jv, inl) + [np.where(inl, err, 0.0)]))

    x = lc.refine(terms, pp.update, [float(c) for c in R] + [float(c) for c in t], 6, pp.LM_STEPS, pp.LM_LAMBDA0)
    return np.array(x[:9]), np.array(x[9:])


def _prepare(kpts0, points3d1, m0, K0, dist):
    kpts0 = np.asarray(kpts0, dtype=np.float32)
    points3d1 = np.asarray(points3d1, dtype=np.float32)
    m0 = np.asarray(m0, dtype=np.int64)
    K0 = np.asarray(K0, dtype=np.float64).reshape(9)
    idx, pix, wld = pp.compact(kpts0, points3d1, m0)
    return m0.shape[0], K0, idx, pix, wld


def absolute_pose_pair(kpts0, points3d1, m0, K0, threshold, max_iters, confidence, seed, dist) -> dict:
    """One pair of geo_absolute_pose_dist: pnp_oracle.absolute_pose_pair with AD1-AD4."""
    M, K0, idx, pix, wld = _prepare(kpts0, points3d1, m0, K0, dist)
    n = pix.shape[0]
    if n < S or not camera_valid(K0, dist):
        return pp._fail(M, 0)
    bear = bearings(K0, pix, dist)
    thr2 = np.float32(threshold * threshold)

    def inl(R, t):
        return inliers(model(R, t), pix, wld, thr2, K0, dist)

    def candidates(h):
        R, t, kept = pp.solutions(seed, h, bear, wld)
        if not kept.any():
            return None
        hh, rr = np.nonzero(kept)
        return inl(R[kept], t[kept]).sum(1), h[hh], rr

    best_cnt, best_h, best_r, drawn = go.ransac_pair(n, S, max_iters, confidence, candidates)
    if best_h < 0:
        return pp._fail(M, drawn)
    R, t, _ = pp.solutions(seed, np.array([best_h]), bear, wld)
    R0, t0 = R[0, best_r], t[0, best_r]
    cands = [(R0, t0, best_cnt)]
    if best_cnt >= pp.REFIT_MIN:
        Rr, tr = refine_lm(R0, t0, K0, pix, wld, inl(R0[None], t0[None])[0], dist)
        cands.append((Rr, tr, int(inl(Rr[None], tr[None])[0].sum())))
    Rf, tf, count = cands[1] if len(cands) == 2 and cands[1][2] >= cands[0][2] else cands[0]
    mask = np.zeros(M, dtype=bool)
    mask[idx[inl(np.asarray(Rf)[None], np.asarray(tf)[None])[0]]] = True
    return {"R": np.asarray(Rf).reshape(3, 3), "t": np.asarray(tf), "inliers": mask, "num_inliers": count,
            "success": True, "best_hypothesis": best_h, "best_solution": best_r, "num_hypotheses": drawn}


def lo_terms(x, K, pix: np.ndarray, wld: np.ndarray, thr2: float, dist) -> np.ndarray:
    """LA7's TERMS fixed-order sums at x on AD3's residuals: the points in front of the camera with err < thr2 give
    J^T J and J^T r, every point its truncated cost."""
    ru, rv, err, z, ju, jv = residuals(x, K, pix, wld, dist)
    with np.errstate(invalid="ignore"):
        inl = (z > 0.0) & (err < thr2)
    return go.fixed_sum(np.stack(pp.normal_sums(ru, rv, ju, jv, inl) + [np.where(inl, err, thr2)]))


def lo_absolute_pose_pair(kpts0, points3d1, m0, K0, threshold, max_iters, confidence, seed, dist) -> dict:
    """One pair of geo_absolute_pose_lo_dist: lo_pnp_oracle.lo_absolute_pose_pair with AD1-AD4."""
    M, K0, idx, pix, wld = _prepare(kpts0, points3d1, m0, K0, dist)
    n = pix.shape[0]
    if n < S or not camera_valid(K0, dist):
        return lp._fail(M, 0)
    bear = bearings(K0, pix, dist)
    thr2 = np.float32(threshold * threshold)

    def refine(x, steps):
        return lc.refine(lambda y: lo_terms(y, K0, pix, wld, float(thr2), dist), pp.update, [float(v) for v in x],
                         lp.DOF, steps, lp.LAMBDA0)

    def rescore(x):
        sc, cnt = lpo.score(errors(model(np.array(x[:9]), np.array(x[9:]))[None], pix, wld, K0, dist)[0], thr2)
        return x, int(sc), int(cnt)

    def candidates(h):
        R, t, kept = pp.solutions(seed, h, bear, wld)
        if not kept.any():
            return None
        sc, cnt = lpo.score(errors(model(R[kept], t[kept]), pix, wld, K0, dist), thr2)
        hh, rr = np.nonzero(kept)
        return sc, cnt, h[hh], rr, lambda i: [float(v) for v in R[hh[i], rr[i]]] + [float(v) for v in t[hh[i], rr[i]]]

    found, nlo, drawn = lc.lo_pair(n, S, max_iters, confidence, candidates, refine, rescore)
    if found is None:
        return lp._fail(M, drawn)
    h, r, x, cost, count = found
    mask = np.zeros(M, dtype=bool)
    mask[idx[inliers(model(np.array(x[:9]), np.array(x[9:]))[None], pix, wld, thr2, K0, dist)[0]]] = True
    return {"R": np.array(x[:9]).reshape(3, 3), "t": np.array(x[9:]), "inliers": mask, "num_inliers": count,
            "success": True, "best_hypothesis": h, "best_solution": r, "num_hypotheses": drawn,
            "num_local_optimizations": nlo, "cost": cost}


def _batched(pair, kpts0, points3d1, matches0, K0, dist, threshold, max_iters, confidence, seed) -> dict:
    outs = [pair(kpts0[b], points3d1[b], matches0[b], K0[b], threshold, max_iters, confidence, seed, dist[b])
            for b in range(len(matches0))]
    return {k: np.stack([np.asarray(o[k]) for o in outs]) for k in outs[0]}


def absolute_pose(kpts0, points3d1, matches0, K0, dist, threshold=8.0, max_iters=100, confidence=0.99, seed=0) -> dict:
    """Batched: [B, M, 2], [B, N, 3], [B, M], K0 [B, 3, 3], dist [B, k] -> geo_absolute_pose_dist's outputs."""
    return _batched(absolute_pose_pair, kpts0, points3d1, matches0, K0, dist, threshold, max_iters, confidence, seed)


def lo_absolute_pose(kpts0, points3d1, matches0, K0, dist, threshold=8.0, max_iters=100, confidence=0.99,
                     seed=0) -> dict:
    """Batched: as absolute_pose -> geo_absolute_pose_lo_dist's outputs."""
    return _batched(lo_absolute_pose_pair, kpts0, points3d1, matches0, K0, dist, threshold, max_iters, confidence,
                    seed)
