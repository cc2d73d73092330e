"""numpy restatement of the LO-RANSAC absolute pose of include/geometry_b200.h (geo_absolute_pose_lo, steps LA1-LA8,
csrc/lo_pnp_api.cu; geo_absolute_pose_lo_dist with pnp_dist_oracle's camera, steps AD1-AD4).

The compaction, camera, samples, Lambda Twist solutions, fp32 error and inlier test are pnp_oracle's; the MSAC score is
lo_pose_oracle's; the Cholesky step, quaternion rotation, LM loop and schedule are lo_common's; the normal sums and
step of (R, t) are pnp_oracle's.  What is new here is the truncated squared reprojection cost that the
Levenberg-Marquardt refinement minimises (elementwise operations only, so the CUDA build compiled with -fmad=false
agrees bit for bit).
"""
from __future__ import annotations

import numpy as np

from oracle import geometry_oracle as go
from oracle import lo_common as lc
from oracle import lo_pose_oracle as lpo
from oracle import pnp_oracle as pnp

S = pnp.S
DOF = 6              # parameters of an LM step: a rotation increment and a translation increment
TERMS = 28           # J^T J upper triangle (21), J^T r (6), truncated cost
QSCALE, STEPS, FINAL_STEPS, LAMBDA0 = lpo.QSCALE, lpo.STEPS, lpo.FINAL_STEPS, lpo.LAMBDA0
residuals, update = pnp.residuals, pnp.update  # A7's residuals, Jacobian and step, as the plain refit's
errors = pnp.errors  # A5's fp32 error, which the LA3 score reads


def terms(x, K, pix: np.ndarray, wld: np.ndarray, thr2: float, camera=None) -> np.ndarray:
    """The TERMS fixed-order sums at x through the camera (None: the pinhole K): the points in front of the camera with
    err < thr2 give J^T J and J^T r, every point its truncated cost (err for those, else thr2)."""
    ru, rv, err, z, ju, jv = (pnp.pinhole(K) if camera is None else camera).residuals(x, pix, wld)
    with np.errstate(invalid="ignore"):
        inl = (z > 0.0) & (err < thr2)
    return go.fixed_sum(np.stack(pnp.normal_sums(ru, rv, ju, jv, inl) + [np.where(inl, err, thr2)]))


def refine(x, K, pix: np.ndarray, wld: np.ndarray, thr2: float, steps: int, camera=None):
    """steps Levenberg-Marquardt steps on the truncated reprojection cost from x, inliers re-selected at every pose."""
    cam = pnp.pinhole(K) if camera is None else camera
    return lc.refine(lambda y: terms(y, K, pix, wld, thr2, cam), update, [float(v) for v in x], DOF, steps, LAMBDA0)


def rescore(x, K, pix: np.ndarray, wld: np.ndarray, thr2: np.float32, camera=None):
    """(LA3 score, count) of x through the camera's model (None: P = K [R | t]) rounded to float."""
    cam = pnp.pinhole(K) if camera is None else camera
    P = cam.model(np.array(x[:9]), np.array(x[9:]))
    sc, cnt = lpo.score(cam.errors(P[None], pix, wld)[0], thr2)
    return int(sc), int(cnt)


def _fail(M: int, drawn: int) -> dict:
    return dict(pnp._fail(M, drawn), num_local_optimizations=0, cost=0)


def lo_absolute_pose_pair(kpts0, points3d1, m0, K0, threshold=8.0, max_iters=100, confidence=0.99, seed=0,
                          camera=None) -> dict:
    """One pair of geo_absolute_pose_lo, or of geo_absolute_pose_lo_dist with camera=pnp_dist_oracle.camera(K0, dist).
    camera=None is pnp_oracle.pinhole(K0)."""
    kpts0 = np.asarray(kpts0, dtype=np.float32)
    points3d1 = np.asarray(points3d1, dtype=np.float32)
    m0 = np.asarray(m0, dtype=np.int64)
    cam = pnp.pinhole(K0) if camera is None else camera
    M = m0.shape[0]
    idx, pix, wld = pnp.compact(kpts0, points3d1, m0)
    n = pix.shape[0]
    if n < S or not cam.valid:
        return _fail(M, 0)
    bear = cam.bearings(pix)
    thr2 = np.float32(threshold * threshold)

    def candidates(h):
        R, t, kept = pnp.solutions(seed, h, bear, wld)
        if not kept.any():
            return None
        sc, cnt = lpo.score(cam.errors(cam.model(R[kept], t[kept]), pix, wld), thr2)
        hh, rr = np.nonzero(kept)
        return sc, cnt, h[hh], rr, lambda i: [float(v) for v in R[hh[i], rr[i]]] + [float(v) for v in t[hh[i], rr[i]]]

    found, nlo, drawn = lc.lo_pair(n, S, max_iters, confidence, candidates,
                                   lambda x, steps: refine(x, K0, pix, wld, float(thr2), steps, cam),
                                   lambda x: (x, *rescore(x, K0, pix, wld, thr2, cam)))
    if found is None:
        return _fail(M, drawn)
    h, r, x, cost, count = found
    P = cam.model(np.array(x[:9]), np.array(x[9:]))
    inliers = np.zeros(M, dtype=bool)
    inliers[idx[pnp.inliers(cam, P[None], pix, wld, thr2)[0]]] = True
    return {"R": np.array(x[:9]).reshape(3, 3), "t": np.array(x[9:]), "inliers": inliers, "num_inliers": count,
            "success": True, "best_hypothesis": h, "best_solution": r, "num_hypotheses": drawn,
            "num_local_optimizations": nlo, "cost": cost}


def lo_absolute_pose(kpts0, points3d1, matches0, K0, threshold=8.0, max_iters=100, confidence=0.99, seed=0) -> dict:
    """Batched: [B, M, 2], [B, N, 3], [B, M], K0 [B, 3, 3] -> the outputs of geo_absolute_pose_lo as numpy arrays."""
    outs = [lo_absolute_pose_pair(kpts0[b], points3d1[b], matches0[b], K0[b], threshold, max_iters, confidence, seed)
            for b in range(len(matches0))]
    return {k: np.stack([np.asarray(o[k]) for o in outs]) for k in outs[0]}


def rotation_error(R, Rt) -> float:
    """Angle in degrees of R Rt^T."""
    c = (np.trace(np.asarray(R).reshape(3, 3) @ np.asarray(Rt).reshape(3, 3).T) - 1.0) / 2.0
    return float(np.degrees(np.arccos(np.clip(c, -1.0, 1.0))))
