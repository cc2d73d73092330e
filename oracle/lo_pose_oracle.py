"""numpy restatement of the LO-RANSAC relative pose of include/geometry_b200.h (geo_relative_pose_lo, steps L1-L8,
csrc/pose_api.cu).

The sampling, the five-point solutions, the fp32 Sampson error and the cheirality test are pose_oracle's; the sums are
geometry_oracle's fixed order; the Cholesky step, quaternion, LM loop and once-per-chunk local optimisation schedule
are lo_common's.  What is new here is the integer MSAC score and the 5-DOF pose update and terms on the truncated
Sampson cost (double, elementwise operations only, so the CUDA build compiled with -fmad=false agrees bit for bit).
"""
from __future__ import annotations

import math

import numpy as np

from oracle import geometry_oracle as go
from oracle import lo_common as lc
from oracle import pose_oracle as po

QSCALE = 65536       # GEO_LO_QSCALE: a point's score at or past the threshold
STEPS = 8            # GEO_LO_STEPS: LM steps of a local optimisation
FINAL_STEPS = 16     # GEO_LO_FINAL_STEPS: LM steps of the final refinement
LAMBDA0 = 1e-3       # GEO_LO_LAMBDA0
TERMS = 21           # J^T J upper triangle (15), J^T r (5), truncated cost


def score(err: np.ndarray, thr2: np.float32):
    """fp32 errors [..., n] -> (uint64 MSAC scores, int64 inlier counts) over the last axis (header step L3).  An
    inlier's term is min(err * w, QSCALE) truncated, and 0 at err == 0, so a subnormal thr2 (w = inf) is defined."""
    thr2 = np.float32(thr2)
    with np.errstate(all="ignore"):
        w = np.float32(QSCALE) / thr2
        inl = err < thr2
        e = np.where(inl, err, np.float32(0.0))
        p = np.where(e == 0, np.float32(0.0), np.fmin(e * w, np.float32(QSCALE)))
        q = p.astype(np.uint32)
    q = np.where(inl, q, np.uint32(QSCALE)).astype(np.uint64)
    return q.sum(-1, dtype=np.uint64), inl.sum(-1)


def _cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def cross_columns(a, M):
    """[a]x M for a 3-vector a and a row-major 3x3 M [9]: column j is a x M[:, j]."""
    cols = [_cross(a, [M[j], M[3 + j], M[6 + j]]) for j in range(3)]
    return [cols[j][i] for i in range(3) for j in range(3)]


def essential(R, t):
    """[t]x R, row-major, not scaled."""
    return cross_columns(t, R)


def tangent_basis(t):
    """b1, b2 of t: m the first index of least |t_m|, b1 = (t x e_m) / |t x e_m|, b2 = t x b1."""
    m = 0
    for i in (1, 2):
        if abs(t[i]) < abs(t[m]):
            m = i
    c = _cross(t, [1.0 if i == m else 0.0 for i in range(3)])
    nc = math.sqrt((c[0] * c[0] + c[1] * c[1]) + c[2] * c[2])
    b1 = [c[i] / nc for i in range(3)]
    return b1, _cross(t, b1)


def derivatives(R, t):
    """dE/d delta_k at delta = 0 for the 5-DOF update (header step L3): [t]x [e_k]x R for k < 3, [b_k]x R after."""
    out = []
    for k in range(3):
        e = [1.0 if i == k else 0.0 for i in range(3)]
        out.append(cross_columns(t, cross_columns(e, R)))
    for b in tangent_basis(t):
        out.append(cross_columns(b, R))
    return out


def _epipolar(E, x, y, u, v):
    a0, a1, a2 = (E[0] * x + E[1] * y) + E[2], (E[3] * x + E[4] * y) + E[5], (E[6] * x + E[7] * y) + E[8]
    d = (u * a0 + v * a1) + a2
    b0, b1 = (E[0] * u + E[3] * v) + E[6], (E[1] * u + E[4] * v) + E[7]
    return a0, a1, b0, b1, d


def residuals(R, t, pts: np.ndarray):
    """Double Sampson residuals r = d / sqrt(den), errors d*d / den and the Jacobian [5, n] of r (header step L3)."""
    x, y, u, v = (pts[:, q].astype(np.float64) for q in range(4))
    a0, a1, b0, b1, d = _epipolar(essential(R, t), x, y, u, v)
    with np.errstate(all="ignore"):
        den = ((a0 * a0 + a1 * a1) + b0 * b0) + b1 * b1
        err = (d * d) / den
        s = np.sqrt(den)
        r = d / s
        J = []
        for dE in derivatives(R, t):
            da0, da1, db0, db1, dd = _epipolar(dE, x, y, u, v)
            dden = ((a0 * da0 + a1 * da1) + b0 * db0) + b1 * db1
            J.append((dd - d * dden / den) / s)
    return r, err, np.stack(J)


def terms(R, t, pts: np.ndarray, thr2: float) -> np.ndarray:
    """The TERMS fixed-order sums at (R, t): inliers (err < thr2) give J^T J and J^T r, every point its truncated cost."""
    r, err, J = residuals(R, t, pts)
    inl = err < thr2
    rows = []
    with np.errstate(all="ignore"):
        for i in range(5):
            for j in range(i, 5):
                rows.append(np.where(inl, J[i] * J[j], 0.0))
        for i in range(5):
            rows.append(np.where(inl, J[i] * r, 0.0))
    rows.append(np.where(inl, err, thr2))
    return go.fixed_sum(np.stack(rows))


def update(R, t, d):
    """R' = Q(d0..2) R with A7's quaternion, t' = normalize(t + d3 b1 + d4 b2)."""
    Q = lc.quat_rotation(d)
    Rn = [Q[3 * i] * R[j] + Q[3 * i + 1] * R[3 + j] + Q[3 * i + 2] * R[6 + j] for i in range(3) for j in range(3)]
    b1, b2 = tangent_basis(t)
    v = [(t[i] + d[3] * b1[i]) + d[4] * b2[i] for i in range(3)]
    nv = math.sqrt((v[0] * v[0] + v[1] * v[1]) + v[2] * v[2])
    return Rn, [v[i] / nv for i in range(3)]


def refine(R, t, pts: np.ndarray, thr2: float, steps: int):
    """steps Levenberg-Marquardt steps on the truncated Sampson cost from (R, t), inliers re-selected at every pose."""
    x = [float(v) for v in R], [float(v) for v in t]
    return lc.refine(lambda m: terms(*m, pts, thr2), lambda m, d: update(*m, d), x, 5, steps, LAMBDA0)


def model_errors(R, t, pts: np.ndarray) -> np.ndarray:
    """fp32 Sampson errors of the unit-scaled [t]x R (header step L8's E)."""
    return po.sampson(po.unit_scale(np.array(essential(R, t)))[None], pts)[0]


def choose_pose(E, pts: np.ndarray, inl: np.ndarray, distance: float):
    """P7 on the points inl: the candidate of E with most passing points (ties: the lowest)."""
    cands = po.pose_candidates(E)
    good = [int(po.cheirality(R, t, pts[inl], distance).sum()) for R, t in cands]
    k = 0
    for j in range(1, 4):
        if good[j] > good[k]:
            k = j
    return [float(v) for v in cands[k][0]], [float(v) for v in cands[k][1]]


def _fail(M: int, drawn: int) -> dict:
    out = po._fail(M, drawn)
    out.update(num_local_optimizations=0, cost=0)
    return out


def lo_relative_pose_pair(kpts0, kpts1, m0, K0, K1, threshold, max_iters, confidence, distance, seed) -> dict:
    kpts0 = np.asarray(kpts0, dtype=np.float32)
    kpts1 = np.asarray(kpts1, dtype=np.float32)
    m0 = np.asarray(m0, dtype=np.int64)
    K0 = np.asarray(K0, dtype=np.float64).reshape(9)
    K1 = np.asarray(K1, dtype=np.float64).reshape(9)
    M = m0.shape[0]
    idx, px = go.compact(kpts0, kpts1, m0)
    n = px.shape[0]
    if n < po.S or not po.k_valid(K0) or not po.k_valid(K1):
        return _fail(M, 0)
    pts = np.concatenate([po.calibrate(K0, px[:, :2]), po.calibrate(K1, px[:, 2:])], 1)
    thr2 = po.threshold2(K0, K1, threshold)

    def candidates(h):
        E, found = po.solutions(seed, h, pts)
        if not found.any():
            return None
        err = po.sampson(E[found], pts)
        sc, cnt = score(err, thr2)
        hh, rr = np.nonzero(found)
        # L4's start: P7's pose choice of the solution's E, widened from fp32, on its inliers
        return sc, cnt, h[hh], rr, lambda i: choose_pose(E[found][i].astype(np.float32).astype(np.float64), pts,
                                                         err[i] < thr2, distance)

    def rescore(x):
        sc, cnt = score(model_errors(*x, pts), thr2)
        return x, int(sc), int(cnt)

    # the output E is [t]x R, not the sampled E: a restored (R, t) is scored again
    found, nlo, drawn = lc.lo_pair(n, po.S, max_iters, confidence, candidates,
                                   lambda x, steps: refine(*x, pts, float(thr2), steps), rescore,
                                   lambda x, sc, cnt: rescore(x))
    if found is None:
        return _fail(M, drawn)
    h, r, (R, t), cost, count = found
    E = po.unit_scale(np.array(essential(R, t)))
    inl = po.sampson(E[None], pts)[0] < thr2
    good = po.cheirality(R, t, pts[inl], distance)
    inliers = np.zeros(M, dtype=bool)
    inliers[idx[inl]] = True
    pose = np.zeros(M, dtype=bool)
    pose[idx[inl][good]] = True
    return {"E": E.reshape(3, 3), "R": np.array(R).reshape(3, 3), "t": np.array(t), "inliers": inliers,
            "num_inliers": count, "pose_inliers": pose, "num_pose_inliers": int(good.sum()), "success": True,
            "best_hypothesis": h, "best_solution": r, "num_hypotheses": drawn, "num_local_optimizations": nlo,
            "cost": cost}


def lo_relative_pose(kpts0, kpts1, matches0, K0, K1, threshold=1.0, max_iters=1000, confidence=0.999, distance=50.0,
                     seed=0) -> dict:
    """Batched: [B, M, 2], [B, N, 2], [B, M], K [B, 3, 3] -> the outputs of geo_relative_pose_lo as numpy arrays."""
    outs = [lo_relative_pose_pair(kpts0[b], kpts1[b], matches0[b], K0[b], K1[b], threshold, max_iters, confidence,
                                  distance, seed) for b in range(len(matches0))]
    return {k: np.stack([np.asarray(o[k]) for o in outs]) for k in outs[0]}
