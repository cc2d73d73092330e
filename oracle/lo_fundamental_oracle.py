"""numpy restatement of the LO-RANSAC fundamental matrix of include/geometry_b200.h (geo_fundamental_lo, steps LF1-LF8,
csrc/lo_hf_api.cu), and the accuracy metric its tests and tools/geometry_bench.py share.

The compaction, Hartley normalisation, samples, eight-point hypotheses, fp32 epipolar errors, denormalisation and
fixed-order sums are geometry_oracle's; the MSAC score is lo_pose_oracle's; the Cholesky step, quaternion, LM loop and
chunk driver are lo_common's.  What is new here is the Levenberg-Marquardt refinement of a rank-2 F in the
orthonormal representation (U, V, sigma) on the truncated Sampson cost in pixels (double, elementwise operations only,
so the CUDA build compiled with -fmad=false agrees bit for bit).
"""
from __future__ import annotations

import math

import numpy as np

from oracle import geometry_oracle as go
from oracle import geometry_synth as gs
from oracle import lo_common as lc
from oracle import lo_pose_oracle as lpo

S = 8                # points per sample
DOF = 7              # parameters of an LM step: rotations of U and V, and sigma
TERMS = 36           # J^T J upper triangle (28), J^T r (7), truncated cost
QSCALE, STEPS, FINAL_STEPS, LAMBDA0 = lpo.QSCALE, lpo.STEPS, lpo.FINAL_STEPS, lpo.LAMBDA0


def normalised_model(norm, F):
    """Fn = (T1^-T F) T0^-1 of a pixel F (header step LF7), as a list of 9 floats."""
    cx0, cy0, s0, cx1, cy1, s1 = norm
    r1, r0 = 1.0 / s1, 1.0 / s0
    T1it = [r1, 0.0, 0.0, 0.0, r1, 0.0, cx1, cy1, 1.0]
    T0i = [r0, 0.0, cx0, 0.0, r0, cy0, 0.0, 0.0, 1.0]
    return go._mm3(go._mm3(T1it, [float(v) for v in np.ravel(F)]), T0i)


def to_pixels(norm, X):
    """(T1^T X) T0 unscaled: a normalised model or direction in pixel coordinates."""
    cx0, cy0, s0, cx1, cy1, s1 = norm
    L = [s1, 0.0, 0.0, 0.0, s1, 0.0, -(s1 * cx1), -(s1 * cy1), 1.0]
    T0 = [s0, 0.0, -(s0 * cx0), 0.0, s0, -(s0 * cy0), 0.0, 0.0, 1.0]
    return go._mm3(go._mm3(L, list(X)), T0)


def factorise(Fn):
    """(U, V, sig) of Fn [9]: step 4's one-sided Jacobi, the first column of least squared norm dropped, u1 and v1 from
    the kept column of larger squared norm (the lower index on a tie), u3 = u1 x u2, v3 = v1 x v2."""
    A = [float(v) for v in Fn]
    W = [1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0]
    for _ in range(go.SVD_SWEEPS):
        for p, q in ((0, 1), (0, 2), (1, 2)):
            al = be = ga = 0.0
            for i in range(3):
                al = al + A[i * 3 + p] * A[i * 3 + p]
                be = be + A[i * 3 + q] * A[i * 3 + q]
                ga = ga + A[i * 3 + p] * A[i * 3 + q]
            if abs(ga) <= 1e-15 * math.sqrt(al * be):
                continue
            z = (be - al) / (2.0 * ga)
            t = (1.0 if z >= 0.0 else -1.0) / (abs(z) + math.sqrt(1.0 + z * z))
            c = 1.0 / math.sqrt(1.0 + t * t)
            s = c * t
            for M in (A, W):
                for i in range(3):
                    mp, mq = M[i * 3 + p], M[i * 3 + q]
                    M[i * 3 + p], M[i * 3 + q] = c * mp - s * mq, s * mp + c * mq
    nrm = []
    for j in range(3):
        nj = 0.0
        for i in range(3):
            nj = nj + A[i * 3 + j] * A[i * 3 + j]
        nrm.append(nj)
    m = 0
    for j in range(1, 3):
        if nrm[j] < nrm[m]:
            m = j
    p, q = [k for k in range(3) if k != m]
    if nrm[q] > nrm[p]:
        p, q = q, p
    s1, s2 = math.sqrt(nrm[p]), math.sqrt(nrm[q])
    u1 = [A[r * 3 + p] / s1 for r in range(3)]
    u2 = [A[r * 3 + q] / s2 for r in range(3)]
    v1 = [W[r * 3 + p] for r in range(3)]
    v2 = [W[r * 3 + q] for r in range(3)]
    u3, v3 = lpo._cross(u1, u2), lpo._cross(v1, v2)
    U = [x for r in range(3) for x in (u1[r], u2[r], u3[r])]
    V = [x for r in range(3) for x in (v1[r], v2[r], v3[r])]
    return U, V, s2 / s1


def compose(U, V, sig):
    """Fn_ab = u1_a*v1_b + sig*u2_a*v2_b."""
    return [U[a * 3] * V[b * 3] + sig * U[a * 3 + 1] * V[b * 3 + 1] for a in range(3) for b in range(3)]


def directions(U, V, sig):
    """dFn/d delta_k at delta = 0: [e_k]x Fn (k < 3), -Fn [e_k]x (row i is e_k x Fn[i, :]), u2 v2^T."""
    Fn = compose(U, V, sig)
    out = []
    for k in range(3):
        e = [1.0 if i == k else 0.0 for i in range(3)]
        out.append(lpo.cross_columns(e, Fn))
    for k in range(3):
        e = [1.0 if i == k else 0.0 for i in range(3)]
        out.append([c for i in range(3) for c in lpo._cross(e, Fn[i * 3:i * 3 + 3])])
    out.append([U[a * 3 + 1] * V[b * 3 + 1] for a in range(3) for b in range(3)])
    return out


def update(U, V, sig, d):
    """U' = Q(d0..2) U, V' = Q(d3..5) V, sig' = sig + d6."""
    return go._mm3(lc.quat_rotation(d[0:3]), list(U)), go._mm3(lc.quat_rotation(d[3:6]), list(V)), sig + d[6]


def _epipolar(f, x, y, u, v):
    a0, a1, a2 = (f[0] * x + f[1] * y) + f[2], (f[3] * x + f[4] * y) + f[5], (f[6] * x + f[7] * y) + f[8]
    d = (u * a0 + v * a1) + a2
    b0, b1 = (f[0] * u + f[3] * v) + f[6], (f[1] * u + f[4] * v) + f[7]
    return a0, a1, b0, b1, d


def residuals(norm, U, V, sig, pts: np.ndarray):
    """Double Sampson residuals r = d / sqrt(den) in pixels, errors d*d / den and the Jacobian [7, n] of r."""
    x, y, u, v = (pts[:, q].astype(np.float64) for q in range(4))
    a0, a1, b0, b1, d = _epipolar(to_pixels(norm, compose(U, V, sig)), x, y, u, v)
    with np.errstate(all="ignore"):
        den = ((a0 * a0 + a1 * a1) + b0 * b0) + b1 * b1
        err = (d * d) / den
        s = np.sqrt(den)
        r = d / s
        J = []
        for D in directions(U, V, sig):
            da0, da1, db0, db1, dd = _epipolar(to_pixels(norm, D), x, y, u, v)
            dden = ((a0 * da0 + a1 * da1) + b0 * db0) + b1 * db1
            J.append((dd - d * dden / den) / s)
    return r, err, np.stack(J)


def terms(norm, U, V, sig, pts: np.ndarray, thr2: float) -> np.ndarray:
    """The TERMS fixed-order sums at (U, V, sig): inliers (err < thr2) give J^T J and J^T r, every point its truncated
    cost."""
    r, err, J = residuals(norm, U, V, sig, pts)
    inl = err < thr2
    rows = []
    with np.errstate(all="ignore"):
        for i in range(DOF):
            for j in range(i, DOF):
                rows.append(np.where(inl, J[i] * J[j], 0.0))
        for i in range(DOF):
            rows.append(np.where(inl, J[i] * r, 0.0))
    rows.append(np.where(inl, err, thr2))
    return go.fixed_sum(np.stack(rows))


def refine(norm, model, pts: np.ndarray, thr2: float, steps: int):
    """steps Levenberg-Marquardt steps on the truncated Sampson cost from model = (U, V, sig), inliers re-selected at
    every model."""
    x = [float(v) for v in model[0]], [float(v) for v in model[1]], float(model[2])
    return lc.refine(lambda m: terms(norm, *m, pts, thr2), lambda m, d: update(*m, d), x, DOF, steps, LAMBDA0)


def rescore(norm, model, pts: np.ndarray, thr2: np.float32):
    """(F in pixels scaled as step 4, its LF3 score, its count)."""
    with np.errstate(all="ignore"):
        F = go.denormalise(go.FUNDAMENTAL, norm, np.array([compose(*model)]))[0]
    sc, cnt = lpo.score(go.errors(go.FUNDAMENTAL, F[None], pts)[0], thr2)
    return F, int(sc), int(cnt)


def start(norm, F):
    """(U, V, sig) of a pixel F."""
    return factorise(normalised_model(norm, F))


def lo_fundamental_pair(kpts0, kpts1, m0, threshold=3.0, max_iters=1000, confidence=0.99, seed=0) -> dict:
    return lc.lo_hf_pair(go.FUNDAMENTAL, S, "F", start, refine, rescore, kpts0, kpts1, m0, threshold, max_iters,
                         confidence, seed)


def lo_fundamental(kpts0, kpts1, matches0, threshold=3.0, max_iters=1000, confidence=0.99, seed=0) -> dict:
    """Batched: [B, M, 2], [B, N, 2], [B, M] -> the outputs of geo_fundamental_lo as numpy arrays."""
    outs = [lo_fundamental_pair(kpts0[b], kpts1[b], matches0[b], threshold, max_iters, confidence, seed)
            for b in range(len(matches0))]
    return {k: np.stack([np.asarray(o[k]) for o in outs]) for k in outs[0]}


def fundamental_error(F, F_true) -> float:
    """Zhang's virtual-correspondence error of F against F_true in pixels of the 640x480 frame: 2000 points x0 uniform
    over the frame (default_rng(12345)); for each, the point of the true line l = F_true x0 at x = 640 t with t uniform
    in [0, 1) (one draw per x0 from one default_rng(7) stream), skipped when |l_1| < 1e-12 or its y is outside
    [0, 480]; the mean of geometry_synth.epipolar_distance(F, x0, x1) over the kept points."""
    x0 = np.random.default_rng(12345).uniform([0.0, 0.0], [gs.W, gs.H], (2000, 2))
    t = np.random.default_rng(7).uniform(size=2000)
    lines = np.concatenate([x0, np.ones((2000, 1))], 1) @ np.asarray(F_true, dtype=np.float64).reshape(3, 3).T
    with np.errstate(all="ignore"):
        x = gs.W * t
        y = -(lines[:, 0] * x + lines[:, 2]) / lines[:, 1]
    keep = (np.abs(lines[:, 1]) >= 1e-12) & (y >= 0.0) & (y <= gs.H)
    x1 = np.stack([x, y], 1)
    return float(np.mean(gs.epipolar_distance(np.asarray(F, dtype=np.float64).reshape(3, 3), x0[keep], x1[keep])))
