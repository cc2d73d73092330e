"""numpy restatement of the LO-RANSAC homography of include/geometry_b200.h (geo_homography_lo, steps LH1-LH8,
csrc/lo_homography_api.cu).

The compaction, Hartley normalisation, samples, four-point hypotheses, fp32 transfer errors, denormalisation and
fixed-order sums are geometry_oracle's; the MSAC score is lo_pose_oracle's.  What is new here is the Levenberg-Marquardt
refinement of the unit-norm normalised homography on the truncated transfer cost in pixels (double, elementwise
operations only, so the CUDA build compiled with -fmad=false agrees bit for bit) and its tangent basis.
"""
from __future__ import annotations

import math

import numpy as np

from oracle import geometry_oracle as go
from oracle import lo_pose_oracle as lpo

S = 4                # points per sample
DOF = 8              # parameters of an LM step: the tangent space of the unit sphere in R^9
TERMS = 45           # J^T J upper triangle (36), J^T r (8), truncated cost
QSCALE, STEPS, FINAL_STEPS, LAMBDA0 = lpo.QSCALE, lpo.STEPS, lpo.FINAL_STEPS, lpo.LAMBDA0


def normalised_model(norm, H):
    """Hn = (T1 H) T0^-1 at unit Frobenius norm (header step LH7), as a list of 9 floats."""
    cx0, cy0, s0, cx1, cy1, s1 = norm
    T1 = [s1, 0.0, -(s1 * cx1), 0.0, s1, -(s1 * cy1), 0.0, 0.0, 1.0]
    r = 1.0 / s0
    T0i = [r, 0.0, cx0, 0.0, r, cy0, 0.0, 0.0, 1.0]
    Hn = go._mm3(go._mm3(T1, [float(v) for v in np.ravel(H)]), T0i)
    f = 0.0
    for v in Hn:
        f = f + v * v
    f = math.sqrt(f)
    return [v / f for v in Hn]


def to_pixels(norm, X):
    """(T1^-1 X) T0 unscaled: a normalised model or tangent vector in pixel coordinates."""
    cx0, cy0, s0, cx1, cy1, s1 = norm
    r = 1.0 / s1
    L = [r, 0.0, cx1, 0.0, r, cy1, 0.0, 0.0, 1.0]
    T0 = [s0, 0.0, -(s0 * cx0), 0.0, s0, -(s0 * cy0), 0.0, 0.0, 1.0]
    return go._mm3(go._mm3(L, list(X)), T0)


def basis(Hn):
    """b_0..b_7: the columns j != m of the Householder reflection I - (2 / v.v) v v^T, v = e_m - Hn, with m the first
    index of least |Hn_m|.  The reflection maps e_m to Hn, so these span the tangent space of the sphere at Hn."""
    m = 0
    for i in range(1, 9):
        if abs(Hn[i]) < abs(Hn[m]):
            m = i
    v = [(1.0 if i == m else 0.0) - Hn[i] for i in range(9)]
    vv = 0.0
    for x in v:
        vv = vv + x * x
    c = 2.0 / vv
    return [[(1.0 if i == j else 0.0) - c * v[i] * v[j] for i in range(9)] for j in range(9) if j != m]


def update(Hn, d):
    """Hn' = x / |x| with x = Hn + d_0 b_0 + ... + d_7 b_7, the basis taken at Hn."""
    B = basis(Hn)
    x = []
    f = 0.0
    for i in range(9):
        v = Hn[i]
        for k in range(DOF):
            v = v + d[k] * B[k][i]
        x.append(v)
        f = f + v * v
    f = math.sqrt(f)
    return [v / f for v in x]


def residuals(norm, Hn, pts: np.ndarray):
    """Double transfer residuals (dx, dy) in pixels, errors dx*dx + dy*dy and the Jacobians [8, n] of dx and dy."""
    h = to_pixels(norm, Hn)
    x, y, u, v = (pts[:, q].astype(np.float64) for q in range(4))
    with np.errstate(all="ignore"):
        w = 1.0 / ((h[6] * x + h[7] * y) + h[8])
        px = ((h[0] * x + h[1] * y) + h[2]) * w
        py = ((h[3] * x + h[4] * y) + h[5]) * w
        dx, dy = u - px, v - py
        err = dx * dx + dy * dy
        jx, jy = [], []
        for b in basis(Hn):
            g = to_pixels(norm, b)
            da, db, dc = (g[0] * x + g[1] * y) + g[2], (g[3] * x + g[4] * y) + g[5], (g[6] * x + g[7] * y) + g[8]
            jx.append(-((da - px * dc) * w))
            jy.append(-((db - py * dc) * w))
    return dx, dy, err, np.stack(jx), np.stack(jy)


def terms(norm, Hn, pts: np.ndarray, thr2: float) -> np.ndarray:
    """The TERMS fixed-order sums at Hn: inliers (err < thr2) give J^T J and J^T r, every point its truncated cost."""
    dx, dy, err, jx, jy = residuals(norm, Hn, pts)
    inl = err < thr2
    rows = []
    with np.errstate(all="ignore"):
        for i in range(DOF):
            for j in range(i, DOF):
                rows.append(np.where(inl, jx[i] * jx[j] + jy[i] * jy[j], 0.0))
        for i in range(DOF):
            rows.append(np.where(inl, jx[i] * dx + jy[i] * dy, 0.0))
    rows.append(np.where(inl, err, thr2))
    return go.fixed_sum(np.stack(rows))


def lm_solve(h, g, lam, n=DOF):
    """lo_pose_oracle.lm_solve (header step A7) for an n x n system: delta of (H, its diagonal times (1 + lam)) delta
    = -g by Cholesky; None on failure.  n = 5 is lo_pose_oracle's, operation for operation."""
    A = [[0.0] * n for _ in range(n)]
    e = 0
    for i in range(n):
        for j in range(i, n):
            A[i][j] = A[j][i] = float(h[e])
            e += 1
    for i in range(n):
        A[i][i] = A[i][i] * (1.0 + lam)
    L = [[0.0] * n for _ in range(n)]
    for j in range(n):
        d = A[j][j]
        for k in range(j):
            d = d - L[j][k] * L[j][k]
        if not d > 0.0:
            return None
        L[j][j] = math.sqrt(d)
        for i in range(j + 1, n):
            s = A[i][j]
            for k in range(j):
                s = s - L[i][k] * L[j][k]
            L[i][j] = s / L[j][j]
    yv = [0.0] * n
    for i in range(n):
        s = -float(g[i])
        for k in range(i):
            s = s - L[i][k] * yv[k]
        yv[i] = s / L[i][i]
    x = [0.0] * n
    for i in range(n - 1, -1, -1):
        s = yv[i]
        for k in range(i + 1, n):
            s = s - L[k][i] * x[k]
        x[i] = s / L[i][i]
    return x if all(math.isfinite(v) for v in x) else None


def refine(norm, Hn, pts: np.ndarray, thr2: float, steps: int):
    """steps Levenberg-Marquardt steps on the truncated transfer cost from Hn, inliers re-selected at every model."""
    Hn = [float(v) for v in Hn]
    sums = terms(norm, Hn, pts, thr2)
    lam = LAMBDA0
    for _ in range(steps):
        d = lm_solve(sums[:36], sums[36:44], lam)
        if d is None:
            lam = lam * 10.0
            continue
        cand = update(Hn, d)
        cs = terms(norm, cand, pts, thr2)
        if cs[44] < sums[44]:
            Hn, sums = cand, cs
            lam = lam / 10.0
        else:
            lam = lam * 10.0
    return Hn


def rescore(norm, Hn, pts: np.ndarray, thr2: np.float32):
    """(H in pixels scaled as step 4, its LH3 score, its count)."""
    with np.errstate(all="ignore"):
        H = go.denormalise(go.HOMOGRAPHY, norm, np.array([Hn]))[0]
    sc, cnt = lpo.score(go.errors(go.HOMOGRAPHY, H[None], pts)[0], thr2)
    return H, int(sc), int(cnt)


def _fail(M: int, drawn: int) -> dict:
    return {"H": np.zeros((3, 3)), "inliers": np.zeros(M, dtype=bool), "num_inliers": 0, "success": False,
            "best_hypothesis": -1, "num_hypotheses": drawn, "num_local_optimizations": 0, "cost": 0}


def lo_homography_pair(kpts0, kpts1, m0, threshold=3.0, max_iters=2000, confidence=0.995, seed=0) -> dict:
    kpts0 = np.asarray(kpts0, dtype=np.float32)
    kpts1 = np.asarray(kpts1, dtype=np.float32)
    m0 = np.asarray(m0, dtype=np.int64)
    M = m0.shape[0]
    thr2 = np.float32(threshold * threshold)
    idx, pts = go.compact(kpts0, kpts1, m0)
    n = pts.shape[0]
    if n < S:
        return _fail(M, 0)
    norm = go.normalisation(pts)
    if norm is None:
        return _fail(M, 0)
    best, nlo, drawn = None, 0, 0  # best: (score, count, h, H)
    for c in range(-(-max_iters // go.CHUNK)):
        h = np.arange(c * go.CHUNK, min((c + 1) * go.CHUNK, max_iters), dtype=np.int64)
        models, ok = go.hypotheses(go.HOMOGRAPHY, seed, h, pts, norm)
        if ok.any():
            sc, cnt = lpo.score(go.errors(go.HOMOGRAPHY, models[ok], pts), thr2)
            i = int(np.argmin(sc))  # first minimum: the lowest hypothesis
            if best is None or sc[i] < best[0]:
                best = (int(sc[i]), int(cnt[i]), int(h[ok][i]), models[ok][i])
                Hl, sl, cl = rescore(norm, refine(norm, normalised_model(norm, best[3]), pts, float(thr2), STEPS), pts,
                                     thr2)
                if sl < best[0]:
                    best = (sl, cl, best[2], Hl)
                    nlo += 1
        drawn = min((c + 1) * go.CHUNK, max_iters)
        ep = 1.0 - (best[1] if best else 0) / n
        if drawn >= max_iters or drawn >= go.update_num_iters(confidence, ep, S, max_iters):
            break
    if best is None:
        return _fail(M, drawn)
    H, cost, count = rescore(norm, refine(norm, normalised_model(norm, best[3]), pts, float(thr2), FINAL_STEPS), pts,
                             thr2)
    if cost > best[0]:
        cost, count, H = best[0], best[1], best[3]
    inliers = np.zeros(M, dtype=bool)
    inliers[idx[go.errors(go.HOMOGRAPHY, H[None], pts)[0] < thr2]] = True
    return {"H": H.reshape(3, 3), "inliers": inliers, "num_inliers": count, "success": True, "best_hypothesis": best[2],
            "num_hypotheses": drawn, "num_local_optimizations": nlo, "cost": cost}


def lo_homography(kpts0, kpts1, matches0, threshold=3.0, max_iters=2000, confidence=0.995, seed=0) -> dict:
    """Batched: [B, M, 2], [B, N, 2], [B, M] -> the outputs of geo_homography_lo as numpy arrays."""
    outs = [lo_homography_pair(kpts0[b], kpts1[b], matches0[b], threshold, max_iters, confidence, seed)
            for b in range(len(matches0))]
    return {k: np.stack([np.asarray(o[k]) for o in outs]) for k in outs[0]}
