"""numpy restatement of the affine and partial affine RANSAC of include/geometry_b200.h (steps AF1-AF7,
lightglue_b200/csrc/affine_api.cu).

Compaction, normalisation, sampling, the fixed-order sums, the stopping rule and the fp32 error are geometry_oracle's
(the error is its homography error on [A; 0 0 1]); the Levenberg-Marquardt loop is lo_common's.  What is new here is
the two minimal solvers, the denormalisation and the refinement's terms.  float64 for the solvers and the refinement,
float32 for the scoring, one operation at a time, so the CUDA build compiled with -fmad=false agrees bit for bit.
"""
from __future__ import annotations

import numpy as np

from oracle import geometry_oracle as go
from oracle import lo_common as lc
from oracle import lo_pose_oracle as lpo

AFFINE, PARTIAL = 3, 4
MAX_REFINE = 100


def sample_size(kind: int) -> int:
    return 3 if kind == AFFINE else 2


def dof(kind: int) -> int:
    return 6 if kind == AFFINE else 4


def _normalised(norm, p):
    cx0, cy0, s0, cx1, cy1, s1 = norm
    return ((p[..., 0].astype(np.float64) - cx0) * s0, (p[..., 1].astype(np.float64) - cy0) * s0,
            (p[..., 2].astype(np.float64) - cx1) * s1, (p[..., 3].astype(np.float64) - cy1) * s1)


def _collinear(dxj, dyj, dxk, dyk, D):
    return np.abs(D) <= go.FLT_EPS * (((np.abs(dxj) + np.abs(dyj)) + np.abs(dxk)) + np.abs(dyk))


def solve(kind: int, norm, sp: np.ndarray):
    """Samples sp [H, s, 4] -> normalised parameters [H, dof] and the mask of non-degenerate samples (AF3), before the
    finiteness test."""
    x, y, u, v = _normalised(norm, sp)
    with np.errstate(all="ignore"):
        if kind == PARTIAL:
            dx, dy, du, dv = x[:, 1] - x[:, 0], y[:, 1] - y[:, 0], u[:, 1] - u[:, 0], v[:, 1] - v[:, 0]
            dd = dx * dx + dy * dy
            ok = (dd > 0.0) & ~((du == 0.0) & (dv == 0.0))
            a = (dx * du + dy * dv) / dd
            b = (dx * dv - dy * du) / dd
            return np.stack([a, b, u[:, 0] - (a * x[:, 0] - b * y[:, 0]), v[:, 0] - (b * x[:, 0] + a * y[:, 0])], 1), ok
        dxj, dyj, dxk, dyk = x[:, 1] - x[:, 0], y[:, 1] - y[:, 0], x[:, 2] - x[:, 0], y[:, 2] - y[:, 0]
        duj, dvj, duk, dvk = u[:, 1] - u[:, 0], v[:, 1] - v[:, 0], u[:, 2] - u[:, 0], v[:, 2] - v[:, 0]
        D = dxj * dyk - dxk * dyj
        ok = ~_collinear(dxj, dyj, dxk, dyk, D) & ~_collinear(duj, dvj, duk, dvk, duj * dvk - duk * dvj)
        a = (duj * dyk - duk * dyj) / D
        b = (dxj * duk - dxk * duj) / D
        d = (dvj * dyk - dvk * dyj) / D
        e = (dxj * dvk - dxk * dvj) / D
        c, f = u[:, 0] - (a * x[:, 0] + b * y[:, 0]), v[:, 0] - (d * x[:, 0] + e * y[:, 0])
        return np.stack([a, b, c, d, e, f], 1), ok


def pixels(kind: int, norm, X: np.ndarray) -> np.ndarray:
    """Normalised parameters [H, dof] -> pixel models [H, 6] (a00, a01, a02, a10, a11, a12), AF3's denormalisation."""
    cx0, cy0, s0, cx1, cy1, s1 = (np.float64(c) for c in norm)
    r = 1.0 / s1
    with np.errstate(all="ignore"):
        if kind == PARTIAL:
            kx, ky = s0 * cx0, s0 * cy0
            a, b = (X[:, 0] * s0) * r, (X[:, 1] * s0) * r
            tx = (X[:, 2] - (X[:, 0] * kx - X[:, 1] * ky)) * r + cx1
            ty = (X[:, 3] - (X[:, 1] * kx + X[:, 0] * ky)) * r + cy1
            return np.stack([a, -b, tx, b, a, ty], 1)
        T0 = [s0, 0.0, -(s0 * cx0), 0.0, s0, -(s0 * cy0), 0.0, 0.0, 1.0]
        L = [r, 0.0, cx1, 0.0, r, cy1, 0.0, 0.0, 1.0]
        T0, L = [np.float64(c) for c in T0], [np.float64(c) for c in L]
        zero = np.zeros(X.shape[0])
        An = [X[:, 0], X[:, 1], X[:, 2], X[:, 3], X[:, 4], X[:, 5], zero, zero, zero + 1.0]
        return np.stack(go._mm3(go._mm3(L, An), T0)[:6], 1)


def hypotheses(kind: int, seed: int, h: np.ndarray, pts: np.ndarray, norm):
    """Normalised parameters [H, dof], pixel models [H, 6] and the mask of non-degenerate hypotheses h of one pair."""
    ids, ok = go.samples(seed, h, pts.shape[0], sample_size(kind))
    X, good = solve(kind, norm, pts[np.where(ok[:, None], ids, 0)])
    A = pixels(kind, norm, X)
    return X, A, ok & good & np.isfinite(X).all(1) & np.isfinite(A).all(1)


def as_h(A: np.ndarray) -> np.ndarray:
    """Pixel models [H, 6] -> [H, 9] homographies with the bottom row (0, 0, 1)."""
    return np.concatenate([A, np.tile([0.0, 0.0, 1.0], (A.shape[0], 1))], 1)


def errors(A: np.ndarray, pts: np.ndarray) -> np.ndarray:
    """AF4's float32 errors [H, n]: step 5's homography error on [A; 0 0 1]."""
    return go.errors(go.HOMOGRAPHY, as_h(A), pts)


def terms(kind: int, norm, pts: np.ndarray, inl: np.ndarray, X) -> list:
    """AF6's fixed-order sums at the parameters X over the inliers: J^T J (upper triangle), J^T r and the cost."""
    x, y, u, v = _normalised(norm, pts)
    one, zero = np.ones_like(x), np.zeros_like(x)
    X = [float(c) for c in X]
    with np.errstate(all="ignore"):
        if kind == PARTIAL:
            rx = ((X[0] * x - X[1] * y) + X[2]) - u
            ry = ((X[1] * x + X[0] * y) + X[3]) - v
            jx, jy = [x, -y, one, zero], [y, x, zero, one]
        else:
            rx = ((X[0] * x + X[1] * y) + X[2]) - u
            ry = ((X[3] * x + X[4] * y) + X[5]) - v
            jx, jy = [x, y, one, zero, zero, zero], [zero, zero, zero, x, y, one]
        k = len(jx)
        vals = [jx[i] * jx[j] + jy[i] * jy[j] for i in range(k) for j in range(i, k)]
        vals += [jx[i] * rx + jy[i] * ry for i in range(k)]
        vals.append(rx * rx + ry * ry)
    return [float(s) for s in go.fixed_sum(np.stack([np.where(inl, val, 0.0) for val in vals]))]


def refine(kind: int, norm, pts: np.ndarray, inl: np.ndarray, X, steps: int) -> np.ndarray:
    """AF6: steps Levenberg-Marquardt steps from the normalised parameters X on the fixed inlier set inl."""
    def update(p, d):
        return [p[i] + d[i] for i in range(len(p))]
    return np.array(lc.refine(lambda p: terms(kind, norm, pts, inl, p), update, [float(c) for c in X], dof(kind), steps,
                             lpo.LAMBDA0))


def _fail(M: int, drawn: int) -> dict:
    return {"model": np.zeros((3, 3)), "inliers": np.zeros(M, dtype=bool), "num_inliers": 0, "success": False,
            "best_hypothesis": -1, "num_hypotheses": drawn}


def estimate_pair(kind, kpts0, kpts1, m0, threshold=3.0, max_iters=2000, confidence=0.99, refine_iters=10,
                  seed=0) -> dict:
    """One pair: the outputs of geo_estimate_affine (model [3, 3] with the bottom row (0, 0, 1))."""
    kpts0 = np.asarray(kpts0, dtype=np.float32)
    kpts1 = np.asarray(kpts1, dtype=np.float32)
    m0 = np.asarray(m0, dtype=np.int64)
    M = m0.shape[0]
    s = sample_size(kind)
    thr2 = np.float32(threshold * threshold)
    idx, pts = go.compact(kpts0, kpts1, m0)
    n = pts.shape[0]
    if n < s:
        return _fail(M, 0)
    norm = go.normalisation(pts)
    if norm is None:
        return _fail(M, 0)

    def candidates(h):
        _, A, ok = hypotheses(kind, seed, h, pts, norm)
        if not ok.any():
            return None
        return (errors(A[ok], pts) < thr2).sum(1), h[ok], np.zeros(int(ok.sum()), dtype=np.int64)

    best_cnt, best_h, _, drawn = go.ransac_pair(n, s, max_iters, confidence, candidates)
    if best_h < 0:
        return _fail(M, drawn)
    X, A, _ = hypotheses(kind, seed, np.array([best_h]), pts, norm)
    model, count = A[0], best_cnt
    if best_cnt >= s and refine_iters > 0:
        inl = errors(A, pts)[0] < thr2
        Ar = pixels(kind, norm, refine(kind, norm, pts, inl, X[0], refine_iters)[None])
        cr = int((errors(Ar, pts)[0] < thr2).sum())
        if cr >= best_cnt:
            model, count = Ar[0], cr
    inliers = np.zeros(M, dtype=bool)
    inliers[idx[errors(model[None], pts)[0] < thr2]] = True
    return {"model": as_h(model[None])[0].reshape(3, 3), "inliers": inliers, "num_inliers": count, "success": True,
            "best_hypothesis": best_h, "num_hypotheses": drawn}


def estimate(kind, kpts0, kpts1, matches0, threshold=3.0, max_iters=2000, confidence=0.99, refine_iters=10,
             seed=0) -> dict:
    """Batched: [B, M, 2], [B, N, 2], [B, M] -> the outputs of geo_estimate_affine as numpy arrays."""
    outs = [estimate_pair(kind, kpts0[b], kpts1[b], matches0[b], threshold, max_iters, confidence, refine_iters, seed)
            for b in range(len(matches0))]
    return {k: np.stack([np.asarray(o[k]) for o in outs]) for k in outs[0]}


def scene(kind: int, m: int, outliers: float, seed: int, noise: float = 0.5, unmatched: float = 0.1,
          size=(640, 480)):
    """A synthetic pair: m keypoints per image in a size[0] x size[1] image, a random affine (or similarity) transform,
    Gaussian noise of `noise` px on the inliers, a fraction `outliers` of uniformly random matches and `unmatched`
    rows of -1.  Returns (kpts0 [m, 2], kpts1 [m, 2], matches0 [m], A [2, 3], true inlier rows [m] bool)."""
    rng = np.random.default_rng(seed)
    w, h = size
    ang, sc = rng.uniform(-0.5, 0.5), rng.uniform(0.7, 1.3)
    R = sc * np.array([[np.cos(ang), -np.sin(ang)], [np.sin(ang), np.cos(ang)]])
    if kind == AFFINE:
        R = R @ np.array([[1.0 + rng.uniform(-0.2, 0.2), rng.uniform(-0.2, 0.2)], [0.0, 1.0 + rng.uniform(-0.2, 0.2)]])
    c = np.array([w / 2, h / 2])
    A = np.concatenate([R, (c - R @ c + rng.uniform(-40, 40, 2))[:, None]], 1)
    x0 = rng.uniform([0, 0], [w, h], (m, 2))
    x1 = x0 @ A[:, :2].T + A[:, 2] + rng.normal(0.0, noise, (m, 2))
    perm = rng.permutation(m)
    out = perm[: int(round(outliers * m))]
    x1[out] = rng.uniform([0, 0], [w, h], (out.size, 2))
    inlier = np.ones(m, dtype=bool)
    inlier[out] = False
    # a random outlier can land within the threshold; it still counts as an outlier of the scene
    m0 = rng.permutation(m)
    k1 = np.empty_like(x1)
    k1[m0] = x1
    drop = rng.random(m) < unmatched
    m0 = np.where(drop, -1, m0)
    inlier &= ~drop
    return x0.astype(np.float32), k1.astype(np.float32), m0.astype(np.int64), A, inlier
