"""numpy restatement of the 3D rigid and similarity RANSAC of include/geometry_b200.h (steps RG1-RG7,
lightglue_b200/csrc/rigid_api.cu).

Compaction, sampling, the fixed-order sums, the stopping rule and the chunk loop are geometry_oracle's (its compaction
works unchanged on three-column points).  What is new here is Horn's closed form with the 4x4 cyclic Jacobi, the
degeneracy rule, the fp32 distance and the refit.  float64 for the solver and the refit, float32 for the scoring, one
operation at a time, so the CUDA build compiled with -fmad=false agrees bit for bit.
"""
from __future__ import annotations

import numpy as np

from oracle import geometry_oracle as go

RIGID, SIMILARITY = 5, 6
S = 3
COLLINEAR_EPS = 1e-10
_COLS = 1 << 14  # points per block of the scoring, to bound its temporaries


def _dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def _cross(a, b):
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1)


def collinear(x: np.ndarray) -> np.ndarray:
    """RG3's degeneracy rule on triangles x [H, 3, 3] (sample, point, coordinate): collinear or coincident."""
    d1, d2 = x[:, 1] - x[:, 0], x[:, 2] - x[:, 0]
    c = _cross(d1, d2)
    return ~(_dot(c, c) > COLLINEAR_EPS * (_dot(d1, d1) * _dot(d2, d2)))


def eigvec_smallest4(A: np.ndarray) -> np.ndarray:
    """Header step 7's cyclic Jacobi on symmetric 4x4 matrices A [H, 4, 4]: the eigenvectors [H, 4] of the first least
    diagonal entry (smallest_eigvec<4>)."""
    A = np.array(A, dtype=np.float64)
    H = A.shape[0]
    V = np.tile(np.eye(4), (H, 1, 1))
    with np.errstate(all="ignore"):
        for _ in range(go.EIG_SWEEPS):
            for p in range(3):
                for q in range(p + 1, 4):
                    apq = A[:, p, q].copy()
                    live = (apq != 0.0)[:, None]
                    z = (A[:, q, q] - A[:, p, p]) / (2.0 * apq)
                    t = np.where(z >= 0.0, 1.0, -1.0) / (np.abs(z) + np.sqrt(z * z + 1.0))
                    c = (1.0 / np.sqrt(t * t + 1.0))[:, None]
                    s = t[:, None] * c
                    for M, rows in ((A, False), (A, True), (V, False)):
                        xp = (M[:, p, :] if rows else M[:, :, p]).copy()
                        xq = (M[:, q, :] if rows else M[:, :, q]).copy()
                        np_, nq_ = np.where(live, c * xp - s * xq, xp), np.where(live, s * xp + c * xq, xq)
                        if rows:
                            M[:, p, :], M[:, q, :] = np_, nq_
                        else:
                            M[:, :, p], M[:, :, q] = np_, nq_
    m = np.zeros(H, dtype=np.int64)
    ar = np.arange(H)
    for k in range(1, 4):
        m = np.where(A[:, k, k] < A[ar, m, m], k, m)
    return V[ar, :, m]


def fit(kind: int, pb: np.ndarray, qb: np.ndarray, Sab: np.ndarray, saa: np.ndarray):
    """RG3's closed form from the centroids pb, qb [H, 3], the cross-covariance Sab [H, 3, 3] (Sab[i, j] = sum a_i b_j)
    and saa [H] = sum |a|^2: solutions [H, 13] (R row-major, t, scale) and the mask of non-degenerate ones."""
    sxx, sxy, sxz = Sab[:, 0, 0], Sab[:, 0, 1], Sab[:, 0, 2]
    syx, syy, syz = Sab[:, 1, 0], Sab[:, 1, 1], Sab[:, 1, 2]
    szx, szy, szz = Sab[:, 2, 0], Sab[:, 2, 1], Sab[:, 2, 2]
    N = np.stack([np.stack([(sxx + syy) + szz, syz - szy, szx - sxz, sxy - syx], -1),
                  np.stack([syz - szy, (sxx - syy) - szz, sxy + syx, szx + sxz], -1),
                  np.stack([szx - sxz, sxy + syx, (syy - sxx) - szz, syz + szy], -1),
                  np.stack([sxy - syx, szx + sxz, syz + szy, (szz - sxx) - syy], -1)], 1)
    v = eigvec_smallest4(-N)
    with np.errstate(all="ignore"):
        nq = np.sqrt(((v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1]) + v[:, 2] * v[:, 2]) + v[:, 3] * v[:, 3])
        w, x, y, z = v[:, 0] / nq, v[:, 1] / nq, v[:, 2] / nq, v[:, 3] / nq
        R = np.stack([1.0 - 2.0 * (y * y + z * z), 2.0 * (x * y - w * z), 2.0 * (x * z + w * y),
                      2.0 * (x * y + w * z), 1.0 - 2.0 * (x * x + z * z), 2.0 * (y * z - w * x),
                      2.0 * (x * z - w * y), 2.0 * (y * z + w * x), 1.0 - 2.0 * (x * x + y * y)], 1)
        if kind == SIMILARITY:
            num = np.zeros(R.shape[0])
            for i in range(3):
                for j in range(3):
                    num = num + R[:, i * 3 + j] * Sab[:, j, i]
            sc = num / saa
        else:
            sc = np.ones(R.shape[0])
        t = np.stack([qb[:, i] - sc * ((R[:, i * 3] * pb[:, 0] + R[:, i * 3 + 1] * pb[:, 1]) + R[:, i * 3 + 2] * pb[:, 2])
                      for i in range(3)], 1)
    x = np.concatenate([R, t, sc[:, None]], 1)
    return x, (sc > 0.0) & np.isfinite(sc) & np.isfinite(x[:, :12]).all(1)


def hypotheses(kind: int, seed: int, h: np.ndarray, p: np.ndarray, q: np.ndarray):
    """Solutions [H, 13] and the mask of non-degenerate hypotheses h of one pair with compacted points p, q [n, 3]."""
    ids, ok = go.samples(seed, h, p.shape[0], S)
    ids = np.where(ok[:, None], ids, 0)
    P, Q = p[ids].astype(np.float64), q[ids].astype(np.float64)  # [H, 3, 3]
    ok &= ~collinear(P) & ~collinear(Q)
    pb = ((P[:, 0] + P[:, 1]) + P[:, 2]) / 3.0
    qb = ((Q[:, 0] + Q[:, 1]) + Q[:, 2]) / 3.0
    a, b = P - pb[:, None], Q - qb[:, None]
    Sab, saa = np.zeros((len(h), 3, 3)), np.zeros(len(h))
    for k in range(S):
        Sab = Sab + a[:, k, :, None] * b[:, k, None, :]
        saa = saa + _dot(a[:, k], a[:, k])
    x, good = fit(kind, pb, qb, Sab, saa)
    return x, ok & good


def float_model(x: np.ndarray) -> np.ndarray:
    """Solutions [H, 13] -> RG4's float32 models [H, 12], [scale R | t] row-major."""
    g = np.empty((x.shape[0], 12))
    with np.errstate(all="ignore"):
        for i in range(3):
            for j in range(3):
                g[:, i * 4 + j] = x[:, 12] * x[:, i * 3 + j]
            g[:, i * 4 + 3] = x[:, 9 + i]
    return g.astype(np.float32)


def errors(g: np.ndarray, p: np.ndarray, q: np.ndarray) -> np.ndarray:
    """RG4's float32 squared distances [H, n] of float32 models g [H, 12] on compacted points p, q [n, 3]."""
    out = np.empty((g.shape[0], p.shape[0]), dtype=np.float32)
    c = [g[:, k:k + 1] for k in range(12)]
    with np.errstate(all="ignore"):
        for lo in range(0, p.shape[0], _COLS):
            x, y, z = (p[None, lo:lo + _COLS, k] for k in range(3))
            e = [(((c[4 * i] * x + c[4 * i + 1] * y) + c[4 * i + 2] * z) + c[4 * i + 3]) - q[None, lo:lo + _COLS, i]
                 for i in range(3)]
            out[:, lo:lo + _COLS] = (e[0] * e[0] + e[1] * e[1]) + e[2] * e[2]
    return out


def refit(kind: int, p: np.ndarray, q: np.ndarray, inl: np.ndarray) -> np.ndarray:
    """RG6: the closed form on the points with inl, by two passes of fixed-order sums; NaN when degenerate."""
    P, Q = p.astype(np.float64), q.astype(np.float64)
    k = float(inl.sum())
    c = go.fixed_sum(np.where(inl, np.concatenate([P, Q], 1).T, 0.0)) / k
    a, b = P - c[:3], Q - c[3:]
    terms = [a[:, i] * b[:, j] for i in range(3) for j in range(3)] + [_dot(a, a)]
    sums = go.fixed_sum(np.where(inl, np.stack(terms), 0.0))
    x, ok = fit(kind, c[None, :3], c[None, 3:], sums[:9].reshape(1, 3, 3), sums[9:])
    return x[0] if ok[0] else np.full(13, np.nan)


def _fail(M: int, drawn: int) -> dict:
    return {"R": np.zeros((3, 3)), "t": np.zeros(3), "scale": 0.0, "inliers": np.zeros(M, dtype=bool),
            "num_inliers": 0, "success": False, "best_hypothesis": -1, "num_hypotheses": drawn}


def estimate_pair(kind, points0, points1, m0, threshold, max_iters=1000, confidence=0.99, seed=0) -> dict:
    """One pair: the outputs of geo_estimate_rigid."""
    points0 = np.asarray(points0, dtype=np.float32)
    points1 = np.asarray(points1, dtype=np.float32)
    m0 = np.asarray(m0, dtype=np.int64)
    M = m0.shape[0]
    thr2 = np.float32(threshold * threshold)
    idx, pts = go.compact(points0, points1, m0)
    p, q = np.ascontiguousarray(pts[:, :3]), np.ascontiguousarray(pts[:, 3:])
    n = p.shape[0]
    if n < S:
        return _fail(M, 0)

    def candidates(h):
        x, ok = hypotheses(kind, seed, h, p, q)
        if not ok.any():
            return None
        return (errors(float_model(x[ok]), p, q) < thr2).sum(1), h[ok], np.zeros(int(ok.sum()), dtype=np.int64)

    best_cnt, best_h, _, drawn = go.ransac_pair(n, S, max_iters, confidence, candidates)
    if best_h < 0:
        return _fail(M, drawn)
    x, _ = hypotheses(kind, seed, np.array([best_h]), p, q)
    model, count = x[0], best_cnt
    if best_cnt >= S:
        xr = refit(kind, p, q, errors(float_model(x), p, q)[0] < thr2)
        cr = int((errors(float_model(xr[None]), p, q)[0] < thr2).sum())
        if cr >= best_cnt:
            model, count = xr, cr
    inliers = np.zeros(M, dtype=bool)
    inliers[idx[errors(float_model(model[None]), p, q)[0] < thr2]] = True
    return {"R": model[:9].reshape(3, 3), "t": model[9:12].copy(), "scale": float(model[12]), "inliers": inliers,
            "num_inliers": count, "success": True, "best_hypothesis": best_h, "num_hypotheses": drawn}


def estimate(kind, points0, points1, matches0, threshold, max_iters=1000, confidence=0.99, seed=0) -> dict:
    """Batched: [B, M, 3], [B, N, 3], [B, M] -> the outputs of geo_estimate_rigid as numpy arrays."""
    outs = [estimate_pair(kind, points0[b], points1[b], matches0[b], threshold, max_iters, confidence, seed)
            for b in range(len(matches0))]
    return {k: np.stack([np.asarray(o[k]) for o in outs]) for k in outs[0]}


def random_rotation(rng) -> np.ndarray:
    q = rng.normal(size=4)
    w, x, y, z = q / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def depth_points(rng, m: int, size=(640, 480), f=525.0, depth=(0.5, 5.0)) -> np.ndarray:
    """m points [m, 3] in a depth camera's view: pixels uniform in the image, depths uniform in `depth` metres."""
    w, h = size
    u, v = rng.uniform(0, w, m), rng.uniform(0, h, m)
    zz = rng.uniform(*depth, m)
    return np.stack([(u - w / 2) / f * zz, (v - h / 2) / f * zz, zz], 1)


def scene(kind: int, m: int, outliers: float, seed: int, noise: float = 0.01, unmatched: float = 0.1):
    """A synthetic pair: m points of a depth camera's view in frame 0, a random SE(3) (or Sim(3), scale in [0.5, 2])
    to frame 1, Gaussian noise of `noise` (frame-1 units) per coordinate on the inliers, a fraction `outliers` of
    matches moved to random points of the view in frame 1, and `unmatched` rows of -1.  Returns (points0 [m, 3],
    points1 [m, 3], matches0 [m], (R, t, scale), true inlier rows [m] bool)."""
    rng = np.random.default_rng(seed)
    R = random_rotation(rng)
    sc = rng.uniform(0.5, 2.0) if kind == SIMILARITY else 1.0
    t = rng.uniform(-1.0, 1.0, 3)
    x0 = depth_points(rng, m)
    x1 = sc * x0 @ R.T + t + rng.normal(0.0, noise, (m, 3))
    out = rng.permutation(m)[: int(round(outliers * m))]
    x1[out] = sc * depth_points(rng, out.size) @ R.T + t
    inlier = np.ones(m, dtype=bool)
    inlier[out] = False
    m0 = rng.permutation(m)
    p1 = np.empty_like(x1)
    p1[m0] = x1
    drop = rng.random(m) < unmatched
    m0 = np.where(drop, -1, m0)
    inlier &= ~drop
    return x0.astype(np.float32), p1.astype(np.float32), m0.astype(np.int64), (R, t, sc), inlier
