"""numpy restatement of the batched RANSAC of include/geometry_b200.h (lightglue_b200/csrc/geo_api.cu).

Every step uses the header's operation order, in float64 for the solvers and float32 for the scoring, so that the CUDA
build (compiled with -fmad=false) and this file agree bit for bit: the same hypotheses, counts, inliers and models.
Hypotheses are vectorised per chunk; the per-pair refit runs on Python floats.
"""
from __future__ import annotations

import math

import numpy as np

HOMOGRAPHY, FUNDAMENTAL = 0, 1
CHUNK = 256
MAX_DRAWS = 64
FLT_EPS = 1.1920928955078125e-07
PIVOT_EPS = 1e-10
SVD_SWEEPS = 8
EIG_SWEEPS = 12
RED = 256
TRIPLES = ((0, 1, 2), (1, 2, 3), (0, 2, 3), (0, 1, 3))


def sample_size(kind: int) -> int:
    return 4 if kind == HOMOGRAPHY else 8


def mix(x: np.ndarray) -> np.ndarray:
    x = np.asarray(x, dtype=np.uint32)
    with np.errstate(over="ignore"):  # 32-bit wrap-around is the hash's arithmetic
        x = x ^ (x >> np.uint32(16))
        x = x * np.uint32(0x7FEB352D)
        x = x ^ (x >> np.uint32(15))
        x = x * np.uint32(0x846CA68B)
        return x ^ (x >> np.uint32(16))


def fixed_sum(v: np.ndarray) -> np.ndarray:
    """Sum over the last axis in the header's order: RED strided partials, then the halving tree."""
    v = np.asarray(v, dtype=np.float64)
    n = v.shape[-1]
    k = max(1, -(-n // RED))
    pad = np.zeros(v.shape[:-1] + (k * RED,))
    pad[..., :n] = v
    p = np.zeros(v.shape[:-1] + (RED,))
    for i in range(k):
        p = p + pad[..., i * RED:(i + 1) * RED]
    h = RED // 2
    while h:
        p = p[..., :h] + p[..., h:2 * h]
        h //= 2
    return p[..., 0]


def compact(kpts0: np.ndarray, kpts1: np.ndarray, m0: np.ndarray):
    """One pair: the valid matches (index in range, both keypoints finite) in ascending row order, as (rows, float32
    [n, 4] of x0, y0, x1, y1)."""
    n1 = kpts1.shape[0]
    ok = (m0 >= 0) & (m0 < n1)
    ok[ok] = np.isfinite(kpts0[ok]).all(1) & np.isfinite(kpts1[m0[ok]]).all(1)
    rows = np.nonzero(ok)[0]
    pts = np.concatenate([kpts0[rows], kpts1[m0[rows]]], axis=1).astype(np.float32)
    return rows, pts


def normalisation(pts: np.ndarray):
    """(cx0, cy0, s0, cx1, cy1, s1), or None when a mean distance is not positive."""
    n = pts.shape[0]
    c = [float(fixed_sum(pts[:, q].astype(np.float64))) / n for q in range(4)]
    out = []
    for img in range(2):
        dx = pts[:, 2 * img].astype(np.float64) - c[2 * img]
        dy = pts[:, 2 * img + 1].astype(np.float64) - c[2 * img + 1]
        d = float(fixed_sum(np.sqrt(dx * dx + dy * dy))) / n
        if not d > 0.0:
            return None
        out += [c[2 * img], c[2 * img + 1], math.sqrt(2.0) / d]
    return tuple(out)


def samples(seed: int, h: np.ndarray, n: int, s: int):
    """[H, s] sample indices and the mask of complete samples."""
    x = mix(mix(np.uint32(seed) ^ np.uint32(0x9E3779B9)) ^ h.astype(np.uint32))
    ids = np.full((h.size, s), -1, dtype=np.int64)
    k = np.zeros(h.size, dtype=np.int64)
    for t in range(MAX_DRAWS):
        r = mix(x + np.uint32(t))
        j = ((r.astype(np.uint64) * np.uint64(n)) >> np.uint64(32)).astype(np.int64)
        take = (k < s) & ~(ids == j[:, None]).any(1)
        ids[take, k[take]] = j[take]
        k[take] += 1
    return ids, k == s


def rows(kind: int, norm, pts: np.ndarray):
    """Normalised DLT rows ([..., 9] each): (ra, rb) for H, (r, None) for F."""
    cx0, cy0, s0, cx1, cy1, s1 = norm
    x = (pts[..., 0].astype(np.float64) - cx0) * s0
    y = (pts[..., 1].astype(np.float64) - cy0) * s0
    u = (pts[..., 2].astype(np.float64) - cx1) * s1
    v = (pts[..., 3].astype(np.float64) - cy1) * s1
    one, zero = np.ones_like(x), np.zeros_like(x)
    if kind == HOMOGRAPHY:
        ra = np.stack([x, y, one, zero, zero, zero, -u * x, -u * y, -u], -1)
        rb = np.stack([zero, zero, zero, x, y, one, -v * x, -v * y, -v], -1)
        return ra, rb
    return np.stack([u * x, u * y, u, v * x, v * y, v, x, y, one], -1), None


def h_sample_ok(xn: np.ndarray) -> np.ndarray:
    """xn [H, 4, 4] normalised (x0, y0, x1, y1): collinearity and orientation tests."""
    ok = np.ones(xn.shape[0], dtype=bool)
    negative = np.zeros(xn.shape[0], dtype=np.int64)
    for i, j, k in TRIPLES:
        D = []
        for img in range(2):
            X, Y = xn[:, :, 2 * img], xn[:, :, 2 * img + 1]
            dxj, dyj, dxk, dyk = X[:, j] - X[:, i], Y[:, j] - Y[:, i], X[:, k] - X[:, i], Y[:, k] - Y[:, i]
            d = dxj * dyk - dxk * dyj
            ok &= ~(np.abs(d) <= FLT_EPS * (((np.abs(dxj) + np.abs(dyj)) + np.abs(dxk)) + np.abs(dyk)))
            D.append(d)
        negative += D[0] * D[1] < 0.0
    return ok & ((negative == 0) | (negative == 4))


def null_vector(A: np.ndarray):
    """A [H, 8, 9] -> ([H, 9] null vectors with v8 = 1, mask of full-rank systems)."""
    A = A.copy()
    H = A.shape[0]
    ar = np.arange(H)
    ok = np.ones(H, dtype=bool)
    for k in range(8):
        col = np.abs(A[:, k:8, k])
        p = k + np.argmax(col, axis=1)
        best = col[ar, p - k]
        ok &= best > PIVOT_EPS
        rk = A[ar, k, k:].copy()
        A[ar, k, k:] = A[ar, p, k:]
        A[ar, p, k:] = rk
        for r in range(k + 1, 8):
            f = A[:, r, k] / A[:, k, k]
            A[:, r, k + 1:] = A[:, r, k + 1:] - f[:, None] * A[:, k, k + 1:]
    v = np.zeros((H, 9))
    v[:, 8] = 1.0
    for k in range(7, -1, -1):
        acc = A[:, k, 8].copy()
        for c in range(k + 1, 8):
            acc = acc + A[:, k, c] * v[:, c]
        v[:, k] = -acc / A[:, k, k]
    return v, ok


def _sgn1(z):
    return np.where(z >= 0.0, 1.0, -1.0)


def rank2(F: np.ndarray) -> np.ndarray:
    """[H, 9] row-major -> rank 2 by one-sided Jacobi on the columns."""
    A = F.copy()
    V = np.tile(np.eye(3).reshape(9), (F.shape[0], 1))
    for _ in range(SVD_SWEEPS):
        for p, q in ((0, 1), (0, 2), (1, 2)):
            al = be = ga = np.zeros(F.shape[0])
            for i in range(3):
                al = al + A[:, i * 3 + p] * A[:, i * 3 + p]
                be = be + A[:, i * 3 + q] * A[:, i * 3 + q]
                ga = ga + A[:, i * 3 + p] * A[:, i * 3 + q]
            skip = np.abs(ga) <= 1e-15 * np.sqrt(al * be)
            z = (be - al) / (2.0 * ga)
            t = _sgn1(z) / (np.abs(z) + np.sqrt(1.0 + z * z))
            c = 1.0 / np.sqrt(1.0 + t * t)
            s = c * t
            for M in (A, V):
                for i in range(3):
                    mp, mq = M[:, i * 3 + p].copy(), M[:, i * 3 + q].copy()
                    M[:, i * 3 + p] = np.where(skip, mp, c * mp - s * mq)
                    M[:, i * 3 + q] = np.where(skip, mq, s * mp + c * mq)
    norms = []
    for j in range(3):
        nj = np.zeros(F.shape[0])
        for i in range(3):
            nj = nj + A[:, i * 3 + j] * A[:, i * 3 + j]
        norms.append(nj)
    m = np.argmin(np.stack(norms, 1), axis=1)
    for i in range(3):
        A[np.arange(F.shape[0]), i * 3 + m] = 0.0
    out = np.empty_like(F)
    for i in range(3):
        for j in range(3):
            out[:, i * 3 + j] = (A[:, i * 3] * V[:, j * 3] + A[:, i * 3 + 1] * V[:, j * 3 + 1]) + A[:, i * 3 + 2] * V[:, j * 3 + 2]
    return out


def _mm3(A, B):
    return [(A[i * 3] * B[j] + A[i * 3 + 1] * B[3 + j]) + A[i * 3 + 2] * B[6 + j] for i in range(3) for j in range(3)]


def denormalise(kind: int, norm, v: np.ndarray) -> np.ndarray:
    """[H, 9] normalised models -> pixel models, scaled as the header says."""
    cx0, cy0, s0, cx1, cy1, s1 = norm
    T0 = [s0, 0.0, -(s0 * cx0), 0.0, s0, -(s0 * cy0), 0.0, 0.0, 1.0]
    if kind == HOMOGRAPHY:
        r = 1.0 / s1
        L = [r, 0.0, cx1, 0.0, r, cy1, 0.0, 0.0, 1.0]
    else:
        L = [s1, 0.0, 0.0, 0.0, s1, 0.0, -(s1 * cx1), -(s1 * cy1), 1.0]
    L = [np.float64(x) for x in L]
    T0 = [np.float64(x) for x in T0]
    out = np.stack(_mm3(_mm3(L, list(v.T)), T0), 1)
    f = np.zeros(v.shape[0])
    for i in range(9):
        f = f + out[:, i] * out[:, i]
    f = np.sqrt(f)
    if kind == HOMOGRAPHY:
        d = np.where(np.abs(out[:, 8]) >= 1e-12 * f, out[:, 8], f)
        return out / d[:, None]
    out = out / f[:, None]
    k = np.argmax(np.abs(out), axis=1)
    neg = out[np.arange(out.shape[0]), k] < 0.0
    return np.where(neg[:, None], -out, out)


def hypotheses(kind: int, seed: int, h: np.ndarray, pts: np.ndarray, norm):
    """Models [H, 9] float64 and the mask of non-degenerate hypotheses h of one pair."""
    s = sample_size(kind)
    ids, ok = samples(seed, h, pts.shape[0], s)
    sp = pts[np.where(ok[:, None], ids, 0)]  # [H, s, 4]
    ra, rb = rows(kind, norm, sp)
    if kind == HOMOGRAPHY:
        cx0, cy0, s0, cx1, cy1, s1 = norm
        xn = np.stack([(sp[..., 0].astype(np.float64) - cx0) * s0, (sp[..., 1].astype(np.float64) - cy0) * s0,
                       (sp[..., 2].astype(np.float64) - cx1) * s1, (sp[..., 3].astype(np.float64) - cy1) * s1], -1)
        ok &= h_sample_ok(xn)
        A = np.stack([ra, rb], 2).reshape(-1, 8, 9)
    else:
        A = ra
    with np.errstate(all="ignore"):
        v, full = null_vector(A)
        ok &= full
        if kind == FUNDAMENTAL:
            v = rank2(v)
        return denormalise(kind, norm, v), ok


def errors(kind: int, h: np.ndarray, pts: np.ndarray) -> np.ndarray:
    """float32 errors [H, n] of float32 models h [H, 9] on points [n, 4]."""
    h = h.astype(np.float32)
    x0, y0, x1, y1 = (pts[None, :, q] for q in range(4))
    g = [h[:, i:i + 1] for i in range(9)]
    one = np.float32(1.0)
    with np.errstate(all="ignore"):
        if kind == HOMOGRAPHY:
            w = one / ((g[6] * x0 + g[7] * y0) + g[8])
            dx = x1 - ((g[0] * x0 + g[1] * y0) + g[2]) * w
            dy = y1 - ((g[3] * x0 + g[4] * y0) + g[5]) * w
            return dx * dx + dy * dy
        a, b, c = (g[0] * x0 + g[1] * y0) + g[2], (g[3] * x0 + g[4] * y0) + g[5], (g[6] * x0 + g[7] * y0) + g[8]
        d2, s2 = (x1 * a + y1 * b) + c, one / (a * a + b * b)
        a, b, c = (g[0] * x1 + g[3] * y1) + g[6], (g[1] * x1 + g[4] * y1) + g[7], (g[2] * x1 + g[5] * y1) + g[8]
        d1, s1 = (x0 * a + y0 * b) + c, one / (a * a + b * b)
        return np.fmax(d1 * d1 * s1, d2 * d2 * s2)


def update_num_iters(p: float, ep: float, s: int, max_iters: int) -> int:
    """OpenCV's RANSACUpdateNumIters, pow as repeated products; confidence >= 1 never stops early."""
    if p >= 1.0:
        return max_iters
    p, ep = min(max(p, 0.0), 1.0), min(max(ep, 0.0), 1.0)
    num = max(1.0 - p, 2.2250738585072014e-308)
    q = 1.0 - ep
    pw = q
    for _ in range(1, s):
        pw = pw * q
    denom = 1.0 - pw
    if denom < 2.2250738585072014e-308:
        return 0
    num, denom = math.log(num), math.log(denom)
    return max_iters if (denom >= 0.0 or -num >= max_iters * (-denom)) else int(round(num / denom))


def ransac_pair(n: int, s: int, max_iters: int, confidence: float, candidates):
    """The chunk loop of one pair of n points and s points per sample (header steps 3 and 6).  candidates(h) gives the
    valid solutions of the samples h in (sample, solution) order as (inlier counts, samples, solution indices), or None
    without one.  The best is the first maximum count: ties go to the lowest (sample, solution).  Returns (best count,
    h, r, samples drawn), with h = r = -1 and count -1 when no sample had a valid solution."""
    best_cnt, best_h, best_r, drawn = -1, -1, -1, 0
    for c in range(-(-max_iters // CHUNK)):
        h = np.arange(c * CHUNK, min((c + 1) * CHUNK, max_iters), dtype=np.int64)
        cands = candidates(h)
        if cands is not None:
            cnt, hs, rs = cands
            i = int(np.argmax(cnt))
            if cnt[i] > best_cnt:
                best_cnt, best_h, best_r = int(cnt[i]), int(hs[i]), int(rs[i])
        drawn = min((c + 1) * CHUNK, max_iters)
        ep = 1.0 - max(best_cnt, 0) / n
        if drawn >= max_iters or drawn >= update_num_iters(confidence, ep, s, max_iters):
            break
    return best_cnt, best_h, best_r, drawn


def ata(ra: np.ndarray, rb, inl: np.ndarray) -> np.ndarray:
    """The symmetric 9x9 A^T A of the refit (header step 7): over the points with inl, each point's row ra [n, 9] and,
    when rb is not None, its second row rb, every upper-triangle entry summed in the fixed order."""
    terms = []
    for i in range(9):
        for j in range(i, 9):
            e = ra[:, i] * ra[:, j] + rb[:, i] * rb[:, j] if rb is not None else ra[:, i] * ra[:, j]
            terms.append(np.where(inl, e, 0.0))
    sums = fixed_sum(np.stack(terms))
    A, e = np.zeros((9, 9)), 0
    for i in range(9):
        for j in range(i, 9):
            A[i, j] = A[j, i] = sums[e]
            e += 1
    return A


def _eigvec_smallest(A):
    A = [[float(x) for x in r] for r in A]
    V = [[1.0 if i == j else 0.0 for j in range(9)] for i in range(9)]
    for _ in range(EIG_SWEEPS):
        for p in range(8):
            for q in range(p + 1, 9):
                apq = A[p][q]
                if apq == 0.0:
                    continue
                z = (A[q][q] - A[p][p]) / (2.0 * apq)
                t = (1.0 if z >= 0.0 else -1.0) / (abs(z) + math.sqrt(z * z + 1.0))
                c = 1.0 / math.sqrt(t * t + 1.0)
                s = t * c
                for k in range(9):
                    akp, akq = A[k][p], A[k][q]
                    A[k][p], A[k][q] = c * akp - s * akq, s * akp + c * akq
                for k in range(9):
                    apk, aqk = A[p][k], A[q][k]
                    A[p][k], A[q][k] = c * apk - s * aqk, s * apk + c * aqk
                for k in range(9):
                    vkp, vkq = V[k][p], V[k][q]
                    V[k][p], V[k][q] = c * vkp - s * vkq, s * vkp + c * vkq
    m = 0
    for k in range(1, 9):
        if A[k][k] < A[m][m]:
            m = k
    return np.array([V[k][m] for k in range(9)])


def _fail(M: int, drawn: int) -> dict:
    return {"model": np.zeros((3, 3)), "inliers": np.zeros(M, dtype=bool), "num_inliers": 0, "success": False,
            "best_hypothesis": -1, "num_hypotheses": drawn}


def estimate_pair(kind, kpts0, kpts1, m0, threshold, max_iters, confidence, seed) -> dict:
    kpts0 = np.asarray(kpts0, dtype=np.float32)
    kpts1 = np.asarray(kpts1, dtype=np.float32)
    m0 = np.asarray(m0, dtype=np.int64)
    M = m0.shape[0]
    s = sample_size(kind)
    thr2 = np.float32(threshold * threshold)
    idx, pts = compact(kpts0, kpts1, m0)
    n = pts.shape[0]
    if n < s:
        return _fail(M, 0)
    norm = normalisation(pts)
    if norm is None:
        return _fail(M, 0)

    def candidates(h):
        models, ok = hypotheses(kind, seed, h, pts, norm)
        if not ok.any():
            return None
        return (errors(kind, models[ok], pts) < thr2).sum(1), h[ok], np.zeros(int(ok.sum()), dtype=np.int64)

    best_cnt, best_h, _, drawn = ransac_pair(n, s, max_iters, confidence, candidates)
    if best_h < 0:
        return _fail(M, drawn)
    hyp, _ = hypotheses(kind, seed, np.array([best_h]), pts, norm)
    cands = [(hyp[0], best_cnt)]
    if best_cnt >= s:
        inl = errors(kind, hyp, pts)[0] < thr2
        v = _eigvec_smallest(ata(*rows(kind, norm, pts), inl))[None]
        with np.errstate(all="ignore"):
            if kind == FUNDAMENTAL:
                v = rank2(v)
            refit = denormalise(kind, norm, v)[0]
        cands.append((refit, int((errors(kind, refit[None], pts)[0] < thr2).sum())))
    model, count = cands[1] if len(cands) == 2 and cands[1][1] >= cands[0][1] else cands[0]
    inliers = np.zeros(M, dtype=bool)
    inliers[idx[errors(kind, model[None], pts)[0] < thr2]] = True
    return {"model": model.reshape(3, 3), "inliers": inliers, "num_inliers": count, "success": True,
            "best_hypothesis": best_h, "num_hypotheses": drawn}


def estimate(kind, kpts0, kpts1, matches0, threshold, max_iters, confidence, seed) -> dict:
    """Batched: [B, M, 2], [B, N, 2], [B, M] -> the outputs of geo_estimate as numpy arrays."""
    outs = [estimate_pair(kind, kpts0[b], kpts1[b], matches0[b], threshold, max_iters, confidence, seed)
            for b in range(len(matches0))]
    return {k: np.stack([np.asarray(o[k]) for o in outs]) for k in outs[0]}
