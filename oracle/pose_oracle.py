"""numpy restatement of the batched relative pose of include/geometry_b200.h (geo_relative_pose, csrc/pose_api.cu).

Every step uses the header's operation order, float64 for the solvers and float32 for the scoring, so that the CUDA build
(compiled with -fmad=false) and this file agree bit for bit: the same samples, solutions, counts, inliers, E, R and t.
Only elementwise operations sit on those paths (no BLAS, no np.sum, no np.linalg), since a library reduction may reorder
or fuse.  The five-point solver and the triangulation are vectorised over a chunk's samples and over a pair's points.

``calibrated_two_view`` draws seeded scenes with a known K0, K1, R and t.
"""
from __future__ import annotations

import math

import numpy as np

from oracle import geometry_oracle as go

S = 5           # points per sample
MAX_SOLS = 10   # real solutions of one sample, at most
PIVOT_EPS = go.PIVOT_EPS
LEAD_EPS = 1e-12
STURM_STEPS = 40
NEWTON_STEPS = 8
REFIT_MIN = 8
CHUNK = go.CHUNK

# monomials x^a y^b z^c of degree <= 3, graded: 1 | x y z | xx xy xz yy yz zz | xxx xxy xxz xyy xyz xzz yyy yyz yzz zzz
MONO = [(0, 0, 0), (1, 0, 0), (0, 1, 0), (0, 0, 1), (2, 0, 0), (1, 1, 0), (1, 0, 1), (0, 2, 0), (0, 1, 1), (0, 0, 2),
        (3, 0, 0), (2, 1, 0), (2, 0, 1), (1, 2, 0), (1, 1, 1), (1, 0, 2), (0, 3, 0), (0, 2, 1), (0, 1, 2), (0, 0, 3)]
_INDEX = {m: i for i, m in enumerate(MONO)}
MUL = [[_INDEX.get(tuple(a + b for a, b in zip(p, q)), -1) for q in MONO] for p in MONO]
# columns of the 10x20 constraint matrix: the ten monomials Gauss-Jordan eliminates, then x*(zz z 1), y*(zz z 1), zzz zz z 1
COLUMNS = [10, 16, 11, 13, 12, 4, 17, 7, 14, 5, 15, 6, 1, 18, 8, 2, 19, 9, 3, 0]
SLOTS = {1: 4, 2: 10, 3: 20}  # monomials of degree <= d


def k_valid(K) -> bool:
    K = [float(v) for v in np.asarray(K, dtype=np.float64).reshape(9)]
    return all(math.isfinite(v) for v in K) and K[0] > 0.0 and K[4] > 0.0 and K[6] == 0.0 and K[7] == 0.0 and K[8] == 1.0


def calibrate(K, xy: np.ndarray) -> np.ndarray:
    """fp32 pixels [n, 2] -> fp32 calibrated coordinates, computed in double: y = (v - cy) / fy, x = ((u - cx) - s*y) / fx."""
    fx, s, cx, _, fy, cy = (np.float64(v) for v in np.asarray(K, dtype=np.float64).reshape(9)[:6])
    u, v = xy[:, 0].astype(np.float64), xy[:, 1].astype(np.float64)
    y = (v - cy) / fy
    x = ((u - cx) - s * y) / fx
    return np.stack([x, y], 1).astype(np.float32)


def threshold2(K0, K1, threshold: float) -> np.float32:
    """The pixel threshold over the pair's mean focal length, squared, in fp32."""
    a, b = np.asarray(K0, dtype=np.float64).reshape(9), np.asarray(K1, dtype=np.float64).reshape(9)
    f = (((float(a[0]) + float(a[4])) + float(b[0])) + float(b[4])) / 4.0
    t = threshold / f
    return np.float32(t * t)


def _pmul(a, b, na, nb):
    """Product of two trivariate polynomials (lists of [H] arrays over MONO), terms added in ascending (i, j)."""
    out = [0.0] * SLOTS[{(1, 1): 2, (1, 2): 3, (2, 1): 3}[(na, nb)]]
    for i in range(SLOTS[na]):
        for j in range(SLOTS[nb]):
            k = MUL[i][j]
            out[k] = out[k] + a[i] * b[j]
    return out


def _sub(a, b):
    return [x - y for x, y in zip(a, b)]


def _umul(a, b):
    """Product of univariate polynomials (lists of [H] arrays, ascending powers), terms added in ascending (i, j)."""
    out = [0.0] * (len(a) + len(b) - 1)
    for i in range(len(a)):
        for j in range(len(b)):
            out[i + j] = out[i + j] + a[i] * b[j]
    return out


def _horner(p, z):
    v = p[-1]
    for c in p[-2::-1]:
        v = v * z + c
    return v


def _sturm(q):
    """Sturm sequence of the monic degree-10 q: members [H, 11 - k] and their validity."""
    H = q.shape[0]
    seq = [q, np.stack([(i + 1.0) * q[:, i + 1] for i in range(10)], 1)]
    valid = [np.ones(H, dtype=bool), np.ones(H, dtype=bool)]
    for k in range(2, 11):
        a, b = seq[k - 2], seq[k - 1]
        da, db = a.shape[1] - 1, b.shape[1] - 1
        qh = a[:, da] / b[:, db]
        r = a[:, :da].copy()
        r[:, 1:] = r[:, 1:] - qh[:, None] * b[:, :db]
        ql = r[:, da - 1] / b[:, db]
        r = r[:, :db] - ql[:, None] * b[:, :db]
        m = np.max(np.abs(r), axis=1)
        seq.append(-r / m[:, None])
        valid.append(valid[k - 1] & np.isfinite(r).all(1) & (r[:, db - 1] != 0.0))
    return seq, valid


def _sgn(v):
    return (v > 0.0).astype(np.float64) - (v < 0.0)


def _sign_changes(signs, valid):
    prev = np.zeros(signs[0].shape)
    v = np.zeros(signs[0].shape, dtype=np.int64)
    for sg, ok in zip(signs, valid):
        sg = np.where(ok if sg.ndim == 1 else ok[:, None], sg, 0.0)
        v = v + ((sg != 0.0) & (prev != 0.0) & (sg != prev))
        prev = np.where(sg != 0.0, sg, prev)
    return v


def _roots(p):
    """p: 11 [H] arrays, ascending powers.  -> z [H, 10], mask [H, 10] of found real roots (ascending)."""
    H = p[0].shape[0]
    P = np.stack(p, 1)
    amax = np.max(np.abs(P), axis=1)
    ok = np.isfinite(P).all(1) & (np.abs(P[:, 10]) > LEAD_EPS * amax)
    q = P / P[:, 10:11]
    rb = 1.0 + np.max(np.abs(q[:, :10]), axis=1)
    seq, valid = _sturm(q)
    lead = [_sgn(s[:, -1]) for s in seq]
    vneg = _sign_changes([ld if k % 2 == 0 else -ld for k, ld in enumerate(lead)], valid)  # degree 10 - k at -inf
    n = np.where(ok, np.maximum(vneg - _sign_changes(lead, valid), 0), 0)
    kk = np.arange(1, 11)[None, :]
    lo = np.broadcast_to(-rb[:, None], (H, 10)).copy()
    hi = np.broadcast_to(rb[:, None], (H, 10)).copy()
    for _ in range(STURM_STEPS):
        mid = 0.5 * (lo + hi)
        cnt = vneg[:, None] - _sign_changes([_sgn(_horner([s[:, i, None] for i in range(s.shape[1])], mid))
                                             for s in seq], valid)
        up = cnt >= kk
        hi = np.where(up, mid, hi)
        lo = np.where(up, lo, mid)
    z = 0.5 * (lo + hi)
    for _ in range(NEWTON_STEPS):
        v, d = q[:, 10, None], 0.0
        for i in range(9, -1, -1):
            d = d * z + v
            v = v * z + q[:, i, None]
        with np.errstate(all="ignore"):
            zn = z - v / d
        z = np.where(np.isfinite(zn), zn, z)
    return z, kk <= n[:, None]


def unit_scale(E: np.ndarray) -> np.ndarray:
    """[..., 9] -> unit Frobenius norm (row-major running sum), first largest-magnitude entry positive."""
    f = np.zeros(E.shape[:-1])
    for i in range(9):
        f = f + E[..., i] * E[..., i]
    E = E / np.sqrt(f)[..., None]
    k = np.argmax(np.abs(E), axis=-1)
    neg = np.take_along_axis(E, k[..., None], -1)[..., 0] < 0.0
    return np.where(neg[..., None], -E, E)


def five_point(sp: np.ndarray):
    """Calibrated points [H, 5, 4] (x0, y0, x1, y1) -> solutions [H, 10, 9] (unit scale, ascending root) and their mask."""
    H = sp.shape[0]
    x, y, u, v = (sp[..., q].astype(np.float64) for q in range(4))
    A = np.stack([u * x, u * y, u, v * x, v * y, v, x, y, np.ones_like(x)], -1)  # [H, 5, 9]
    ar = np.arange(H)
    ok = np.ones(H, dtype=bool)
    for k in range(5):
        col = np.abs(A[:, k:5, k])
        p = k + np.argmax(col, axis=1)
        ok &= col[ar, p - k] > PIVOT_EPS
        rk = A[ar, k, k:].copy()
        A[ar, k, k:] = A[ar, p, k:]
        A[ar, p, k:] = rk
        for r in range(k + 1, 5):
            f = A[:, r, k] / A[:, k, k]
            A[:, r, k + 1:] = A[:, r, k + 1:] - f[:, None] * A[:, k, k + 1:]
    basis = []  # X, Y, Z, W: the null vectors with free column 5, 6, 7, 8 set to 1
    for fc in range(5, 9):
        b = np.zeros((H, 9))
        b[:, fc] = 1.0
        for k in range(4, -1, -1):
            acc = A[:, k, fc].copy()
            for c in range(k + 1, 5):
                acc = acc + A[:, k, c] * b[:, c]
            b[:, k] = -acc / A[:, k, k]
        basis.append(b)
    for i in range(4):  # modified Gram-Schmidt in the order X, Y, Z, W
        for j in range(i):
            d = 0.0
            for e in range(9):
                d = d + basis[i][:, e] * basis[j][:, e]
            basis[i] = basis[i] - d[:, None] * basis[j]
        nn = 0.0
        for e in range(9):
            nn = nn + basis[i][:, e] * basis[i][:, e]
        basis[i] = basis[i] / np.sqrt(nn)[:, None]
    X, Y, Z, W = basis
    E = [[W[:, e], X[:, e], Y[:, e], Z[:, e]] for e in range(9)]  # E_e = W + x X + y Y + z Z over MONO
    d0 = _sub(_pmul(E[4], E[8], 1, 1), _pmul(E[5], E[7], 1, 1))
    d1 = _sub(_pmul(E[3], E[8], 1, 1), _pmul(E[5], E[6], 1, 1))
    d2 = _sub(_pmul(E[3], E[7], 1, 1), _pmul(E[4], E[6], 1, 1))
    rows = [[(a - b) + c for a, b, c in zip(_pmul(E[0], d0, 1, 2), _pmul(E[1], d1, 1, 2), _pmul(E[2], d2, 1, 2))]]
    EE = [[[(a + b) + c for a, b, c in zip(_pmul(E[3 * i], E[3 * j], 1, 1), _pmul(E[3 * i + 1], E[3 * j + 1], 1, 1),
                                            _pmul(E[3 * i + 2], E[3 * j + 2], 1, 1))] for j in range(3)] for i in range(3)]
    tr = [(a + b) + c for a, b, c in zip(EE[0][0], EE[1][1], EE[2][2])]
    for i in range(3):
        for j in range(3):
            T = [(a + b) + c for a, b, c in zip(_pmul(EE[i][0], E[j], 2, 1), _pmul(EE[i][1], E[3 + j], 2, 1),
                                                 _pmul(EE[i][2], E[6 + j], 2, 1))]
            rows.append([2.0 * a - b for a, b in zip(T, _pmul(tr, E[3 * i + j], 2, 1))])
    G = np.stack([np.stack([r[c] for c in COLUMNS], 1) for r in rows], 1)  # [H, 10, 20]
    amax = np.max(np.abs(G).reshape(H, -1), axis=1)
    ok &= np.isfinite(G).reshape(H, -1).all(1)
    for k in range(10):
        col = np.abs(G[:, k:10, k])
        p = k + np.argmax(col, axis=1)
        ok &= col[ar, p - k] > PIVOT_EPS * amax
        rk = G[ar, k, k:].copy()
        G[ar, k, k:] = G[ar, p, k:]
        G[ar, p, k:] = rk
        G[:, k, k + 1:] = G[:, k, k + 1:] / G[:, k, k, None]
        for r in range(10):
            if r != k:
                G[:, r, k + 1:] = G[:, r, k + 1:] - G[:, r, k, None] * G[:, k, k + 1:]
    R = G[:, :, 10:]

    def hidden(e, f):  # row e - z * row f: polynomials in z of x, y and 1
        a, b = R[:, e], R[:, f]
        return ([a[:, 2], a[:, 1] - b[:, 2], a[:, 0] - b[:, 1], -b[:, 0]],
                [a[:, 5], a[:, 4] - b[:, 5], a[:, 3] - b[:, 4], -b[:, 3]],
                [a[:, 9], a[:, 8] - b[:, 9], a[:, 7] - b[:, 8], a[:, 6] - b[:, 7], -b[:, 6]])
    (kx, ky, k1), (lx, ly, l1), (mx, my, m1) = hidden(4, 5), hidden(6, 7), hidden(8, 9)
    c0 = _sub(_umul(ly, m1), _umul(l1, my))
    c1 = _sub(_umul(lx, m1), _umul(l1, mx))
    c2 = _sub(_umul(lx, my), _umul(ly, mx))
    det = [(a - b) + c for a, b, c in zip(_umul(kx, c0), _umul(ky, c1), _umul(k1, c2))]
    z, found = _roots(det)
    found &= ok[:, None]
    B = [[_horner([c[:, None] for c in poly], z) for poly in row] for row in ((kx, ky, k1), (lx, ly, l1), (mx, my, m1))]

    def cross(a, b):
        return (a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0])
    cands = [cross(B[0], B[1]), cross(B[0], B[2]), cross(B[1], B[2])]
    best = cands[0]
    for c in cands[1:]:
        take = np.abs(c[2]) > np.abs(best[2])
        best = tuple(np.where(take, ci, bi) for ci, bi in zip(c, best))
    xs, ys = best[0] / best[2], best[1] / best[2]
    Es = np.stack([((xs * X[:, e, None] + ys * Y[:, e, None]) + z * Z[:, e, None]) + W[:, e, None] for e in range(9)], -1)
    f = np.zeros(Es.shape[:-1])
    for i in range(9):
        f = f + Es[..., i] * Es[..., i]
    found &= np.isfinite(f) & (f > 0.0)
    return unit_scale(Es), found


def sampson(E: np.ndarray, pts: np.ndarray) -> np.ndarray:
    """fp32 squared Sampson errors [H, n] of models E [H, 9] (cast to fp32) on calibrated points [n, 4]."""
    g = [E.astype(np.float32)[:, i:i + 1] for i in range(9)]
    x, y, u, v = (pts[None, :, q] for q in range(4))
    with np.errstate(all="ignore"):
        a0, a1, a2 = (g[0] * x + g[1] * y) + g[2], (g[3] * x + g[4] * y) + g[5], (g[6] * x + g[7] * y) + g[8]
        d = (u * a0 + v * a1) + a2
        b0, b1 = (g[0] * u + g[3] * v) + g[6], (g[1] * u + g[4] * v) + g[7]
        return (d * d) / (((a0 * a0 + a1 * a1) + b0 * b0) + b1 * b1)


def solutions(seed: int, h: np.ndarray, pts: np.ndarray):
    """Samples h of a pair -> ([H, 10, 9] solutions, [H, 10] mask), non-degenerate ones first-to-last per sample."""
    ids, ok = go.samples(seed, h, pts.shape[0], S)
    with np.errstate(all="ignore"):
        E, found = five_point(pts[np.where(ok[:, None], ids, 0)])
    found &= ok[:, None]
    order = np.argsort(~found, axis=1, kind="stable")  # kept solutions first, in root order
    return np.take_along_axis(E, order[..., None], 1), np.take_along_axis(found, order, 1)


def eigvec_smallest(A: np.ndarray) -> np.ndarray:
    """[..., N, N] symmetric -> the eigenvector of the least diagonal after GEO_EIG_SWEEPS cyclic Jacobi sweeps."""
    A = A.copy()
    N = A.shape[-1]
    V = np.broadcast_to(np.eye(N), A.shape).copy()
    for _ in range(go.EIG_SWEEPS):
        for p in range(N - 1):
            for q in range(p + 1, N):
                apq = A[..., p, q].copy()
                skip = apq == 0.0
                with np.errstate(all="ignore"):
                    z = (A[..., q, q] - A[..., p, p]) / (2.0 * apq)
                    t = np.where(z >= 0.0, 1.0, -1.0) / (np.abs(z) + np.sqrt(z * z + 1.0))
                c = np.where(skip, 1.0, 1.0 / np.sqrt(t * t + 1.0))
                s = np.where(skip, 0.0, t * c)
                for M, cols in ((A, True), (A, False), (V, True)):
                    if cols:
                        mp, mq = M[..., :, p].copy(), M[..., :, q].copy()
                    else:
                        mp, mq = M[..., p, :].copy(), M[..., q, :].copy()
                    np_ = np.where(skip[..., None], mp, c[..., None] * mp - s[..., None] * mq)
                    nq = np.where(skip[..., None], mq, s[..., None] * mp + c[..., None] * mq)
                    if cols:
                        M[..., :, p], M[..., :, q] = np_, nq
                    else:
                        M[..., p, :], M[..., q, :] = np_, nq
    d = np.stack([A[..., k, k] for k in range(N)], -1)
    m = np.argmin(d, axis=-1)
    return np.take_along_axis(V, m[..., None, None], -1)[..., 0]


def _svd3(E):
    """One-sided Jacobi of E [9] (geometry step 4): u1, u2 of the two larger columns in ascending index, v1, v2."""
    A = [float(e) for e in E]
    V = [1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0]
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
            for M in (A, V):
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
    i, j = [k for k in range(3) if k != m]
    si, sj = math.sqrt(nrm[i]), math.sqrt(nrm[j])
    u1 = [A[r * 3 + i] / si for r in range(3)]
    u2 = [A[r * 3 + j] / sj for r in range(3)]
    return u1, u2, [V[r * 3 + i] for r in range(3)], [V[r * 3 + j] for r in range(3)]


def _cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def essential_projection(e: np.ndarray) -> np.ndarray:
    """U diag(1, 1, 0) V^T of the one-sided Jacobi, unit scale."""
    u1, u2, v1, v2 = _svd3(e)
    return unit_scale(np.array([u1[a] * v1[b] + u2[a] * v2[b] for a in range(3) for b in range(3)]))


def pose_candidates(E):
    """The four (R [9], t [3]) of E in recoverPose's order: (R1, t), (R2, t), (R1, -t), (R2, -t)."""
    u1, u2, v1, v2 = _svd3(E)
    u3, v3 = _cross(u1, u2), _cross(v1, v2)
    R1 = [(u2[a] * v1[b] - u1[a] * v2[b]) + u3[a] * v3[b] for a in range(3) for b in range(3)]
    R2 = [(u1[a] * v2[b] - u2[a] * v1[b]) + u3[a] * v3[b] for a in range(3) for b in range(3)]
    t, nt = u3, [-c for c in u3]
    return [(R1, t), (R2, t), (R1, nt), (R2, nt)]


def cheirality(R, t, pts: np.ndarray, distance: float) -> np.ndarray:
    """recoverPose's test on calibrated points [n, 4] for one (R, t): linear triangulation by the 4x4 DLT normal matrix."""
    x, y, u, v = (pts[:, q].astype(np.float64) for q in range(4))
    zero, one = np.zeros_like(x), np.ones_like(x)
    P = [[R[0], R[1], R[2], t[0]], [R[3], R[4], R[5], t[1]], [R[6], R[7], R[8], t[2]]]
    r = [[-one, zero, x, zero], [zero, -one, y, zero],
         [u * P[2][c] - P[0][c] for c in range(4)], [v * P[2][c] - P[1][c] for c in range(4)]]
    N = np.stack([np.stack([((r[0][i] * r[0][j] + r[1][i] * r[1][j]) + r[2][i] * r[2][j]) + r[3][i] * r[3][j]
                            for j in range(4)], -1) for i in range(4)], -2)
    Q = eigvec_smallest(N)
    with np.errstate(all="ignore"):
        X, Y, Zc = Q[:, 0] / Q[:, 3], Q[:, 1] / Q[:, 3], Q[:, 2] / Q[:, 3]
        z1 = ((R[6] * X + R[7] * Y) + R[8] * Zc) + t[2]
        return (Q[:, 2] * Q[:, 3] > 0.0) & (Zc < distance) & (z1 > 0.0) & (z1 < distance)


def _fail(M: int, drawn: int) -> dict:
    return {"E": np.zeros((3, 3)), "R": np.zeros((3, 3)), "t": np.zeros(3), "inliers": np.zeros(M, dtype=bool),
            "num_inliers": 0, "pose_inliers": np.zeros(M, dtype=bool), "num_pose_inliers": 0, "success": False,
            "best_hypothesis": -1, "best_solution": -1, "num_hypotheses": drawn}


def relative_pose_pair(kpts0, kpts1, m0, K0, K1, threshold, max_iters, confidence, distance, seed) -> dict:
    kpts0 = np.asarray(kpts0, dtype=np.float32)
    kpts1 = np.asarray(kpts1, dtype=np.float32)
    m0 = np.asarray(m0, dtype=np.int64)
    K0 = np.asarray(K0, dtype=np.float64).reshape(9)
    K1 = np.asarray(K1, dtype=np.float64).reshape(9)
    M = m0.shape[0]
    idx, px = go.compact(kpts0, kpts1, m0)
    n = px.shape[0]
    if n < S or not k_valid(K0) or not k_valid(K1):
        return _fail(M, 0)
    pts = np.concatenate([calibrate(K0, px[:, :2]), calibrate(K1, px[:, 2:])], 1)
    thr2 = threshold2(K0, K1, threshold)

    def candidates(h):
        E, found = solutions(seed, h, pts)
        if not found.any():
            return None
        hh, rr = np.nonzero(found)
        return (sampson(E[found], pts) < thr2).sum(1), h[hh], rr

    best_cnt, best_h, best_r, drawn = go.ransac_pair(n, S, max_iters, confidence, candidates)
    if best_h < 0:
        return _fail(M, drawn)
    E, _ = solutions(seed, np.array([best_h]), pts)
    cands = [(E[0, best_r], best_cnt)]
    if best_cnt >= REFIT_MIN:
        inl = sampson(E[0, best_r][None], pts)[0] < thr2
        x, y, u, v = (pts[:, q].astype(np.float64) for q in range(4))
        ra = np.stack([u * x, u * y, u, v * x, v * y, v, x, y, np.ones_like(x)], 1)
        with np.errstate(all="ignore"):
            refit = essential_projection(eigvec_smallest(go.ata(ra, None, inl)))
        cands.append((refit, int((sampson(refit[None], pts)[0] < thr2).sum())))
    Ef, count = cands[1] if len(cands) == 2 and cands[1][1] >= cands[0][1] else cands[0]
    inl = sampson(Ef[None], pts)[0] < thr2
    good = [cheirality(R, t, pts[inl], distance) for R, t in pose_candidates(Ef)]
    k = 0
    for j in range(1, 4):
        if good[j].sum() > good[k].sum():
            k = j
    R, t = pose_candidates(Ef)[k]
    inliers = np.zeros(M, dtype=bool)
    inliers[idx[inl]] = True
    pose = np.zeros(M, dtype=bool)
    pose[idx[inl][good[k]]] = True
    return {"E": Ef.reshape(3, 3), "R": np.array(R).reshape(3, 3), "t": np.array(t), "inliers": inliers,
            "num_inliers": count, "pose_inliers": pose, "num_pose_inliers": int(good[k].sum()), "success": True,
            "best_hypothesis": best_h, "best_solution": best_r, "num_hypotheses": drawn}


def relative_pose(kpts0, kpts1, matches0, K0, K1, threshold=1.0, max_iters=1000, confidence=0.999, distance=50.0,
                  seed=0) -> dict:
    """Batched: [B, M, 2], [B, N, 2], [B, M], K [B, 3, 3] -> the outputs of geo_relative_pose as numpy arrays."""
    outs = [relative_pose_pair(kpts0[b], kpts1[b], matches0[b], K0[b], K1[b], threshold, max_iters, confidence,
                               distance, seed) for b in range(len(matches0))]
    return {k: np.stack([np.asarray(o[k]) for o in outs]) for k in outs[0]}


def calibrated_two_view(m: int, outliers: float, seed: int, noise: float = 0.5, unmatched: float = 0.1, K0=None, K1=None):
    """(kpts0, kpts1, matches0, true inliers, K0, K1, R, t) of a point cloud seen by two calibrated cameras, x1 = R x0 + t
    with |t| = 1; the conventions of oracle/geometry_synth.py (noise in image 1, uniform outliers, shuffled image 1)."""
    from oracle import geometry_synth as gs
    rng = np.random.default_rng(seed)
    K0 = np.array([[500.0, 0.0, gs.W / 2], [0.0, 500.0, gs.H / 2], [0.0, 0.0, 1.0]]) if K0 is None else np.asarray(K0)
    K1 = K0 if K1 is None else np.asarray(K1)
    R = gs._rot(rng)
    t = np.array([1.0, rng.uniform(-0.3, 0.3), rng.uniform(-0.2, 0.2)])
    t = t / np.linalg.norm(t)
    X = np.stack([rng.uniform(-4, 4, m), rng.uniform(-3, 3, m), rng.uniform(4, 12, m)], 1)
    p0 = X @ K0.T
    x0 = p0[:, :2] / p0[:, 2:3]
    p1 = (X @ R.T + t) @ K1.T
    x1 = p1[:, :2] / p1[:, 2:3] + rng.normal(0.0, noise, (m, 2))
    inlier = rng.random(m) >= outliers
    x1[~inlier] = rng.uniform([0, 0], [gs.W, gs.H], ((~inlier).sum(), 2))
    return (*gs._assemble(rng, x0, x1, inlier, unmatched), K0, K1, R, t)
