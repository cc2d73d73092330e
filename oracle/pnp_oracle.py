"""numpy restatement of the batched absolute pose of include/geometry_b200.h (geo_absolute_pose, csrc/pnp_api.cu).

Every step uses the header's operation order, float64 for the solver and the refit and float32 for the scoring, so that
the CUDA build (compiled with -fmad=false) and this file agree bit for bit: the same samples, solutions, counts,
inliers, R and t.  Only elementwise operations sit on those paths (no BLAS, no np.sum, no np.linalg), since a library
reduction may reorder or fuse.  The P3P solver is vectorised over a chunk's samples; the refit's per-point terms over a
pair's points, its 6x6 solve on Python floats.

The camera enters only through a ``Camera``: ``pinhole(K0)``, or pnp_dist_oracle.camera(K0, dist) with lens
distortion (steps AD1-AD4).  The pair loops here and in lo_pnp_oracle take either.

``localization_scene`` draws seeded query images of a known 3D point cloud with a known K, R and t.
"""
from __future__ import annotations

from typing import Callable, NamedTuple

import numpy as np

from oracle import geometry_oracle as go
from oracle import lo_common as lc
from oracle import pose_oracle as po

S = 3               # points per sample
MAX_SOLS = 4        # real solutions of one sample, at most
COLLINEAR_EPS = 1e-10
BISECT_STEPS = 60
NEWTON_STEPS = 4
GN_STEPS = 3
LM_STEPS = 10
LM_LAMBDA0 = 1e-3
REFIT_MIN = 6
CHUNK = go.CHUNK

k_valid = po.k_valid
calibrate = po.calibrate


def compact(kpts0, points3d1, m0):
    """One pair: rows of the valid matches (index in range, finite pixel and 3D point) in ascending order, their
    float32 pixels [n, 2] and float32 world points [n, 3]."""
    n1 = points3d1.shape[0]
    ok = (m0 >= 0) & (m0 < n1)
    ok[ok] = np.isfinite(points3d1[m0[ok]]).all(1) & np.isfinite(kpts0[ok]).all(1)
    rows = np.nonzero(ok)[0]
    return rows, kpts0[rows].astype(np.float32), points3d1[m0[rows]].astype(np.float32)


def _dot(a, b):
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]


def _sub(a, b):
    return [a[0] - b[0], a[1] - b[1], a[2] - b[2]]


def _cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def _root2(b, c):
    """Both roots of z^2 + b z + c, the larger-magnitude one first; a negative discriminant counts as 0."""
    y = np.sqrt(np.fmax(b * b - 4.0 * c, 0.0))
    q = -0.5 * (b + np.where(b >= 0.0, y, -y))
    return q, c / q


def _inverse3(x):
    """Inverse of the 3x3 x[i][j] by cofactors."""
    C = [[x[1][1] * x[2][2] - x[1][2] * x[2][1], x[1][2] * x[2][0] - x[1][0] * x[2][2], x[1][0] * x[2][1] - x[1][1] * x[2][0]],
         [x[0][2] * x[2][1] - x[0][1] * x[2][2], x[0][0] * x[2][2] - x[0][2] * x[2][0], x[0][1] * x[2][0] - x[0][0] * x[2][1]],
         [x[0][1] * x[1][2] - x[0][2] * x[1][1], x[0][2] * x[1][0] - x[0][0] * x[1][2], x[0][0] * x[1][1] - x[0][1] * x[1][0]]]
    det = x[0][0] * C[0][0] + x[0][1] * C[0][1] + x[0][2] * C[0][2]
    return [[C[j][i] / det for j in range(3)] for i in range(3)]


def p3p(bear: np.ndarray, world: np.ndarray):
    """Lambda Twist.  Calibrated (x, y) [H, 3, 2] and world points [H, 3, 3], float32 -> R [H, 4, 9], t [H, 4, 3] and
    the mask of kept solutions [H, 4], in the solver's order (+v: tau1, tau2; -v: tau1, tau2)."""
    H = bear.shape[0]
    y = []
    for k in range(3):
        xx, yy = bear[:, k, 0].astype(np.float64), bear[:, k, 1].astype(np.float64)
        n = np.sqrt(xx * xx + yy * yy + 1.0)
        y.append([xx / n, yy / n, 1.0 / n])
    X = [[world[:, k, i].astype(np.float64) for i in range(3)] for k in range(3)]
    b12, b13, b23 = -2.0 * _dot(y[0], y[1]), -2.0 * _dot(y[0], y[2]), -2.0 * _dot(y[1], y[2])
    d12, d13, d23 = _sub(X[0], X[1]), _sub(X[0], X[2]), _sub(X[1], X[2])
    a12, a13, a23 = _dot(d12, d12), _dot(d13, d13), _dot(d23, d23)
    nrm = _cross(d12, d13)
    ok = _dot(nrm, nrm) > COLLINEAR_EPS * (a12 * a13)
    c31, c23, c12 = -0.5 * b13, -0.5 * b23, -0.5 * b12
    blob = c12 * c23 * c31 - 1.0
    s31, s23, s12 = 1.0 - c31 * c31, 1.0 - c23 * c23, 1.0 - c12 * c12
    p3 = a13 * (a23 * s31 - a13 * s23)
    p2 = 2.0 * blob * a23 * a13 + a13 * (2.0 * a12 + a13) * s23 + a23 * (a23 - a12) * s31
    p1 = a23 * (a13 - a23) * s12 - a12 * a12 * s23 - 2.0 * a12 * (blob * a23 + a13 * s23)
    p0 = a12 * (a12 * s23 - a23 * s12)
    cb, cc, cd = p2 / p3, p1 / p3, p0 / p3
    ok &= np.isfinite(cb) & np.isfinite(cc) & np.isfinite(cd)

    def cubic(g):
        return ((g + cb) * g + cc) * g + cd
    rb = 1.0 + np.fmax(np.fmax(np.abs(cb), np.abs(cc)), np.abs(cd))
    disc = cb * cb - 3.0 * cc
    v = np.sqrt(np.fmax(disc, 0.0))
    t1 = (-cb - v) / 3.0
    left = (disc >= 0.0) & (cubic(t1) > 0.0)
    right = (disc >= 0.0) & ~(cubic(t1) > 0.0)
    lo = np.where(right, (-cb + v) / 3.0, -rb)
    hi = np.where(left, t1, rb)
    for _ in range(BISECT_STEPS):
        mid = 0.5 * (lo + hi)
        up = cubic(mid) > 0.0
        hi, lo = np.where(up, mid, hi), np.where(up, lo, mid)
    g = 0.5 * (lo + hi)
    for _ in range(NEWTON_STEPS):
        gn = g - cubic(g) / ((3.0 * g + 2.0 * cb) * g + cc)
        g = np.where(np.isfinite(gn), gn, g)
    A00 = a23 * (1.0 - g)
    A01 = a23 * b12 * 0.5
    A02 = a23 * b13 * g * -0.5
    A11 = a23 - a12 + a13 * g
    A12 = b23 * (a13 * g - a12) * 0.5
    A22 = g * (a13 - a23) - a12
    e1, e2 = _root2(-A00 - A11 - A22, -(A01 * A01) - A02 * A02 - A12 * A12 + A00 * (A11 + A22) + A11 * A22)
    sw = np.abs(e1) < np.abs(e2)
    e1, e2 = np.where(sw, e2, e1), np.where(sw, e1, e2)
    mx = -(A00 * A11)
    pr0 = A01 * A12 - A02 * A11
    pr1 = A01 * A02 - A00 * A12

    def evec(e):
        tmp = 1.0 / (e * (A00 + A11) + mx - e * e + A01 * A01)
        a1 = -(e * A02 + pr0) * tmp
        a2 = -(e * A12 + pr1) * tmp
        rn = 1.0 / np.sqrt(a1 * a1 + a2 * a2 + 1.0)
        return a1 * rn, a2 * rn, rn
    V00, V10, V20 = evec(e1)
    V01, V11, V21 = evec(e2)
    sv = np.sqrt(np.fmax(0.0, -e2 / e1))
    Xi = _inverse3([[d12[i], d13[i], nrm[i]] for i in range(3)])
    Rs, ts, keep = [], [], []
    for s in (sv, -sv):
        w2 = 1.0 / (s * V01 - V00)
        w0 = (V10 - s * V11) * w2
        w1 = (V20 - s * V21) * w2
        ia = 1.0 / ((a13 - a12) * w1 * w1 - a12 * b13 * w1 - a12)
        qb = (a13 * b12 * w1 - a12 * b13 * w0 - 2.0 * w0 * w1 * (a12 - a13)) * ia
        qc = ((a13 - a12) * w0 * w0 + a13 * b12 * w0 + a13) * ia
        real = qb * qb - 4.0 * qc >= 0.0
        for tau in _root2(qb, qc):
            d = a23 / (tau * (b23 + tau) + 1.0)
            l2 = np.sqrt(d)
            l3 = tau * l2
            l1 = w0 * l2 + w1 * l3
            kp = ok & real & (tau > 0.0) & (d > 0.0) & (l1 >= 0.0)
            for _ in range(GN_STEPS):
                r1 = l1 * l1 + l2 * l2 + b12 * l1 * l2 - a12
                r2 = l1 * l1 + l3 * l3 + b13 * l1 * l3 - a13
                r3 = l2 * l2 + l3 * l3 + b23 * l2 * l3 - a23
                v0, v1 = 2.0 * l1 + b12 * l2, 2.0 * l2 + b12 * l1
                v3, v5 = 2.0 * l1 + b13 * l3, 2.0 * l3 + b13 * l1
                v7, v8 = 2.0 * l2 + b23 * l3, 2.0 * l3 + b23 * l2
                det = -(v0 * v5 * v7) - v1 * v3 * v8
                j0 = -(v5 * v7) * r1 - v1 * v8 * r2 + v1 * v5 * r3
                j1 = -(v3 * v8) * r1 + v0 * v8 * r2 - v0 * v5 * r3
                j2 = v3 * v7 * r1 - v0 * v7 * r2 - v1 * v3 * r3
                n1, n2, n3 = l1 - j0 / det, l2 - j1 / det, l3 - j2 / det
                fin = np.isfinite(n1) & np.isfinite(n2) & np.isfinite(n3)
                l1, l2, l3 = np.where(fin, n1, l1), np.where(fin, n2, l2), np.where(fin, n3, l3)
            ry = [[y[k][i] * lk for i in range(3)] for k, lk in enumerate((l1, l2, l3))]
            yd1, yd2 = _sub(ry[0], ry[1]), _sub(ry[0], ry[2])
            yc = _cross(yd1, yd2)
            Y = [[yd1[i], yd2[i], yc[i]] for i in range(3)]
            R = [Y[i][0] * Xi[0][j] + Y[i][1] * Xi[1][j] + Y[i][2] * Xi[2][j] for i in range(3) for j in range(3)]
            t = [ry[0][i] - (R[3 * i] * X[0][0] + R[3 * i + 1] * X[0][1] + R[3 * i + 2] * X[0][2]) for i in range(3)]
            for c in R + t:
                kp &= np.isfinite(c)
            Rs.append(np.stack(R, -1))
            ts.append(np.stack(t, -1))
            keep.append(kp)
    return np.stack(Rs, 1), np.stack(ts, 1), np.stack(keep, 1)


def projection(R: np.ndarray, t: np.ndarray, K) -> np.ndarray:
    """[..., 9], [..., 3] and K [9] -> P = K [R | t] [..., 12] float64, P_ij = (K_i0*M_0j + K_i1*M_1j) + K_i2*M_2j."""
    K = [np.float64(k) for k in np.asarray(K, dtype=np.float64).reshape(9)]
    M = [[R[..., 3 * i + j] for j in range(3)] + [t[..., i]] for i in range(3)]
    return np.stack([K[3 * i] * M[0][j] + K[3 * i + 1] * M[1][j] + K[3 * i + 2] * M[2][j]
                     for i in range(3) for j in range(4)], -1)


def errors(P: np.ndarray, pix: np.ndarray, wld: np.ndarray) -> np.ndarray:
    """fp32 errors [H, n] of projections P [H, 12] (cast to fp32) on pixels [n, 2] and world points [n, 3] (header
    steps A5 and LA3): du*du + dv*dv in front of the camera (w > 0), +inf behind it, so that the inlier test err < thr2
    and the LA3 score both count such a point as an outlier."""
    g = [P.astype(np.float32)[:, i:i + 1] for i in range(12)]
    u, v = pix[None, :, 0], pix[None, :, 1]
    X, Y, Z = wld[None, :, 0], wld[None, :, 1], wld[None, :, 2]
    with np.errstate(all="ignore"):
        w = g[8] * X + g[9] * Y + g[10] * Z + g[11]
        iw = np.float32(1.0) / w
        du = u - (g[0] * X + g[1] * Y + g[2] * Z + g[3]) * iw
        dv = v - (g[4] * X + g[5] * Y + g[6] * Z + g[7]) * iw
        return np.where(w > 0.0, du * du + dv * dv, np.float32(np.inf))


def inliers(camera, M: np.ndarray, pix: np.ndarray, wld: np.ndarray, thr2: np.float32) -> np.ndarray:
    """The fp32 inlier masks [H, n] of the camera's models M [H, 12]: err < thr2 (A5, AD2)."""
    with np.errstate(invalid="ignore"):
        return camera.errors(M, pix, wld) < thr2


def reproj_inliers(P: np.ndarray, pix: np.ndarray, wld: np.ndarray, thr2: np.float32) -> np.ndarray:
    """fp32 inlier masks [H, n] of projections P [H, 12] (cast to fp32) on pixels [n, 2] and world points [n, 3]: depth
    w > 0 and squared reprojection error below thr2."""
    with np.errstate(invalid="ignore"):
        return errors(P, pix, wld) < thr2


def solutions(seed: int, h: np.ndarray, bear: np.ndarray, wld: np.ndarray):
    """Samples h of a pair -> (R [H, 4, 9], t [H, 4, 3], mask [H, 4]), kept solutions first, in the solver's order."""
    ids, ok = go.samples(seed, h, bear.shape[0], S)
    ids = np.where(ok[:, None], ids, 0)
    with np.errstate(all="ignore"):
        R, t, kept = p3p(bear[ids], wld[ids])
    kept &= ok[:, None]
    order = np.argsort(~kept, axis=1, kind="stable")
    return (np.take_along_axis(R, order[..., None], 1), np.take_along_axis(t, order[..., None], 1),
            np.take_along_axis(kept, order, 1))


def residuals(x, K, pix: np.ndarray, wld: np.ndarray):
    """At x = R (9, row-major) + t (3): double residuals (ru, rv) in pixels, errors ru*ru + rv*rv, depths Xc2 and the
    Jacobian rows ju, jv [6, n] of A7 (header steps A7 and LA7)."""
    R, t = x[:9], x[9:]
    fx, s, cx, fy, cy = (float(K[i]) for i in (0, 1, 2, 4, 5))
    u, v = pix[:, 0].astype(np.float64), pix[:, 1].astype(np.float64)
    W = [wld[:, i].astype(np.float64) for i in range(3)]
    with np.errstate(all="ignore"):
        Xc = [R[3 * i] * W[0] + R[3 * i + 1] * W[1] + R[3 * i + 2] * W[2] + t[i] for i in range(3)]
        iz = 1.0 / Xc[2]
        a, b = Xc[0] * iz, Xc[1] * iz
        pu = fx * a + s * b
        ru, rv = pu + cx - u, fy * b + cy - v
        gu = [fx * iz, s * iz, -(pu * iz)]
        gv = [np.zeros_like(iz), fy * iz, -(fy * b * iz)]

        def jrow(g):
            return [g[2] * Xc[1] - g[1] * Xc[2], g[0] * Xc[2] - g[2] * Xc[0], g[1] * Xc[0] - g[0] * Xc[1], g[0], g[1], g[2]]
        ju, jv = np.stack(jrow(gu)), np.stack(jrow(gv))
        err = ru * ru + rv * rv
    return ru, rv, err, Xc[2], ju, jv


def normal_sums(ru, rv, ju, jv, inl) -> list:
    """J^T J (upper triangle, row order) and J^T r over the points with inl, unsummed: 27 [n] arrays."""
    with np.errstate(all="ignore"):
        rows = [np.where(inl, ju[i] * ju[j] + jv[i] * jv[j], 0.0) for i in range(6) for j in range(i, 6)]
        return rows + [np.where(inl, ju[i] * ru + jv[i] * rv, 0.0) for i in range(6)]


def update(x, d):
    """R' = Q R, t' = Q t + d[3:] with Q the rotation of the unit quaternion (1, d[:3] / 2) / norm (A7's step)."""
    R, t = x[:9], x[9:]
    Q = lc.quat_rotation(d)
    Rn = [Q[3 * i] * R[j] + Q[3 * i + 1] * R[3 + j] + Q[3 * i + 2] * R[6 + j] for i in range(3) for j in range(3)]
    tn = [Q[3 * i] * t[0] + Q[3 * i + 1] * t[1] + Q[3 * i + 2] * t[2] + d[3 + i] for i in range(3)]
    return Rn + tn


class Camera(NamedTuple):
    """What the pair loops of both estimators read of a pair's camera."""
    valid: bool          # K0 (and the coefficients) let the pair run
    bearings: Callable   # fp32 pixels [n, 2] -> the fp32 calibrated (x, y) [n, 2] that P3P reads
    model: Callable      # (R [..., 9], t [..., 3]) -> the model [..., 12] that is rounded to fp32 and scored
    errors: Callable     # (models [H, 12], pixels, world points) -> fp32 errors [H, n], +inf behind the camera
    residuals: Callable  # (x, pixels, world points) -> (ru, rv, err, depth, ju, jv) in double, as residuals below


def pinhole(K) -> Camera:
    """The pinhole camera K (header steps A1-A8): K^-1, P = K [R | t], the fp32 error in pixels and A7's residuals."""
    K = np.asarray(K, dtype=np.float64).reshape(9)
    return Camera(k_valid(K), lambda pix: calibrate(K, pix), lambda R, t: projection(R, t, K), errors,
                  lambda x, pix, wld: residuals(x, K, pix, wld))


def refine_lm(R, t, K, pix, wld, inl, camera=None):
    """GEO_PNP_LM_STEPS Levenberg-Marquardt steps on the squared reprojection error of the inliers, from (R, t), through
    the camera (None: pinhole(K))."""
    cam = pinhole(K) if camera is None else camera

    def terms(x):
        ru, rv, err, _, ju, jv = cam.residuals(x, pix, wld)
        return go.fixed_sum(np.stack(normal_sums(ru, rv, ju, jv, inl) + [np.where(inl, err, 0.0)]))

    x = lc.refine(terms, update, [float(c) for c in R] + [float(c) for c in t], 6, LM_STEPS, LM_LAMBDA0)
    return np.array(x[:9]), np.array(x[9:])


def _fail(M: int, drawn: int) -> dict:
    return {"R": np.zeros((3, 3)), "t": np.zeros(3), "inliers": np.zeros(M, dtype=bool), "num_inliers": 0,
            "success": False, "best_hypothesis": -1, "best_solution": -1, "num_hypotheses": drawn}


def absolute_pose_pair(kpts0, points3d1, m0, K0, threshold, max_iters, confidence, seed, camera=None) -> dict:
    """One pair of geo_absolute_pose, or of geo_absolute_pose_dist with camera=pnp_dist_oracle.camera(K0, dist).
    camera=None is pinhole(K0)."""
    kpts0 = np.asarray(kpts0, dtype=np.float32)
    points3d1 = np.asarray(points3d1, dtype=np.float32)
    m0 = np.asarray(m0, dtype=np.int64)
    cam = pinhole(K0) if camera is None else camera
    M = m0.shape[0]
    idx, pix, wld = compact(kpts0, points3d1, m0)
    n = pix.shape[0]
    if n < S or not cam.valid:
        return _fail(M, 0)
    bear = cam.bearings(pix)
    thr2 = np.float32(threshold * threshold)

    def inl(R, t):
        return inliers(cam, cam.model(R, t), pix, wld, thr2)

    def candidates(h):
        R, t, kept = solutions(seed, h, bear, wld)
        if not kept.any():
            return None
        hh, rr = np.nonzero(kept)
        return inl(R[kept], t[kept]).sum(1), h[hh], rr

    best_cnt, best_h, best_r, drawn = go.ransac_pair(n, S, max_iters, confidence, candidates)
    if best_h < 0:
        return _fail(M, drawn)
    R, t, _ = solutions(seed, np.array([best_h]), bear, wld)
    R0, t0 = R[0, best_r], t[0, best_r]
    cands = [(R0, t0, best_cnt)]
    if best_cnt >= REFIT_MIN:
        Rr, tr = refine_lm(R0, t0, K0, pix, wld, inl(R0[None], t0[None])[0], cam)
        cands.append((Rr, tr, int(inl(Rr[None], tr[None])[0].sum())))
    Rf, tf, count = cands[1] if len(cands) == 2 and cands[1][2] >= cands[0][2] else cands[0]
    mask = np.zeros(M, dtype=bool)
    mask[idx[inl(np.asarray(Rf)[None], np.asarray(tf)[None])[0]]] = True
    return {"R": np.asarray(Rf).reshape(3, 3), "t": np.asarray(tf), "inliers": mask, "num_inliers": count,
            "success": True, "best_hypothesis": best_h, "best_solution": best_r, "num_hypotheses": drawn}


def absolute_pose(kpts0, points3d1, matches0, K0, threshold=8.0, max_iters=100, confidence=0.99, seed=0) -> dict:
    """Batched: [B, M, 2], [B, N, 3], [B, M], K0 [B, 3, 3] -> the outputs of geo_absolute_pose as numpy arrays."""
    outs = [absolute_pose_pair(kpts0[b], points3d1[b], matches0[b], K0[b], threshold, max_iters, confidence, seed)
            for b in range(len(matches0))]
    return {k: np.stack([np.asarray(o[k]) for o in outs]) for k in outs[0]}


def localization_scene(m: int, outliers: float, seed: int, unmatched: float = 0.1, missing3d: float = 0.05, K=None,
                       planar: bool = False, noise: float = 0.5):
    """(kpts0 [m, 2], points3d1 [m, 3], matches0 [m], true inliers [m], K, R, t) of a query camera x = K (R X + t)
    seeing m world points at depths 4..12 (on one plane with ``planar``), with ``noise`` px of Gaussian noise, a share
    ``outliers`` of the matched rows moved uniformly over the 640x480 image, a share ``unmatched`` of the rows of
    matches0 set to -1 and a share ``missing3d`` of the 3D rows set to NaN.  points3d1 is shuffled, as a database
    image's keypoints would be."""
    from oracle import geometry_synth as gs
    rng = np.random.default_rng(seed)
    K = np.array([[500.0, 0.0, gs.W / 2], [0.0, 500.0, gs.H / 2], [0.0, 0.0, 1.0]]) if K is None else np.asarray(K)
    R = gs._rot(rng)
    t = rng.uniform(-1.0, 1.0, 3)
    a, b = rng.uniform(-4, 4, m), rng.uniform(-3, 3, m)
    z = 8.0 + 0.3 * a - 0.2 * b if planar else rng.uniform(4, 12, m)
    Xc = np.stack([a, b, z], 1)
    p = Xc @ K.T
    x0 = p[:, :2] / p[:, 2:3] + rng.normal(0.0, noise, (m, 2))
    inlier = rng.random(m) >= outliers
    x0[~inlier] = rng.uniform([0, 0], [gs.W, gs.H], ((~inlier).sum(), 2))
    X = (Xc - t) @ R  # R^T (Xc - t)
    kpts0, pts3d, matches0, truth = gs._assemble(rng, x0, X, inlier, unmatched)
    miss = rng.random(m) < missing3d
    pts3d[miss] = np.nan
    truth &= ~miss[np.maximum(matches0, 0)]
    return kpts0, pts3d, matches0, truth, K, R, t
