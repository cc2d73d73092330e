"""numpy restatement of the lens distortion of include/geometry_b200.h (steps D1-D3, csrc/camera_api.cu).

Elementwise operations only, in the header's order, so that the CUDA build compiled with -fmad=false agrees bit for
bit.  ``distort`` runs in the dtype of its inputs: float64 for D1-D2, float32 for the absolute pose's inlier test
(step AD2), whose coefficients are rounded to float.
"""
from __future__ import annotations

import numpy as np

NCOEFFS = 12
LENGTHS = (4, 5, 8, 12)


def pad(dist) -> np.ndarray:
    """(k1, k2, p1, p2[, k3[, k4, k5, k6[, s1, s2, s3, s4]]]) -> the 12 coefficients, missing ones zero."""
    d = np.asarray(dist, dtype=np.float64).reshape(-1)
    assert d.shape[0] in LENGTHS, d.shape
    return np.concatenate([d, np.zeros(NCOEFFS - d.shape[0])])


def k_valid(K) -> bool:
    K = np.asarray(K, dtype=np.float64).reshape(9)
    return bool(np.isfinite(K).all() and K[0] > 0 and K[4] > 0 and K[6] == 0 and K[7] == 0 and K[8] == 1)


def distort(d, x, y):
    """D1 on normalised (x, y); d the 12 coefficients as scalars of the computation's dtype."""
    one, two = x.dtype.type(1), x.dtype.type(2)
    with np.errstate(all="ignore"):
        r2 = x * x + y * y
        r4 = r2 * r2
        r6 = r4 * r2
        a1 = two * x * y
        a2 = r2 + two * x * x
        a3 = r2 + two * y * y
        cdist = one + d[0] * r2 + d[1] * r4 + d[4] * r6
        icdist2 = one / (one + d[5] * r2 + d[6] * r4 + d[7] * r6)
        xd = x * cdist * icdist2 + d[2] * a1 + d[3] * a2 + d[8] * r2 + d[9] * r4
        yd = y * cdist * icdist2 + d[2] * a3 + d[3] * a1 + d[10] * r2 + d[11] * r4
    return xd, yd


def distort_jacobian(d, x, y):
    """D1's Jacobian [J00, J01, J10, J11] at normalised (x, y), float64 (header step AD3)."""
    with np.errstate(all="ignore"):
        r2 = x * x + y * y
        r4 = r2 * r2
        id_ = 1.0 / (1.0 + d[5] * r2 + d[6] * r4 + d[7] * r2 * r4)
        c = (1.0 + d[0] * r2 + d[1] * r4 + d[4] * r2 * r4) * id_
        dc = (d[0] + 2.0 * d[1] * r2 + 3.0 * d[4] * r4 - c * (d[5] + 2.0 * d[6] * r2 + 3.0 * d[7] * r4)) * id_
        gx = d[8] + 2.0 * d[9] * r2
        gy = d[10] + 2.0 * d[11] * r2
        return [c + 2.0 * x * (x * dc + gx) + 2.0 * d[2] * y + 6.0 * d[3] * x,
                2.0 * y * (x * dc + d[3] + gx) + 2.0 * d[2] * x,
                2.0 * x * (y * dc + d[2] + gy) + 2.0 * d[3] * y,
                c + 2.0 * y * (y * dc + gy) + 6.0 * d[2] * y + 2.0 * d[3] * x]


def _k5(K):
    K = np.asarray(K, dtype=np.float64).reshape(9)
    return K[0], K[1], K[2], K[4], K[5]


def undistort_normalised(K, d, u, v, max_iters: int = 5, eps: float = 0.0):
    """D2: the normalised (x, y) of float64 pixels (u, v) [n], OpenCV's fixed-point iteration point by point (an
    iteration count and EPS stop per point, as the kernel's thread per point runs it)."""
    fx, s, cx, fy, cy = _k5(K)
    with np.errstate(all="ignore"):
        y0 = (v - cy) / fy
        x0 = ((u - cx) - s * y0) / fx
    x, y = x0.copy(), y0.copy()
    err = np.full(u.shape, np.finfo(np.float64).max)
    live = np.ones(u.shape, dtype=bool)
    for _ in range(max_iters):
        live &= ~(err < eps)
        if not live.any():
            break
        with np.errstate(all="ignore"):
            r2 = x * x + y * y
            icdist = (1.0 + ((d[7] * r2 + d[6]) * r2 + d[5]) * r2) / (1.0 + ((d[4] * r2 + d[1]) * r2 + d[0]) * r2)
            neg = live & (icdist < 0.0)
            dx = 2.0 * d[2] * x * y + d[3] * (r2 + 2.0 * x * x) + d[8] * r2 + d[9] * r2 * r2
            dy = d[2] * (r2 + 2.0 * y * y) + 2.0 * d[3] * x * y + d[10] * r2 + d[11] * r2 * r2
            nx, ny = (x0 - dx) * icdist, (y0 - dy) * icdist
        x = np.where(neg, x0, np.where(live, nx, x))
        y = np.where(neg, y0, np.where(live, ny, y))
        live &= ~neg
        if eps > 0.0:
            xd, yd = distort(d, x, y)
            with np.errstate(all="ignore"):
                du = fx * xd + s * yd + cx - u
                dv = fy * yd + cy - v
                err = np.where(live, np.sqrt(du * du + dv * dv), err)
    return x, y


def _pair(kind: str, pts, K, dist, max_iters: int, eps: float) -> np.ndarray:
    pts = np.asarray(pts)
    out = np.full(pts.shape, np.nan, dtype=np.float64)
    d = [np.float64(c) for c in pad(dist)]
    if not (k_valid(K) and np.isfinite(np.asarray(dist, dtype=np.float64)).all()):
        return out.astype(pts.dtype)
    u, v = pts[:, 0].astype(np.float64), pts[:, 1].astype(np.float64)
    ok = np.isfinite(u) & np.isfinite(v)
    u, v = np.where(ok, u, 0.0), np.where(ok, v, 0.0)
    fx, s, cx, fy, cy = _k5(K)
    if kind == "undistort":
        x, y = undistort_normalised(K, d, u, v, max_iters, eps)
    else:
        with np.errstate(all="ignore"):
            y0 = (v - cy) / fy
            x0 = ((u - cx) - s * y0) / fx
        x, y = distort(d, x0, y0)
    with np.errstate(all="ignore"):
        out[:, 0] = np.where(ok, fx * x + s * y + cx, np.nan)
        out[:, 1] = np.where(ok, fy * y + cy, np.nan)
    return out.astype(pts.dtype)


def _batched(kind, pts, K, dist, max_iters, eps) -> np.ndarray:
    pts = np.asarray(pts)
    B = pts.shape[0]
    K = np.broadcast_to(np.asarray(K, dtype=np.float64), (B, 3, 3))
    dist = np.asarray(dist, dtype=np.float64)
    dist = np.broadcast_to(dist, (B, dist.shape[-1]))
    return np.stack([_pair(kind, pts[b], K[b], dist[b], max_iters, eps) for b in range(B)]) if B else pts.copy()


def undistort_points(pts, K, dist, max_iters: int = 5, eps: float = 0.0) -> np.ndarray:
    """[B, N, 2] pixels (float32 or float64), K [3, 3] or [B, 3, 3], dist [k] or [B, k] -> D2's pixels, in the
    input's dtype."""
    return _batched("undistort", pts, K, dist, max_iters, eps)


def distort_points(pts, K, dist) -> np.ndarray:
    """D1 through K of [B, N, 2] undistorted pixels, in the input's dtype."""
    return _batched("distort", pts, K, dist, 0, 0.0)
