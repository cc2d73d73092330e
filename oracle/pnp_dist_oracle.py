"""numpy restatement of the lens distortion of the absolute pose in include/geometry_b200.h (steps AD1-AD4 on A1-A8
and LA1-LA8; geo_absolute_pose_dist in csrc/pnp_api.cu and geo_absolute_pose_lo_dist in csrc/lo_pnp_api.cu).

``camera(K0, dist)`` is the pnp_oracle.Camera that pnp_oracle.absolute_pose_pair and
lo_pnp_oracle.lo_absolute_pose_pair take to run those entry points; everything else is theirs, and the pair functions,
inlier mask and refit below only pass the camera on to them.  What it adds: the
calibrated coordinates of D2 (AD1), the fp32 error in distorted pixels on [R | t] (AD2), and the double residuals and
Jacobian through D1 (AD3), with D1 and D2 from camera_oracle.  Elementwise operations only, so the CUDA build compiled
with -fmad=false agrees bit for bit.

``scene`` draws pnp_oracle's localization scenes seen through a distorting lens.
"""
from __future__ import annotations

import numpy as np

from oracle import camera_oracle as co
from oracle import lo_pnp_oracle as lp
from oracle import pnp_oracle as pp

UNDISTORT_ITERS = 5  # AD1: cv2.solvePnP's undistortion


def scene(m: int, outliers: float, seed: int, dist, **kw):
    """pnp_oracle.localization_scene(m, outliers, seed, **kw) with every query pixel moved through the lens: K^-1,
    D1 with the coefficients dist, then K.  Returns the same tuple."""
    kpts0, pts3d, matches0, truth, K, R, t = pp.localization_scene(m, outliers, seed, **kw)
    kpts0 = co.distort_points(kpts0[None].astype(np.float64), K, dist)[0].astype(kpts0.dtype)
    return kpts0, pts3d, matches0, truth, K, R, t


def camera_valid(K, dist) -> bool:
    """A8 and AD1: K0 valid, and the coefficients all finite."""
    return pp.k_valid(K) and bool(np.isfinite(np.asarray(dist, dtype=np.float64)).all())


def bearings(K, pix: np.ndarray, dist) -> np.ndarray:
    """AD1: the fp32 calibrated coordinates P3P reads, D2's with 5 iterations and no EPS stop."""
    x, y = co.undistort_normalised(K, [np.float64(c) for c in co.pad(dist)], pix[:, 0].astype(np.float64),
                                   pix[:, 1].astype(np.float64), UNDISTORT_ITERS, 0.0)
    return np.stack([x, y], 1).astype(np.float32)


def model(R: np.ndarray, t: np.ndarray) -> np.ndarray:
    """M = [R | t] [..., 12] row-major: the model AD2 rounds to float."""
    return np.stack([R[..., 3 * i + j] if j < 3 else t[..., i] for i in range(3) for j in range(4)], -1)


def errors(M: np.ndarray, pix: np.ndarray, wld: np.ndarray, K, dist) -> np.ndarray:
    """AD2's fp32 errors [H, n] of models M [H, 12] (cast to fp32): du*du + dv*dv in distorted pixels in front of the
    camera, +inf behind it."""
    g = [M.astype(np.float32)[:, i:i + 1] for i in range(12)]
    Kf = np.asarray(K, dtype=np.float64).reshape(9).astype(np.float32)
    fx, s, cx, fy, cy = Kf[0], Kf[1], Kf[2], Kf[4], Kf[5]
    d = [np.float32(c) for c in co.pad(dist)]
    u, v = pix[None, :, 0], pix[None, :, 1]
    X, Y, Z = wld[None, :, 0], wld[None, :, 1], wld[None, :, 2]
    with np.errstate(all="ignore"):
        X0 = g[0] * X + g[1] * Y + g[2] * Z + g[3]
        X1 = g[4] * X + g[5] * Y + g[6] * Z + g[7]
        w = g[8] * X + g[9] * Y + g[10] * Z + g[11]
        xd, yd = co.distort(d, X0 / w, X1 / w)
        du = u - (fx * xd + s * yd + cx)
        dv = v - (fy * yd + cy)
        return np.where(w > 0.0, du * du + dv * dv, np.float32(np.inf))


def residuals(x, K, pix: np.ndarray, wld: np.ndarray, dist):
    """AD3 at x = R (9, row-major) + t (3): double residuals (ru, rv) in distorted pixels, errors ru*ru + rv*rv, depths
    Xc2 and the Jacobian rows ju, jv [6, n] (pnp_oracle.residuals' layout)."""
    R, t = x[:9], x[9:]
    K = np.asarray(K, dtype=np.float64).reshape(9)
    fx, s, cx, fy, cy = (float(K[i]) for i in (0, 1, 2, 4, 5))
    d = [np.float64(c) for c in co.pad(dist)]
    u, v = pix[:, 0].astype(np.float64), pix[:, 1].astype(np.float64)
    W = [wld[:, i].astype(np.float64) for i in range(3)]
    with np.errstate(all="ignore"):
        Xc = [R[3 * i] * W[0] + R[3 * i + 1] * W[1] + R[3 * i + 2] * W[2] + t[i] for i in range(3)]
        iz = 1.0 / Xc[2]
        a, b = Xc[0] * iz, Xc[1] * iz
        xd, yd = co.distort(d, a, b)
        ru, rv = fx * xd + s * yd + cx - u, fy * yd + cy - v
        J = co.distort_jacobian(d, a, b)
        ua, ub, va, vb = fx * J[0] + s * J[2], fx * J[1] + s * J[3], fy * J[2], fy * J[3]
        gu = [ua * iz, ub * iz, -((ua * a + ub * b) * iz)]
        gv = [va * iz, vb * iz, -((va * a + vb * b) * iz)]

        def jrow(g):
            return [g[2] * Xc[1] - g[1] * Xc[2], g[0] * Xc[2] - g[2] * Xc[0], g[1] * Xc[0] - g[0] * Xc[1],
                    g[0], g[1], g[2]]
        ju, jv = np.stack(jrow(gu)), np.stack(jrow(gv))
        err = ru * ru + rv * rv
    return ru, rv, err, Xc[2], ju, jv


def camera(K, dist) -> pp.Camera:
    """The camera K with the coefficients dist, for the pair loops of both estimators."""
    K = np.asarray(K, dtype=np.float64).reshape(9)
    return pp.Camera(camera_valid(K, dist), lambda pix: bearings(K, pix, dist), model,
                     lambda M, pix, wld: errors(M, pix, wld, K, dist),
                     lambda x, pix, wld: residuals(x, K, pix, wld, dist))


def inliers(M: np.ndarray, pix: np.ndarray, wld: np.ndarray, thr2: np.float32, K, dist) -> np.ndarray:
    """AD2's inlier masks [H, n] of models M [H, 12]: w > 0 and err < thr2."""
    return pp.inliers(camera(K, dist), M, pix, wld, thr2)


def refine_lm(R, t, K, pix, wld, inl, dist):
    """A7's GEO_PNP_LM_STEPS Levenberg-Marquardt steps on AD3's squared error of the fixed inliers inl, from (R, t)."""
    return pp.refine_lm(R, t, K, pix, wld, inl, camera(K, dist))


def absolute_pose_pair(kpts0, points3d1, m0, K0, threshold, max_iters, confidence, seed, dist) -> dict:
    """One pair of geo_absolute_pose_dist."""
    return pp.absolute_pose_pair(kpts0, points3d1, m0, K0, threshold, max_iters, confidence, seed, camera(K0, dist))


def lo_absolute_pose_pair(kpts0, points3d1, m0, K0, threshold, max_iters, confidence, seed, dist) -> dict:
    """One pair of geo_absolute_pose_lo_dist."""
    return lp.lo_absolute_pose_pair(kpts0, points3d1, m0, K0, threshold, max_iters, confidence, seed, camera(K0, dist))
