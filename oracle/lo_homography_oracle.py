"""numpy restatement of the LO-RANSAC homography of include/geometry_b200.h (geo_homography_lo, steps LH1-LH8,
csrc/lo_hf_api.cu).

The compaction, Hartley normalisation, samples, four-point hypotheses, fp32 transfer errors, denormalisation and
fixed-order sums are geometry_oracle's; the MSAC score is lo_pose_oracle's; the Cholesky step, LM loop and chunk
driver are lo_common's.  What is new here is the Levenberg-Marquardt refinement of the unit-norm normalised homography
on the truncated transfer cost in pixels (double, elementwise operations only, so the CUDA build compiled with
-fmad=false agrees bit for bit) and its tangent basis.
"""
from __future__ import annotations

import math

import numpy as np

from oracle import geometry_oracle as go
from oracle import lo_common as lc
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


def refine(norm, Hn, pts: np.ndarray, thr2: float, steps: int):
    """steps Levenberg-Marquardt steps on the truncated transfer cost from Hn, inliers re-selected at every model."""
    return lc.refine(lambda x: terms(norm, x, pts, thr2), update, [float(v) for v in Hn], DOF, steps, LAMBDA0)


def rescore(norm, Hn, pts: np.ndarray, thr2: np.float32):
    """(H in pixels scaled as step 4, its LH3 score, its count)."""
    with np.errstate(all="ignore"):
        H = go.denormalise(go.HOMOGRAPHY, norm, np.array([Hn]))[0]
    sc, cnt = lpo.score(go.errors(go.HOMOGRAPHY, H[None], pts)[0], thr2)
    return H, int(sc), int(cnt)


def lo_homography_pair(kpts0, kpts1, m0, threshold=3.0, max_iters=2000, confidence=0.995, seed=0) -> dict:
    return lc.lo_hf_pair(go.HOMOGRAPHY, S, "H", normalised_model, refine, rescore, kpts0, kpts1, m0, threshold,
                         max_iters, confidence, seed)


def lo_homography(kpts0, kpts1, matches0, threshold=3.0, max_iters=2000, confidence=0.995, seed=0) -> dict:
    """Batched: [B, M, 2], [B, N, 2], [B, M] -> the outputs of geo_homography_lo as numpy arrays."""
    outs = [lo_homography_pair(kpts0[b], kpts1[b], matches0[b], threshold, max_iters, confidence, seed)
            for b in range(len(matches0))]
    return {k: np.stack([np.asarray(o[k]) for o in outs]) for k in outs[0]}
