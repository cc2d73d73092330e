"""numpy restatement of the MAGSAC++ homography and fundamental matrix of include/geometry_b200.h
(geo_homography_magsac and geo_fundamental_magsac, steps MH1-MH8 and MF1-MF8, csrc/lo_hf_api.cu and the Magsac loss of
csrc/lo_common.cuh).

Everything but the loss is the LO-RANSAC oracles': compaction, normalisation, samples and hypotheses are
geometry_oracle's, the residuals, Jacobians and LM updates lo_homography_oracle's and lo_fundamental_oracle's, and the
LM loop and chunk schedule lo_common's.  What is new here is the MAGSAC++ score (MH3, fp32) and the weighted LM sums
(MH7, double), both read from the tables of csrc/magsac_table.h by linear interpolation; the tables are parsed from
that header, so this module needs no scipy.  Elementwise numpy only, so the CUDA build compiled with -fmad=false agrees
bit for bit.
"""
from __future__ import annotations

import os
import re

import numpy as np

from oracle import geometry_oracle as go
from oracle import lo_common as lc
from oracle import lo_fundamental_oracle as lf
from oracle import lo_homography_oracle as lh

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "lightglue_b200", "csrc",
                      "magsac_table.h")
QSCALE = lh.QSCALE


def _parse(path: str):
    text = open(path).read()
    out = {}
    for name in ("MAGSAC_RHO", "MAGSAC_W"):
        body = re.search(name + r"\[[^\]]*\]\s*=\s*\{([^}]*)\}", text).group(1)
        out[name] = np.array([float.fromhex(v.strip()) for v in body.split(",") if v.strip()], dtype=np.float64)
    return out["MAGSAC_RHO"], out["MAGSAC_W"]


RHO, W = _parse(HEADER)
KNOTS = len(RHO) - 1
RHO32 = RHO.astype(np.float32)


def mt2_of(max_threshold) -> np.float32:
    """mt2 = (float)(T * T)."""
    return np.float32(float(max_threshold) * float(max_threshold))


def score_terms(err, thr2, mt2) -> np.ndarray:
    """MH3's q of each fp32 err (uint64), without the count."""
    e = np.asarray(err, dtype=np.float32)
    ks = np.float32(KNOTS) / np.float32(mt2)
    with np.errstate(all="ignore"):
        u = e * ks
        inside = u < np.float32(KNOTS)
        i = np.where(inside, u, np.float32(0.0)).astype(np.int64)
        f = u - i.astype(np.float32)
        r = RHO32[i] + f * (RHO32[i + 1] - RHO32[i])
        q = np.minimum(r * np.float32(QSCALE), np.float32(QSCALE))
        return np.where(inside, q, np.float32(QSCALE)).astype(np.uint64)


def score(err, thr2, mt2):
    """MH3 / MF3 of errors [..., n]: (score, count), summed over the last axis."""
    e = np.asarray(err, dtype=np.float32)
    return score_terms(e, thr2, mt2).sum(-1, dtype=np.uint64), (e < np.float32(thr2)).sum(-1)


def loss(err, mt2: float):
    """MH7's (inside, cost, weight) of double errors at the scale mt2 (a double)."""
    err = np.asarray(err, dtype=np.float64)
    with np.errstate(all="ignore"):
        u = err * (float(KNOTS) / mt2)
        inside = u < float(KNOTS)
        i = np.where(inside, u, 0.0).astype(np.int64)
        f = u - i.astype(np.float64)
        cost = np.where(inside, RHO[i] + f * (RHO[i + 1] - RHO[i]), 1.0)
        wt = np.where(inside, W[i] + f * (W[i + 1] - W[i]), 0.0)
    return inside, cost, wt


def h_terms(norm, Hn, pts: np.ndarray, mt2: float) -> np.ndarray:
    """The 45 fixed-order sums at Hn (MH7): every point within T adds its weighted J^T J and J^T r, every point its
    loss."""
    dx, dy, err, jx, jy = lh.residuals(norm, Hn, pts)
    inl, cost, wt = loss(err, mt2)
    rows = []
    with np.errstate(all="ignore"):
        for i in range(lh.DOF):
            for j in range(i, lh.DOF):
                rows.append(np.where(inl, wt * (jx[i] * jx[j] + jy[i] * jy[j]), 0.0))
        for i in range(lh.DOF):
            rows.append(np.where(inl, wt * (jx[i] * dx + jy[i] * dy), 0.0))
    rows.append(cost)
    return go.fixed_sum(np.stack(rows))


def f_terms(norm, U, V, sig, pts: np.ndarray, mt2: float) -> np.ndarray:
    """The 36 fixed-order sums at (U, V, sig) (MF7), weighted as h_terms."""
    r, err, J = lf.residuals(norm, U, V, sig, pts)
    inl, cost, wt = loss(err, mt2)
    rows = []
    with np.errstate(all="ignore"):
        for i in range(lf.DOF):
            for j in range(i, lf.DOF):
                rows.append(np.where(inl, wt * (J[i] * J[j]), 0.0))
        for i in range(lf.DOF):
            rows.append(np.where(inl, wt * (J[i] * r), 0.0))
    rows.append(cost)
    return go.fixed_sum(np.stack(rows))


def h_refine(norm, Hn, pts, mt2: float, steps: int):
    return lc.refine(lambda x: h_terms(norm, x, pts, mt2), lh.update, [float(v) for v in Hn], lh.DOF, steps,
                     lh.LAMBDA0)


def f_refine(norm, model, pts, mt2: float, steps: int):
    x = [float(v) for v in model[0]], [float(v) for v in model[1]], float(model[2])
    return lc.refine(lambda m: f_terms(norm, *m, pts, mt2), lambda m, d: lf.update(*m, d), x, lf.DOF, steps,
                     lh.LAMBDA0)


def _pixels(kind, norm, x):
    with np.errstate(all="ignore"):
        return go.denormalise(kind, norm, np.array([x if kind == go.HOMOGRAPHY else lf.compose(*x)]))[0]


def magsac_hf_pair(kind, kpts0, kpts1, m0, threshold, max_threshold, max_iters, confidence, seed) -> dict:
    """One pair of MH1-MH8 (kind go.HOMOGRAPHY) or MF1-MF8 (go.FUNDAMENTAL): lo_common.lo_hf_pair with the loss
    replaced."""
    s, key = (lh.S, "H") if kind == go.HOMOGRAPHY else (lf.S, "F")
    start = lh.normalised_model if kind == go.HOMOGRAPHY else lf.start
    refine = h_refine if kind == go.HOMOGRAPHY else f_refine
    kpts0 = np.asarray(kpts0, dtype=np.float32)
    kpts1 = np.asarray(kpts1, dtype=np.float32)
    m0 = np.asarray(m0, dtype=np.int64)
    M = m0.shape[0]
    thr2 = np.float32(threshold * threshold)
    mt2 = mt2_of(max_threshold)
    idx, pts = go.compact(kpts0, kpts1, m0)
    n = pts.shape[0]
    norm = go.normalisation(pts) if n >= s else None
    fail = {key: np.zeros((3, 3)), "inliers": np.zeros(M, dtype=bool), "num_inliers": 0, "success": False,
            "best_hypothesis": -1, "num_hypotheses": 0, "num_local_optimizations": 0, "cost": 0}
    if norm is None:
        return fail

    def candidates(h):
        models, ok = go.hypotheses(kind, seed, h, pts, norm)
        if not ok.any():
            return None
        sc, cnt = score(go.errors(kind, models[ok], pts), thr2, mt2)
        return sc, cnt, h[ok], np.zeros(len(sc), dtype=np.int64), lambda i: models[ok][i]

    def rescore(x):
        model = _pixels(kind, norm, x)
        sc, cnt = score(go.errors(kind, model[None], pts)[0], thr2, mt2)
        return model, int(sc), int(cnt)

    found, nlo, drawn = lc.lo_pair(n, s, max_iters, confidence, candidates,
                                   lambda model, steps: refine(norm, start(norm, model), pts, float(mt2), steps),
                                   rescore)
    if found is None:
        return dict(fail, num_hypotheses=drawn)
    h, _, model, cost, count = found
    inliers = np.zeros(M, dtype=bool)
    inliers[idx[go.errors(kind, model[None], pts)[0] < thr2]] = True
    return {key: model.reshape(3, 3), "inliers": inliers, "num_inliers": count, "success": True,
            "best_hypothesis": h, "num_hypotheses": drawn, "num_local_optimizations": nlo, "cost": cost}


def magsac_homography_pair(kpts0, kpts1, m0, threshold=3.0, max_threshold=7.5, max_iters=2000, confidence=0.995,
                           seed=0) -> dict:
    return magsac_hf_pair(go.HOMOGRAPHY, kpts0, kpts1, m0, threshold, max_threshold, max_iters, confidence, seed)


def magsac_fundamental_pair(kpts0, kpts1, m0, threshold=3.0, max_threshold=7.5, max_iters=1000, confidence=0.99,
                            seed=0) -> dict:
    return magsac_hf_pair(go.FUNDAMENTAL, kpts0, kpts1, m0, threshold, max_threshold, max_iters, confidence, seed)
