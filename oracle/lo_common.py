"""numpy restatement of csrc/geo_lm.cuh and lo_common.cuh: the damped Cholesky step and A7's quaternion rotation that
every Levenberg-Marquardt refinement takes, the LM loop of the LO-RANSAC estimators (header steps L7, LH7, LF7 and
LA7), the schedule of L4-L6 that they all run (LH, LF and LA likewise), and the pair of the LO-RANSAC homography and
fundamental matrix (steps LH1-LH8 and LF1-LF8).

Python floats and elementwise numpy only, so the CUDA build compiled with -fmad=false agrees bit for bit.
"""
from __future__ import annotations

import math

import numpy as np

from oracle import geometry_oracle as go
from oracle import lo_pose_oracle as lpo


def lm_solve(h, g, lam, n):
    """delta of (H, its diagonal times (1 + lam)) delta = -g by Cholesky for an n x n system (header step A7), H given
    by its row-major upper triangle h; None on a pivot <= 0 or a non-finite delta."""
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


def quat_rotation(d):
    """A7's row-major rotation of the unit quaternion (1, d0/2, d1/2, d2/2) / norm."""
    qw, qx, qy, qz = 1.0, d[0] * 0.5, d[1] * 0.5, d[2] * 0.5
    n = math.sqrt(qw * qw + qx * qx + qy * qy + qz * qz)
    qw, qx, qy, qz = qw / n, qx / n, qy / n, qz / n
    return [1.0 - 2.0 * (qy * qy + qz * qz), 2.0 * (qx * qy - qw * qz), 2.0 * (qx * qz + qw * qy),
            2.0 * (qx * qy + qw * qz), 1.0 - 2.0 * (qx * qx + qz * qz), 2.0 * (qy * qz - qw * qx),
            2.0 * (qx * qz - qw * qy), 2.0 * (qy * qz + qw * qx), 1.0 - 2.0 * (qx * qx + qy * qy)]


def refine(terms, update, x, dof, steps: int, lam0: float):
    """steps Levenberg-Marquardt steps on a cost from the model x.  terms(x) gives its fixed-order sums: the J^T J upper
    triangle, J^T r (dof each) and the cost last; update(x, d) the candidate of the step d.  A candidate is taken when
    its cost is lower; the damping starts at lam0 and falls or rises tenfold."""
    nh = dof * (dof + 1) // 2
    sums = terms(x)
    lam = lam0
    for _ in range(steps):
        d = lm_solve(sums[:nh], sums[nh:nh + dof], lam, dof)
        if d is None:
            lam = lam * 10.0
            continue
        cand = update(x, d)
        cs = terms(cand)
        if cs[-1] < sums[-1]:
            x, sums = cand, cs
            lam = lam / 10.0
        else:
            lam = lam * 10.0
    return x


def lo_pair(n, s, max_iters, confidence, candidates, refine, rescore, restore=None):
    """L4-L6 of one pair of n points and s points per sample.  candidates(h) gives the valid solutions of the samples h
    in (sample, solution) order as (scores, counts, samples, solution indices, seed), or None without one; seed(i) is
    the model of solution i.  refine(model, steps) gives the LM result of steps steps from a model and rescore(x) the
    (model, score, count) of an LM result.  After the final refinement, a score above the pair's gives restore(model,
    score, count) of the pair's model (default: as it is).  Returns ((h, r, model, score, count) or None, local
    optimisations adopted, samples drawn)."""
    best, nlo, drawn = None, 0, 0  # best: (score, count, h, r, model)
    for c in range(-(-max_iters // go.CHUNK)):
        h = np.arange(c * go.CHUNK, min((c + 1) * go.CHUNK, max_iters), dtype=np.int64)
        cands = candidates(h)
        if cands is not None:
            sc, cnt, hs, rs, seed = cands
            i = int(np.argmin(sc))  # first minimum: the lowest (sample, solution)
            if best is None or sc[i] < best[0]:
                best = (int(sc[i]), int(cnt[i]), int(hs[i]), int(rs[i]), seed(i))
                model, sl, cl = rescore(refine(best[4], lpo.STEPS))
                if sl < best[0]:
                    best = (sl, cl, best[2], best[3], model)
                    nlo += 1
        drawn = min((c + 1) * go.CHUNK, max_iters)
        ep = 1.0 - (best[1] if best else 0) / n
        if drawn >= max_iters or drawn >= go.update_num_iters(confidence, ep, s, max_iters):
            break
    if best is None:
        return None, nlo, drawn
    model, cost, count = rescore(refine(best[4], lpo.FINAL_STEPS))
    if cost > best[0]:  # the refinement is kept unless its score rises
        model, cost, count = (restore or (lambda *m: m))(best[4], best[0], best[1])
    return (best[2], best[3], model, cost, count), nlo, drawn


def lo_hf_pair(kind, s, key, start, refine_model, rescore, kpts0, kpts1, m0, threshold, max_iters, confidence,
               seed) -> dict:
    """One pair of the LO-RANSAC homography (LH1-LH8) or fundamental matrix (LF1-LF8), kind and s its step 4 model and
    sample size, key the output name of the model.  start(norm, model) is the LM start of a pixel model,
    refine_model(norm, x, pts, thr2, steps) its LM and rescore(norm, x, pts, thr2) its (pixel model, score, count)."""
    kpts0 = np.asarray(kpts0, dtype=np.float32)
    kpts1 = np.asarray(kpts1, dtype=np.float32)
    m0 = np.asarray(m0, dtype=np.int64)
    M = m0.shape[0]
    thr2 = np.float32(threshold * threshold)
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
        sc, cnt = lpo.score(go.errors(kind, models[ok], pts), thr2)
        return sc, cnt, h[ok], np.zeros(len(sc), dtype=np.int64), lambda i: models[ok][i]

    found, nlo, drawn = lo_pair(n, s, max_iters, confidence, candidates,
                                lambda model, steps: refine_model(norm, start(norm, model), pts, float(thr2), steps),
                                lambda x: rescore(norm, x, pts, thr2))
    if found is None:
        return dict(fail, num_hypotheses=drawn)
    h, _, model, cost, count = found
    inliers = np.zeros(M, dtype=bool)
    inliers[idx[go.errors(kind, model[None], pts)[0] < thr2]] = True
    return {key: model.reshape(3, 3), "inliers": inliers, "num_inliers": count, "success": True,
            "best_hypothesis": h, "num_hypotheses": drawn, "num_local_optimizations": nlo, "cost": cost}
