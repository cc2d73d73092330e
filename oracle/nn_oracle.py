"""The nearest-neighbour matcher's semantics (include/nn_b200.h) in float64 numpy.

``match`` restates the rules row by row: the nearest neighbour is the lowest index among the maxima, the second best is
the largest similarity over every other column, and the ratio and distance tests compare squared distances
D = 2 (1 - s) with r^2 and t^2 rounded to float as the device forms them.  Besides the outputs it returns, per side,
the margins of each row's decisions (top-1 gap, ratio and distance), so a test against the split-bf16 device path can
leave out the rows whose decision the rounding could flip.
"""
from __future__ import annotations

import numpy as np


def thresholds(ratio_thresh, distance_thresh):
    """(r2, t2) as the device uses them: the threshold as the float the config holds, squared in double, rounded to
    float; None when the test is off."""
    def sq(v):
        if v is None:
            return None
        x = float(np.float32(v))
        return float(np.float32(x * x))
    return sq(ratio_thresh), sq(distance_thresh)


def one_way(S: np.ndarray, r2, t2) -> dict:
    """One direction on the similarity block S [rows, cols] (float64): j1, s1, s2, D1, D2, keep and the margins."""
    rows, cols = S.shape
    out = {k: np.zeros(rows) for k in ("s1", "s2", "d1", "d2", "gap", "ratio_margin", "dist_margin")}
    out["j1"] = np.full(rows, -1, dtype=np.int64)
    out["keep"] = np.zeros(rows, dtype=bool)
    for i in range(rows):
        if cols == 0:
            out["s1"][i] = out["s2"][i] = -np.inf
            out["gap"][i] = out["ratio_margin"][i] = out["dist_margin"][i] = np.inf
            continue
        row = S[i]
        best = row.max()
        j1 = int(np.flatnonzero(row == best)[0])  # the lowest j among the maxima
        others = np.delete(row, j1)
        s2 = others.max() if others.size else -np.inf
        d1 = 2.0 * (1.0 - best)
        d2 = 2.0 * (1.0 - s2) if s2 != -np.inf else np.inf
        keep = True
        if r2 is not None:
            keep &= d1 <= r2 * d2
        if t2 is not None:
            keep &= d1 <= t2
        out["j1"][i], out["s1"][i], out["s2"][i], out["d1"][i], out["d2"][i] = j1, best, s2, d1, d2
        out["keep"][i] = keep
        out["gap"][i] = best - s2
        out["ratio_margin"][i] = abs(d1 - r2 * d2) if r2 is not None and d2 != np.inf else np.inf
        out["dist_margin"][i] = abs(d1 - t2) if t2 is not None else np.inf
    return out


def match(desc0, desc1, lens0=None, lens1=None, ratio_thresh=None, distance_thresh=None, mutual_check=True) -> dict:
    """desc0 [B, M, D], desc1 [B, N, D] (any float array) -> matches0 [B, M], matches1 [B, N] int64,
    matching_scores0 / 1 float32, matches / scores lists per pair, and ``sides[b] = (one_way 0->1, one_way 1->0)``."""
    d0 = np.asarray(desc0, dtype=np.float64)
    d1 = np.asarray(desc1, dtype=np.float64)
    B, M, _ = d0.shape
    N = d1.shape[1]
    r2, t2 = thresholds(ratio_thresh, distance_thresh)
    m0 = np.full((B, M), -1, dtype=np.int64)
    m1 = np.full((B, N), -1, dtype=np.int64)
    sc0 = np.zeros((B, M), dtype=np.float32)
    sc1 = np.zeros((B, N), dtype=np.float32)
    matches, scores, sides = [], [], []
    for b in range(B):
        m = M if lens0 is None else int(min(max(int(lens0[b]), 0), M))
        n = N if lens1 is None else int(min(max(int(lens1[b]), 0), N))
        S = d0[b, :m] @ d1[b, :n].T if m and n else np.zeros((m, n))
        a, c = one_way(S, r2, t2), one_way(S.T, r2, t2)  # an empty side keeps nothing
        for i in range(m):
            j = int(a["j1"][i])
            if a["keep"][i] and (not mutual_check or (c["keep"][j] and c["j1"][j] == i)):
                m0[b, i] = j
                sc0[b, i] = np.float32((a["s1"][i] + 1.0) / 2.0)
        for j in range(n):
            i = int(c["j1"][j])
            if c["keep"][j] and (not mutual_check or (a["keep"][i] and a["j1"][i] == j)):
                m1[b, j] = i
                sc1[b, j] = np.float32((c["s1"][j] + 1.0) / 2.0)
        rows = np.flatnonzero(m0[b] >= 0)
        matches.append(np.stack([rows, m0[b, rows]], axis=1).astype(np.int64).reshape(-1, 2))
        scores.append(sc0[b, rows])
        sides.append((a, c))
    return {"matches0": m0, "matches1": m1, "matching_scores0": sc0, "matching_scores1": sc1, "matches": matches,
            "scores": scores, "sides": sides}


def decided(res: dict, b: int, side: int, tol_s: float, tol_d: float, mutual_check: bool) -> np.ndarray:
    """Rows of pair b on `side` whose outcome no perturbation of the similarities below tol_s (tol_d on D) can change:
    the row's own top-1 gap and test margins are above the tolerances, and with the mutual check also those of the row
    it names on the other side."""
    a, c = res["sides"][b] if side == 0 else res["sides"][b][::-1]

    def own(o):
        return (o["gap"] > tol_s) & (o["ratio_margin"] > tol_d) & (o["dist_margin"] > tol_d)

    ok = own(a)
    if mutual_check and len(c["j1"]):
        partner_ok = own(c)
        j = a["j1"]
        ok &= np.where(j >= 0, partner_ok[np.clip(j, 0, len(partner_ok) - 1)], True)
    return ok
