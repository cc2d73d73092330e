"""Guided nearest-neighbour matching (include/nn_b200.h, ``nn_match_guided``) in float64 numpy.

``gate`` is the guided gate: step 5 of include/geometry_b200.h, the estimators' fp32 inlier error
(``geometry_oracle.errors``), below max_error^2 rounded to float; the device reproduces it bit for bit.  ``match`` takes
that bool mask [B, M, N] and restates nn_oracle.match's rules over the gated columns of each row only: the nearest
neighbour is the lowest gated index among the maxima, the second best the largest similarity over the other gated
columns (-inf when there are none), and a row with no gated column matches nothing.  Its result has nn_oracle.match's
keys and ``sides``, so ``nn_oracle.decided`` applies to it unchanged; the margins are over gated columns only.  With
``gate=None`` it is nn_oracle.match.  ``chunk_gate`` builds the same gate a block of rows at a time in torch, for
nn_oracle.match_chunked.
"""
from __future__ import annotations

import numpy as np
import torch

from . import geometry_oracle as geo
from . import nn_oracle


def gate(kind, model, kpts0, kpts1, max_error, valid=None) -> np.ndarray:
    """The guided gate [B, M, N] (bool): err(i, j) < (float)(max_error^2) with err the estimators' float32 error of
    model[b] ([B, 3, 3] or [B, 9]; kind geometry_oracle.HOMOGRAPHY or FUNDAMENTAL) on kpts0[b, i], kpts1[b, j].  A NaN
    error fails.  All True for a pair with valid[b] == 0."""
    model = np.asarray(model, dtype=np.float64).reshape(len(model), 9)
    k0 = np.asarray(kpts0, dtype=np.float32)
    k1 = np.asarray(kpts1, dtype=np.float32)
    B, M, N = k0.shape[0], k0.shape[1], k1.shape[1]
    t2 = np.float32(float(max_error) * float(max_error))
    out = np.ones((B, M, N), dtype=bool)
    for b in range(B):
        if valid is not None and not valid[b]:
            continue
        pts = np.concatenate([np.repeat(k0[b], N, axis=0), np.tile(k1[b], (M, 1))], axis=1)
        with np.errstate(invalid="ignore"):
            out[b] = (geo.errors(kind, model[b:b + 1], pts)[0] < t2).reshape(M, N)
    return out


def one_way(S: np.ndarray, r2, t2, G: np.ndarray | None = None) -> dict:
    """nn_oracle.one_way over the gated columns: with a gate G [rows, cols] only the gated columns of a row compete,
    and the margins are over them alone; a row with no gated column keeps nothing (j1 = -1, s1 = s2 = -inf, infinite
    margins: nothing can change its outcome).  G None: every column, as nn_oracle.one_way."""
    if G is None:
        return nn_oracle.one_way(S, r2, t2)
    rows, cols = S.shape
    out = {k: np.zeros(rows) for k in ("s1", "s2", "d1", "d2", "gap", "ratio_margin", "dist_margin")}
    out["j1"] = np.full(rows, -1, dtype=np.int64)
    out["keep"] = np.zeros(rows, dtype=bool)
    for i in range(rows):
        live = np.flatnonzero(G[i])
        if live.size == 0:
            out["s1"][i] = out["s2"][i] = -np.inf
            out["gap"][i] = out["ratio_margin"][i] = out["dist_margin"][i] = np.inf
            continue
        # the gated columns in ascending order: nn_oracle.one_way's rules on them, mapped back to column indices
        o = nn_oracle.one_way(S[i:i + 1, live], r2, t2)
        for k in out:
            out[k][i] = o[k][0]
        out["j1"][i] = live[o["j1"][0]]
    return out


def block_errors(kind, model9, x0, x1):
    """geometry_oracle.errors of one model ([9] float64 torch) on every (x0[i], x1[j]), x0 [m, 2] and x1 [n, 2] fp32
    torch on one device -> [m, n] fp32: the same fp32 operations in the same order, each a separate eager op, so each
    is rounded on its own as numpy rounds it."""
    g = model9.float()
    one = torch.ones((), dtype=torch.float32, device=g.device)
    a0, b0 = x0[:, 0:1], x0[:, 1:2]  # [m, 1]
    a1, b1 = x1[None, :, 0], x1[None, :, 1]  # [1, n]
    if kind == geo.HOMOGRAPHY:
        w = one / ((g[6] * a0 + g[7] * b0) + g[8])
        dx = a1 - ((g[0] * a0 + g[1] * b0) + g[2]) * w
        dy = b1 - ((g[3] * a0 + g[4] * b0) + g[5]) * w
        return dx * dx + dy * dy
    la, lb, lc = (g[0] * a0 + g[1] * b0) + g[2], (g[3] * a0 + g[4] * b0) + g[5], (g[6] * a0 + g[7] * b0) + g[8]
    d2, s2 = (a1 * la + b1 * lb) + lc, one / (la * la + lb * lb)
    la, lb, lc = (g[0] * a1 + g[3] * b1) + g[6], (g[1] * a1 + g[4] * b1) + g[7], (g[2] * a1 + g[5] * b1) + g[8]
    d1, s1 = (a0 * la + b0 * lb) + lc, one / (la * la + lb * lb)
    return torch.fmax(d1 * d1 * s1, d2 * d2 * s2)


def chunk_gate(kind, model, kpts0, kpts1, max_error, valid=None, lens0=None, lens1=None, device="cpu"):
    """``gate`` for nn_oracle.match_chunked: a function (b, side, r0, r1) -> the bool gate [r1 - r0, partner length] of
    rows r0 .. r1 - 1 of pair b's image `side`, built on `device` with fp32 torch ops (block_errors), bit for bit
    ``gate``'s; None (every column) for a pair with valid[b] == 0."""
    model = torch.as_tensor(np.asarray(model, dtype=np.float64)).reshape(-1, 9).to(device)
    k0 = torch.as_tensor(np.asarray(kpts0, dtype=np.float32)).to(device)
    k1 = torch.as_tensor(np.asarray(kpts1, dtype=np.float32)).to(device)
    M, N = k0.shape[1], k1.shape[1]
    t2 = torch.tensor(float(np.float32(float(max_error) * float(max_error))), dtype=torch.float32, device=device)

    def fn(b, side, r0, r1):
        if valid is not None and not valid[b]:
            return None
        m = nn_oracle._pair_len(lens0, b, M)
        n = nn_oracle._pair_len(lens1, b, N)
        if side == 0:
            return block_errors(kind, model[b], k0[b, r0:r1], k1[b, :n]) < t2  # NaN fails
        return (block_errors(kind, model[b], k0[b, :m], k1[b, r0:r1]) < t2).T
    return fn


def match(desc0, desc1, lens0=None, lens1=None, ratio_thresh=None, distance_thresh=None, mutual_check=True,
          gate=None, split=False) -> dict:
    """nn_oracle.match with the gate [B, M, N] bool (see ``gate``) restricting both sides to the gated pairs (i, j);
    gate None: nn_oracle.match itself.  split: s from the device's split-bf16 products, as nn_oracle.match."""
    if gate is None:
        return nn_oracle.match(desc0, desc1, lens0, lens1, ratio_thresh, distance_thresh, mutual_check, split)
    d0 = np.asarray(desc0, dtype=np.float64)
    d1 = np.asarray(desc1, dtype=np.float64)
    B, M, _ = d0.shape
    N = d1.shape[1]
    r2, t2 = nn_oracle.thresholds(ratio_thresh, distance_thresh)
    m0 = np.full((B, M), -1, dtype=np.int64)
    m1 = np.full((B, N), -1, dtype=np.int64)
    sc0 = np.zeros((B, M), dtype=np.float32)
    sc1 = np.zeros((B, N), dtype=np.float32)
    matches, scores, sides = [], [], []
    for b in range(B):
        m = M if lens0 is None else int(min(max(int(lens0[b]), 0), M))
        n = N if lens1 is None else int(min(max(int(lens1[b]), 0), N))
        S = nn_oracle.similarity(d0[b, :m], d1[b, :n], split) if m and n else np.zeros((m, n))
        G = np.asarray(gate[b], dtype=bool)[:m, :n]
        a, c = one_way(S, r2, t2, G), one_way(S.T, r2, t2, G.T)  # an empty side keeps nothing
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


decided = nn_oracle.decided  # works on this match's result unchanged
