"""The nearest-neighbour matcher's semantics (include/nn_b200.h) in float64 numpy, and the same rules vectorised in torch.

``match`` restates the rules row by row: the nearest neighbour is the lowest index among the maxima, the second best is
the largest similarity over every other column, and the ratio and distance tests compare squared distances
D = 2 (1 - s) with r^2 and t^2 rounded to float as the device forms them; D1, D2, the product r^2 D2 and the
comparisons are fp32, as the header says.  Besides the outputs it returns, per side, the margins of each row's decisions
(top-1 gap, ratio and distance, in float64), so a test against the split-bf16 device path can leave out the rows whose
decision the rounding could flip.

``split=True`` takes s from the device's split instead of the exact dot product: hi = bf16_rn(d), lo = bf16_rn(d - hi)
and s = hi0 . hi1 + hi0 . lo1 + lo0 . hi1 in float64 (lo0 . lo1 dropped).  ``match_chunked`` is ``match`` in torch,
float64 on any device, one block of rows at a time, for shapes the row loop cannot afford.
"""
from __future__ import annotations

import numpy as np
import torch


def thresholds(ratio_thresh, distance_thresh):
    """(r2, t2) as the device uses them: the threshold as the float the config holds, squared in double, rounded to
    float; None when the test is off."""
    def sq(v):
        if v is None:
            return None
        x = float(np.float32(v))
        return float(np.float32(x * x))
    return sq(ratio_thresh), sq(distance_thresh)


def split(d):
    """(hi, lo) of the device's split (tc_split in lightglue_b200/csrc/lg_tc.h) as float64 arrays: hi = bf16_rn(d),
    lo = bf16_rn(d - hi), with d rounded to fp32 first.  torch's bf16 conversion rounds to nearest even, as
    __float2bfloat16_rn does; d - hi is exact in fp32."""
    d = torch.as_tensor(np.asarray(d, dtype=np.float32))
    hi = d.bfloat16().float()
    lo = (d - hi).bfloat16().float()
    return hi.double().numpy(), lo.double().numpy()


def similarity(a, b, split_bf16=False):
    """s = a b^T in float64 ([m, D] x [n, D]); split_bf16: the three products of the device's split."""
    if not split_bf16:
        return a @ b.T
    ah, al = split(a)
    bh, bl = split(b)
    return ah @ bh.T + ah @ bl.T + al @ bh.T


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
        f1, f2 = np.float32(d1), np.float32(d2)  # the header's fp32 D1, D2
        keep = True
        if r2 is not None:
            keep &= bool(f1 <= np.float32(np.float32(r2) * f2))  # the product rounded to fp32
        if t2 is not None:
            keep &= bool(f1 <= np.float32(t2))
        out["j1"][i], out["s1"][i], out["s2"][i], out["d1"][i], out["d2"][i] = j1, best, s2, d1, d2
        out["keep"][i] = keep
        out["gap"][i] = best - s2
        out["ratio_margin"][i] = abs(d1 - r2 * d2) if r2 is not None and d2 != np.inf else np.inf
        out["dist_margin"][i] = abs(d1 - t2) if t2 is not None else np.inf
    return out


def _pair_len(lens, b, cap):
    return cap if lens is None else int(min(max(int(lens[b]), 0), cap))


def match(desc0, desc1, lens0=None, lens1=None, ratio_thresh=None, distance_thresh=None, mutual_check=True,
          split=False) -> dict:
    """desc0 [B, M, D], desc1 [B, N, D] (any float array) -> matches0 [B, M], matches1 [B, N] int64,
    matching_scores0 / 1 float32, matches / scores lists per pair, and ``sides[b] = (one_way 0->1, one_way 1->0)``.
    split: s from the device's split-bf16 products (see the module docstring)."""
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
        m, n = _pair_len(lens0, b, M), _pair_len(lens1, b, N)
        S = similarity(d0[b, :m], d1[b, :n], split) if m and n else np.zeros((m, n))
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


# ----------------------------------------------------------------------------------------------- vectorised, chunked
def _split_t(d):
    hi = d.bfloat16().float()
    return hi.double(), (d - hi).bfloat16().double()


def _one_way_t(A, Bm, r2, t2, gate_rows, chunk):
    """one_way on S = A Bm^T (float64 torch, or (hi, lo) pairs for the split), chunk rows at a time; gate_rows(r0, r1)
    gives the bool gate of rows r0 .. r1 - 1 against every column, or None for all columns."""
    splitm = isinstance(A, tuple)
    rows = A[0].shape[0] if splitm else A.shape[0]
    cols = Bm[0].shape[0] if splitm else Bm.shape[0]
    dev = A[0].device if splitm else A.device
    f64 = dict(dtype=torch.float64, device=dev)
    out = {k: torch.zeros(rows, **f64) for k in ("s1", "s2", "d1", "d2", "gap", "ratio_margin", "dist_margin")}
    out["j1"] = torch.full((rows,), -1, dtype=torch.int64, device=dev)
    out["keep"] = torch.zeros(rows, dtype=torch.bool, device=dev)
    if cols == 0:
        for k in ("s1", "s2"):
            out[k].fill_(-np.inf)
        for k in ("gap", "ratio_margin", "dist_margin"):
            out[k].fill_(np.inf)
        return out
    idx = torch.arange(cols, device=dev)
    for r0 in range(0, rows, chunk):
        r1 = min(r0 + chunk, rows)
        if splitm:
            S = A[0][r0:r1] @ Bm[0].T + A[0][r0:r1] @ Bm[1].T + A[1][r0:r1] @ Bm[0].T
        else:
            S = A[r0:r1] @ Bm.T
        G = gate_rows(r0, r1) if gate_rows is not None else None
        if G is not None:
            S = S.masked_fill(~G, -np.inf)
        s1 = S.max(1).values
        j1 = torch.where(S == s1[:, None], idx, cols).min(1).values  # the lowest j among the maxima
        none = s1 == -np.inf  # gated: no gated column
        s2 = S.scatter(1, j1.clamp(max=cols - 1)[:, None], -np.inf).max(1).values if cols > 1 else torch.full_like(s1, -np.inf)
        s2 = torch.where(none, -np.inf, s2)
        d1 = 2.0 * (1.0 - s1)
        d2 = torch.where(s2 == -np.inf, np.inf, 2.0 * (1.0 - s2))
        f1, f2 = d1.float(), d2.float()
        keep = ~none
        if r2 is not None:
            keep &= f1 <= torch.tensor(r2, dtype=torch.float32, device=dev) * f2
        if t2 is not None:
            keep &= f1 <= torch.tensor(t2, dtype=torch.float32, device=dev)
        inf = torch.full_like(s1, np.inf)
        out["j1"][r0:r1] = torch.where(none, -1, j1)
        out["s1"][r0:r1], out["s2"][r0:r1] = s1, s2
        out["d1"][r0:r1] = torch.where(none, 0.0, d1)
        out["d2"][r0:r1] = torch.where(none, 0.0, d2)
        out["keep"][r0:r1] = keep
        out["gap"][r0:r1] = torch.where(none, inf, s1 - s2)
        out["ratio_margin"][r0:r1] = (torch.where(none | (d2 == np.inf), inf, (d1 - r2 * d2).abs())
                                      if r2 is not None else inf)
        out["dist_margin"][r0:r1] = torch.where(none, inf, (d1 - t2).abs()) if t2 is not None else inf
    return out


def match_chunked(desc0, desc1, lens0=None, lens1=None, ratio_thresh=None, distance_thresh=None, mutual_check=True,
                  split=False, gate=None, device="cpu", chunk=2048) -> dict:
    """``match``'s rules and result (``sides`` as numpy arrays, margins included) in torch float64 on `device`, chunk
    rows of S at a time.  gate(b, side, r0, r1) -> bool tensor [r1 - r0, partner length] on `device`, the gate of rows
    r0 .. r1 - 1 of pair b's image `side` against the other image's columns, or None for every column (see
    nn_guided_oracle.chunk_gate)."""
    d0 = desc0 if torch.is_tensor(desc0) else torch.as_tensor(np.asarray(desc0, dtype=np.float64))
    d1 = desc1 if torch.is_tensor(desc1) else torch.as_tensor(np.asarray(desc1, dtype=np.float64))
    B, M, _ = d0.shape
    N = d1.shape[1]
    r2, t2 = thresholds(ratio_thresh, distance_thresh)
    m0 = np.full((B, M), -1, dtype=np.int64)
    m1 = np.full((B, N), -1, dtype=np.int64)
    sc0 = np.zeros((B, M), dtype=np.float32)
    sc1 = np.zeros((B, N), dtype=np.float32)
    matches, scores, sides = [], [], []
    for b in range(B):
        m, n = _pair_len(lens0, b, M), _pair_len(lens1, b, N)
        if split:
            x0, x1 = _split_t(d0[b, :m].to(device).float()), _split_t(d1[b, :n].to(device).float())
        else:
            x0, x1 = d0[b, :m].to(device).double(), d1[b, :n].to(device).double()
        g0 = g1 = None
        if gate is not None:
            g0 = lambda r0, r1: gate(b, 0, r0, r1)  # noqa: E731
            g1 = lambda r0, r1: gate(b, 1, r0, r1)  # noqa: E731
        a = _one_way_t(x0, x1, r2, t2, g0, chunk)
        c = _one_way_t(x1, x0, r2, t2, g1, chunk)
        ka, kc = a["keep"], c["keep"]
        ja, jc = a["j1"], c["j1"]
        ok0, ok1 = ka.clone(), kc.clone()
        if mutual_check:
            if m and n:
                ok0 &= kc[ja.clamp(0, n - 1)] & (jc[ja.clamp(0, n - 1)] == torch.arange(m, device=ja.device))
                ok1 &= ka[jc.clamp(0, m - 1)] & (ja[jc.clamp(0, m - 1)] == torch.arange(n, device=jc.device))
            else:
                ok0[:], ok1[:] = False, False
        m0[b, :m] = torch.where(ok0, ja, -1).cpu().numpy()
        m1[b, :n] = torch.where(ok1, jc, -1).cpu().numpy()
        sc0[b, :m] = np.where(ok0.cpu().numpy(), ((a["s1"].cpu().numpy() + 1.0) / 2.0).astype(np.float32), 0)
        sc1[b, :n] = np.where(ok1.cpu().numpy(), ((c["s1"].cpu().numpy() + 1.0) / 2.0).astype(np.float32), 0)
        rows = np.flatnonzero(m0[b] >= 0)
        matches.append(np.stack([rows, m0[b, rows]], axis=1).astype(np.int64).reshape(-1, 2))
        scores.append(sc0[b, rows])
        sides.append(tuple({k: v.cpu().numpy() for k, v in o.items()} for o in (a, c)))
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
