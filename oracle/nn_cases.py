"""Constructed inputs of the nearest-neighbour matcher's stage tests (tests/test_gpu_nn_stages.py, test_nn_emulation.py)
and host restatements of its stages (include/nn_b200.h, nn_workspace_layout).

``split_grid`` descriptors make every pass of the split exact and non-zero: hi is on the k / 16 grid (|k| <= 2) and lo
a single bit, 2^(e - 10) for hi = +-2^e, below half an ulp of hi in bf16 on both sides of it (so bf16_rn(hi + lo) = hi
with no tie).  Every product hi hi, hi lo, lo hi is then a multiple of 2^-18 and every sum of D <= 512 of them stays
below 16, so it holds in 22 significant bits and is exact in fp32 in any order: the device's s equals the float64
split oracle's bit for bit.

``plant`` puts exact ties at the columns where the sweep's reductions meet (one lane, neighbouring lanes of a quad, a
128-column slot edge, a 256-column tile edge) and duplicate rows of image 0 across the tail's 1024-row chunks.
``slot_partials``, ``tail`` and ``outputs`` restate the sweep's per-slot partials, the tail's merge and tests, and the
output writes, each from the stage before it.
"""
from __future__ import annotations

import numpy as np
import torch

from . import nn_oracle as nno

# (columns of image 1 that tie for one row of image 0, what the tie straddles).  Column c sits in lane (c % 8) // 2 of
# the quad that reduces its row, in slot c // 128 and tile c // 256.
TIES = (
    ((0, 8), "one lane"),
    ((16, 18), "lanes 0 / 1"),
    ((33, 34), "lanes 0 / 1, odd and even column"),
    ((48, 54), "lanes 0 / 3"),
    ((127, 128), "slot edge"),
    ((255, 256), "tile edge"),
    ((64, 70, 200), "three-way, two lanes and two slots"),
    ((1023, 1024, 4096), "three-way, slots 7 / 8 / 32"),
)
# rows of image 0 that repeat an earlier row: several rows name one j, and image 1's rows tie across these columns
DUP_ROWS = ((20, 21), (127, 128), (1000, 1030), (2040, 2050, 3100))


def split_grid(g: np.random.Generator, shape) -> np.ndarray:
    """fp32 descriptors hi + lo on the split grid (module docstring)."""
    k = g.integers(-2, 3, shape)
    e = np.where(np.abs(k) == 2, -3, -4)
    lo = np.where(k == 0, 0.0, g.choice([-1.0, 1.0], shape) * np.exp2(e - 10.0))
    return (k / 16 + lo).astype(np.float32)


def _loud(g, d):
    """A split-grid row of the largest norm: its self-similarity beats every other split-grid row's dot with it."""
    return (g.choice([-1.0, 1.0], d) * (2 / 16 + 2.0 ** -13)).astype(np.float32)


def plant(g, d0, d1, b, m, n):
    """Plants, in pair b with m and n live rows, every tie of TIES and every duplicate of DUP_ROWS that fits.  Returns
    [(row, columns)] of the planted ties (each row's maxima are exactly those columns) and the duplicate row groups."""
    ties, dups = [], []
    row = 1
    for cols, _ in TIES:
        if max(cols) >= n or row >= m:
            continue
        v = _loud(g, d0.shape[-1])
        d0[b, row] = v
        d1[b, list(cols)] = v
        ties.append((row, cols))
        row += 3
    for rows in DUP_ROWS:
        if max(rows) < m:
            d0[b, list(rows[1:])] = d0[b, rows[0]]
            dups.append(rows)
    return ties, dups


def make_pair(seed, B, M, N, D, lens0=None, lens1=None, copies=0.5):
    """Split-grid descriptors [B, M, D], [B, N, D] where a share `copies` of each pair's image-1 rows repeat image-0
    rows (so rows match on both sides of every chunk), with the ties of ``plant`` in every pair.  Returns d0, d1 and
    the planted ties and duplicates per pair."""
    g = np.random.default_rng(seed)
    d0, d1 = split_grid(g, (B, M, D)), split_grid(g, (B, N, D))
    planted = []
    for b in range(B):
        m = M if lens0 is None else min(max(int(lens0[b]), 0), M)
        n = N if lens1 is None else min(max(int(lens1[b]), 0), N)
        k = int(copies * min(m, n))
        if k:
            d1[b, g.permutation(n)[:k]] = d0[b, g.permutation(m)[:k]]
        planted.append(plant(g, d0, d1, b, m, n))
    return d0, d1, planted


def ratio_pair(ratio, D=64):
    """One row of image 0 and two of image 1 whose s1 = k1 / 256 and s2 = k2 / 256 put the fp32 ratio test exactly on
    its boundary: D1 == fp32(r2 * D2) while r2 * D2 < D1 in float64, so the header keeps the row and a float64
    product would not.  r = 0.5: D1 = r2 D2 exactly.  Returns d0 [1, 1, D], d1 [1, 2, D], (k1, k2)."""
    k1, k2 = {0.5: (224, 128), 0.7: (109, -44), 0.95: (-105, -144)}[ratio]
    d0 = np.zeros((1, 1, D), np.float32)
    d1 = np.zeros((1, 2, D), np.float32)
    d0[0, 0, 0] = 1 / 16
    d1[0, :, 0] = (k1 / 16, k2 / 16)
    return d0, d1, (k1, k2)


# --------------------------------------------------------------------------------------------------- stage restatements
def slot_partials(S: torch.Tensor, n: int, G: torch.Tensor | None = None):
    """The sweep's partials of the rows of S [rows, >= n] (float64, exact fp32 values) over columns < n, per 128-column
    slot t < ceil(n / 128): s1 the slot's maximum over its live (and gated) columns, j1 the lowest column among the
    maxima, s2 the maximum over the slot's other such columns; s1 = s2 = -inf and j1 = INT32_MAX with none."""
    rows = S.shape[0]
    nt = (n + 127) // 128
    X = torch.full((rows, nt * 128), -np.inf, dtype=torch.float64, device=S.device)
    X[:, :n] = S[:, :n] if G is None else S[:, :n].masked_fill(~G[:, :n], -np.inf)
    live = torch.zeros(nt * 128, dtype=torch.bool, device=S.device)
    live[:n] = True
    L = live[None].expand(rows, -1) if G is None else torch.cat(
        [G[:, :n], torch.zeros(rows, nt * 128 - n, dtype=torch.bool, device=S.device)], 1)
    X, L = X.view(rows, nt, 128), L.reshape(rows, nt, 128)
    col = torch.arange(nt * 128, device=S.device).view(1, nt, 128)
    s1 = X.max(2).values
    hit = L & (X == s1[..., None])
    j1 = torch.where(hit, col, 2**31 - 1).min(2).values
    s2 = X.scatter(2, (j1 % 128)[..., None], -np.inf).max(2).values
    s2 = torch.where(L.any(2), s2, -np.inf)
    j1 = torch.where(L.any(2), j1, 2**31 - 1)
    return s1.float(), s2.float(), j1.int()


def tail(part: np.ndarray, parg: np.ndarray, cols: int, r2, t2):
    """nn_tail_kernel's merge and tests from the partials of some rows ([rows, >= nt, 2] fp32, [rows, >= nt] int32):
    slots in ascending order, a later slot wins only when strictly greater; D1, D2, the product and the comparisons in
    fp32.  r2 / t2 None or <= 0: the test is off.  Returns (jbest, sbest)."""
    rows = part.shape[0]
    nt = (cols + 127) // 128
    s1 = np.full(rows, -np.inf, np.float32)
    s2 = np.full(rows, -np.inf, np.float32)
    j = np.full(rows, -1, np.int64)
    for t in range(nt):
        vx, vy = part[:, t, 0], part[:, t, 1]
        win = vx > s1
        s2 = np.where(win, np.fmax(s1, vy), np.fmax(s2, vx)).astype(np.float32)
        j = np.where(win, parg[:, t], j)
        s1 = np.where(win, vx, s1).astype(np.float32)
    one, two = np.float32(1), np.float32(2)
    with np.errstate(over="ignore", invalid="ignore"):
        d1, d2 = two * (one - s1), two * (one - s2)
        keep = np.ones(rows, bool)
        if r2 is not None and r2 > 0:
            keep &= d1 <= np.float32(r2) * d2
        if t2 is not None and t2 > 0:
            keep &= d1 <= np.float32(t2)
    jbest = np.where(keep & (j >= 0) & (j < cols), j, -1).astype(np.int32)
    return jbest, s1


def outputs(jb0, sb0, jb1, sb1, M, N, mutual):
    """nn_tail_kernel's writes for one pair from its rows' jbest / sbest (m and n live rows): matches0 / 1 and their
    fp32 scores (s1 + 1) * 0.5, the ascending `matches` list, its scores and its count."""
    m, n = len(jb0), len(jb1)
    half, one = np.float32(0.5), np.float32(1)
    m1 = np.full(N, -1, np.int64)
    for j in range(n):
        i = int(jb1[j])
        if i >= 0 and mutual and jb0[i] != j:
            i = -1
        m1[j] = i
    m0 = np.full(M, -1, np.int64)
    for i in range(m):
        j = int(jb0[i])
        if j >= 0 and mutual and jb1[j] != i:
            j = -1
        m0[i] = j
    sc0 = np.zeros(M, np.float32)
    sc1 = np.zeros(N, np.float32)
    sc0[:m] = np.where(m0[:m] >= 0, (sb0 + one) * half, 0)
    sc1[:n] = np.where(m1[:n] >= 0, (sb1 + one) * half, 0)
    rows = np.flatnonzero(m0 >= 0)
    return {"matches0": m0, "matches1": m1, "matching_scores0": sc0, "matching_scores1": sc1,
            "matches": np.stack([rows, m0[rows]], 1), "scores": sc0[rows], "n_matches": len(rows)}


# ------------------------------------------------------------------------------------------------ arithmetic emulation
PASSES = ("hh", "hl", "lh")  # the device's three products; "ll" is the dropped lo0 lo1


def emulate(a, b, passes=PASSES, k_step=16, block=64):
    """s = a b^T ([m, D] x [n, D], fp32 values) as the sweep forms it, in this order: for each 64-wide K block, the
    products of `passes` in turn, each over k steps of 16 (one tensor-core instruction each); a step's 16 exact
    products are summed exactly and added to the fp32 accumulator with one rounding.  Returns float64 of the fp32 s."""
    a = torch.as_tensor(np.asarray(a, np.float32))
    b = torch.as_tensor(np.asarray(b, np.float32))
    parts = {}
    for name, x in (("a", a), ("b", b)):
        hi = x.bfloat16().float()
        parts[name] = {"h": hi.double(), "l": (x - hi).bfloat16().double()}
    acc = torch.zeros(a.shape[0], b.shape[0], dtype=torch.float32)
    for k0 in range(0, a.shape[1], block):
        for p in passes:
            x, y = parts["a"][p[0]], parts["b"][p[1]]
            for k in range(k0, min(k0 + block, a.shape[1]), k_step):
                step = x[:, k:k + k_step] @ y[:, k:k + k_step].T  # 16 products of 16 bits each: exact in float64
                acc = (acc.double() + step).float()
    return acc.double()
