"""Seeded two-view scenes for the RANSAC tests and tools/geometry_bench.py.

``planar`` draws correspondences of a plane under a known homography, ``two_view`` of a 3-D point cloud seen by two
cameras with known K, R and t.  Inliers get Gaussian noise of ``noise`` px in image 1; outliers (a share ``outliers``
of the matched rows) are uniform over image 1; a share ``unmatched`` of the rows of matches0 is -1.  image 1 holds its
points in a random order, so matches0 is a permutation, as a matcher's would be.
"""
from __future__ import annotations

import numpy as np

W, H = 640.0, 480.0


def true_homography(rng: np.random.Generator) -> np.ndarray:
    a = rng.uniform(-0.3, 0.3)
    sc = rng.uniform(0.8, 1.2)
    c, s = np.cos(a) * sc, np.sin(a) * sc
    A = np.array([[c, -s, 0.0], [s, c, 0.0], [rng.uniform(-3e-4, 3e-4), rng.uniform(-3e-4, 3e-4), 1.0]])
    C = np.array([[1.0, 0.0, -W / 2], [0.0, 1.0, -H / 2], [0.0, 0.0, 1.0]])
    T = np.array([[1.0, 0.0, W / 2 + rng.uniform(-40, 40)], [0.0, 1.0, H / 2 + rng.uniform(-40, 40)], [0.0, 0.0, 1.0]])
    Hm = T @ A @ C
    return Hm / Hm[2, 2]


def apply_h(Hm: np.ndarray, x: np.ndarray) -> np.ndarray:
    y = x @ Hm[:, :2].T + Hm[:, 2]
    return y[:, :2] / y[:, 2:3]


def _skew(t):
    return np.array([[0.0, -t[2], t[1]], [t[2], 0.0, -t[0]], [-t[1], t[0], 0.0]])


def _rot(rng):
    w = rng.uniform(-0.15, 0.15, 3)
    th = np.linalg.norm(w)
    k = _skew(w / th)
    return np.eye(3) + np.sin(th) * k + (1 - np.cos(th)) * (k @ k)


def _assemble(rng, x0, x1, inlier, unmatched):
    """Shuffle image 1, add outliers and unmatched rows: (kpts0, kpts1, matches0, true inlier mask)."""
    m = x0.shape[0]
    perm = rng.permutation(m)
    kpts1 = np.empty_like(x1)
    kpts1[perm] = x1
    matches0 = perm.astype(np.int64)
    drop = rng.random(m) < unmatched
    matches0[drop] = -1
    return x0.astype(np.float32), kpts1.astype(np.float32), matches0, inlier & ~drop


def planar(m: int, outliers: float, seed: int, noise: float = 0.5, unmatched: float = 0.1):
    """(kpts0 [m, 2], kpts1 [m, 2], matches0 [m], true inliers [m], H)."""
    rng = np.random.default_rng(seed)
    Hm = true_homography(rng)
    x0 = rng.uniform([0, 0], [W, H], (m, 2))
    x1 = apply_h(Hm, x0) + rng.normal(0.0, noise, (m, 2))
    inlier = rng.random(m) >= outliers
    x1[~inlier] = rng.uniform([0, 0], [W, H], ((~inlier).sum(), 2))
    return (*_assemble(rng, x0, x1, inlier, unmatched), Hm)


def two_view(m: int, outliers: float, seed: int, noise: float = 0.5, unmatched: float = 0.1):
    """(kpts0, kpts1, matches0, true inliers, F) with x1^T F x0 = 0."""
    rng = np.random.default_rng(seed)
    K = np.array([[500.0, 0.0, W / 2], [0.0, 500.0, H / 2], [0.0, 0.0, 1.0]])
    R = _rot(rng)
    t = np.array([1.0, rng.uniform(-0.3, 0.3), rng.uniform(-0.2, 0.2)])
    X = np.stack([rng.uniform(-4, 4, m), rng.uniform(-3, 3, m), rng.uniform(4, 12, m)], 1)
    p0 = X @ K.T
    x0 = p0[:, :2] / p0[:, 2:3]
    p1 = (X @ R.T + t) @ K.T
    x1 = p1[:, :2] / p1[:, 2:3] + rng.normal(0.0, noise, (m, 2))
    inlier = rng.random(m) >= outliers
    x1[~inlier] = rng.uniform([0, 0], [W, H], ((~inlier).sum(), 2))
    Ki = np.linalg.inv(K)
    F = Ki.T @ _skew(t) @ R @ Ki
    return (*_assemble(rng, x0, x1, inlier, unmatched), F / np.linalg.norm(F))


def batch(kind: str, m: int, outliers, seeds, unmatched=0.1):
    """Stacked pairs: outliers and unmatched may be one value or one per pair."""
    make = planar if kind == "H" else two_view
    n = len(seeds)
    outs = np.broadcast_to(np.asarray(outliers, dtype=float), (n,))
    unm = np.broadcast_to(np.asarray(unmatched, dtype=float), (n,))
    pairs = [make(m, o, s, unmatched=u) for o, s, u in zip(outs, seeds, unm)]
    return tuple(np.stack([p[i] for p in pairs]) for i in range(5))


def epipolar_distance(F: np.ndarray, x0: np.ndarray, x1: np.ndarray) -> np.ndarray:
    """Symmetric-max point-to-epipolar-line distance in float64."""
    h0 = np.concatenate([x0, np.ones((len(x0), 1))], 1)
    h1 = np.concatenate([x1, np.ones((len(x1), 1))], 1)
    l1, l0 = h0 @ F.T, h1 @ F
    s = np.abs((h1 * l1).sum(1))
    return np.maximum(s / np.hypot(l1[:, 0], l1[:, 1]), s / np.hypot(l0[:, 0], l0[:, 1]))


CORNERS = np.array([[0.0, 0.0], [W, 0.0], [W, H], [0.0, H]])
