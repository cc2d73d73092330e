"""Lens distortion on the GPU (lightglue_b200.camera.undistort_points and the dist_coeffs0 argument of
estimate_absolute_pose and estimate_absolute_pose_lo) against OpenCV on the host.

Prints one JSON line:
  * the card's name and power limit, read in this run;
  * undistort_points ms per batch (CUDA events) at 32 x 2048 and 8 x 8192 points, float32, OpenCV's defaults (5
    iterations), against cv2.undistortPoints in a 16-thread host pool (null without cv2);
  * estimate_absolute_pose and estimate_absolute_pose_lo ms per batch at 32 pairs x 2048 matches, 50 % outliers,
    cv2.solvePnPRansac's defaults, with and without dist_coeffs0 (the two alternated within one run, the median of
    several rounds), against cv2.solvePnPRansac(..., distCoeffs) in the pool.
The scenes come from oracle/pnp_dist_oracle.scene with k = (-0.3, 0.09, 1e-3, -5e-4, -0.01); nothing is
written to disk.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from lightglue_b200.camera import undistort_points  # noqa: E402
from lightglue_b200.geometry import estimate_absolute_pose, estimate_absolute_pose_lo  # noqa: E402
from oracle import pnp_dist_oracle as pd  # noqa: E402
from oracle import pnp_oracle as pp  # noqa: E402
from tools.geometry_bench import gpu_info, time_gpu  # noqa: E402

D = np.array([-0.3, 0.09, 1e-3, -5e-4, -0.01])
K = np.array([[500.0, 0.0, 320.0], [0.0, 500.0, 240.0], [0.0, 0.0, 1.0]])


def pool_ms(fn, n, threads):
    with ThreadPoolExecutor(threads) as ex:
        list(ex.map(fn, range(min(n, threads))))  # warm up
        t = time.perf_counter()
        list(ex.map(fn, range(n)))
        return (time.perf_counter() - t) * 1e3


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--threads", type=int, default=16)
    args = ap.parse_args()
    try:
        import cv2
        cv2.setNumThreads(1)
    except ImportError:
        cv2 = None
    res = {"bench": "camera", **gpu_info()}
    rng = np.random.default_rng(0)
    Kt, Dt = torch.from_numpy(K).cuda(), torch.from_numpy(D).cuda()
    for B, N in ((32, 2048), (8, 8192)):
        px = np.stack([rng.uniform(0, 640, (B, N)), rng.uniform(0, 480, (B, N))], -1).astype(np.float32)
        tp = torch.from_numpy(px).cuda()
        gpu = time_gpu(lambda: undistort_points(tp, Kt, Dt), args.reps)
        cpu = None if cv2 is None else pool_ms(
            lambda b: cv2.undistortPoints(px[b][:, None].astype(np.float64), K, D, P=K), B, args.threads)
        res[f"undistort_{B}x{N}"] = {"gpu_ms": round(gpu, 4), "opencv_pool_ms": None if cpu is None else round(cpu, 3)}
    B, M = 32, 2048
    sc = [pd.scene(M, 0.5, 500 + b, D) for b in range(B)]
    k0, p3, m0 = (np.stack([s[i] for s in sc]) for i in range(3))
    t0, t3, tm = (torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in (k0, p3, m0))
    for name, fn in (("pnp", estimate_absolute_pose), ("pnp_lo", estimate_absolute_pose_lo)):
        plain, dist = [], []
        for _ in range(args.rounds):  # alternated, so both see the same clocks and neighbours
            plain.append(time_gpu(lambda: fn(t0, t3, tm, Kt), args.reps))
            dist.append(time_gpu(lambda: fn(t0, t3, tm, Kt, dist_coeffs0=Dt), args.reps))
        cpu = None
        if cv2 is not None:
            def one(b):
                _, pix, wld = pp.compact(k0[b], p3[b], m0[b])
                cv2.solvePnPRansac(wld.astype(np.float64), pix.astype(np.float64), K, D, iterationsCount=100,
                                   reprojectionError=8.0, confidence=0.99)
            cpu = pool_ms(one, B, args.threads)
        out = fn(t0, t3, tm, Kt, dist_coeffs0=Dt)
        res[f"{name}_{B}x{M}"] = {"gpu_ms": round(float(np.median(plain)), 4),
                                  "gpu_ms_dist": round(float(np.median(dist)), 4),
                                  "gpu_ms_dist_range": [round(min(dist), 4), round(max(dist), 4)],
                                  "opencv_dist_pool_ms": None if cpu is None else round(cpu, 3),
                                  "success_dist": int(out["success"].sum())}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
