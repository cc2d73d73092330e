"""Lens distortion on the GPU (lightglue_b200.camera.undistort_points and the dist_coeffs0 argument of
estimate_absolute_pose and estimate_absolute_pose_lo) against OpenCV on the host.

Prints one JSON line:
  * the card's name and power limit, read in this run;
  * undistort_points ms per batch (CUDA events) at 32 x 2048 and 8 x 8192 points, float32, OpenCV's defaults (5
    iterations), against cv2.undistortPoints in a 16-thread host pool (null without cv2);
  * estimate_absolute_pose and estimate_absolute_pose_lo ms per batch at 32 pairs x 2048 matches, 50 % outliers,
    cv2.solvePnPRansac's defaults, with and without dist_coeffs0 (the two alternated within one run, the median of
    several rounds), against cv2.solvePnPRansac(..., distCoeffs) in the pool.
  * fisheye_undistort_points ms per batch at 32 x 2048 and 8 x 8192 points, float32, OpenCV's default criteria,
    against cv2.fisheye.undistortPoints in the pool;
  * estimate_absolute_pose_fisheye and estimate_absolute_pose_lo_fisheye at 32 pairs x 2048 matches, 50 % outliers,
    alternated with the dist_coeffs0 call in one run (median of rounds), against cv2.fisheye.solvePnPRansac in the
    pool; and, on the same fisheye scenes with a full budget of 256 samples, the pinhole, dist_coeffs0 and fisheye calls
    alternated, which isolates the lens's cost.
The scenes come from oracle/pnp_dist_oracle.scene with k = (-0.3, 0.09, 1e-3, -5e-4, -0.01) and from
oracle/fisheye_oracle.scene (field angles up to 85 degrees); nothing is written to disk.
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

from lightglue_b200.camera import fisheye_undistort_points, undistort_points  # noqa: E402
from lightglue_b200.geometry import (estimate_absolute_pose, estimate_absolute_pose_fisheye,  # noqa: E402
                                     estimate_absolute_pose_lo, estimate_absolute_pose_lo_fisheye)
from oracle import fisheye_oracle as fo  # noqa: E402
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
    fisheye(res, args, cv2, t0, t3, tm, Kt, Dt)
    print(json.dumps(res))


def fisheye(res, args, cv2, td0, td3, tdm, Kt, Dt):
    """The fisheye arms; the distortion scene's tensors give the alternated dist_coeffs0 call."""
    rng = np.random.default_rng(1)
    Kf, Df = fo.K_SCENE, fo.D_SCENE
    Kft, Dft = torch.from_numpy(Kf).cuda(), torch.from_numpy(Df).cuda()
    for B, N in ((32, 2048), (8, 8192)):
        px = rng.uniform(140, 884, (B, N, 2)).astype(np.float32)
        tp = torch.from_numpy(px).cuda()
        gpu = time_gpu(lambda: fisheye_undistort_points(tp, Kft, Dft), args.reps)
        cpu = None if cv2 is None else pool_ms(
            lambda b: cv2.fisheye.undistortPoints(px[b][:, None].astype(np.float64), Kf, Df, P=Kf), B, args.threads)
        res[f"fisheye_undistort_{B}x{N}"] = {"gpu_ms": round(gpu, 4),
                                              "opencv_pool_ms": None if cpu is None else round(cpu, 3)}
    B, M = 32, 2048
    sc = [fo.scene(M, 0.5, 700 + b) for b in range(B)]
    k0, p3, m0 = (np.stack([s[i] for s in sc]) for i in range(3))
    t0, t3, tm = (torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in (k0, p3, m0))
    for name, fn, ff in (("pnp", estimate_absolute_pose, estimate_absolute_pose_fisheye),
                         ("pnp_lo", estimate_absolute_pose_lo, estimate_absolute_pose_lo_fisheye)):
        fish, dist = [], []
        for _ in range(args.rounds):  # alternated, so both see the same clocks and neighbours
            fish.append(time_gpu(lambda: ff(t0, t3, tm, Kft, Dft), args.reps))
            dist.append(time_gpu(lambda: fn(td0, td3, tdm, Kt, dist_coeffs0=Dt), args.reps))
        cpu = None
        if cv2 is not None:
            def one(b):
                _, pix, wld = pp.compact(k0[b], p3[b], m0[b])
                cv2.fisheye.solvePnPRansac(wld[:, None].astype(np.float64), pix[:, None].astype(np.float64), Kf, Df,
                                           iterationsCount=100, reprojectionError=8.0, confidence=0.99)
            cpu = pool_ms(one, B, args.threads)
        out = ff(t0, t3, tm, Kft, Dft)
        res[f"{name}_fisheye_{B}x{M}"] = {"gpu_ms_fisheye": round(float(np.median(fish)), 4),
                                          "gpu_ms_fisheye_range": [round(min(fish), 4), round(max(fish), 4)],
                                          "gpu_ms_dist": round(float(np.median(dist)), 4),
                                          "opencv_fisheye_pool_ms": None if cpu is None else round(cpu, 3),
                                          "success_fisheye": int(out["success"].sum())}
        # the lens's own cost: the same fisheye scenes and a full budget of 256 samples per pair (no adaptive stop),
        # through the pinhole K, the rational lens with 4 coefficients and the fisheye lens, alternated
        arms = {"pinhole": lambda: fn(t0, t3, tm, Kft, max_iters=256, confidence=1.0),
                "dist": lambda: fn(t0, t3, tm, Kft, max_iters=256, confidence=1.0, dist_coeffs0=Dft),
                "fisheye": lambda: ff(t0, t3, tm, Kft, Dft, max_iters=256, confidence=1.0)}
        times = {a: [] for a in arms}
        for _ in range(args.rounds):
            for a, f in arms.items():
                times[a].append(time_gpu(f, args.reps))
        row = {f"gpu_ms_{a}": round(float(np.median(v)), 4) for a, v in times.items()}
        row.update({f"gpu_ms_{a}_range": [round(min(v), 4), round(max(v), 4)] for a, v in times.items()})
        if name == "pnp_lo":  # the LO steps run depend on the scores, so they may differ between the arms
            row.update({f"local_optimizations_{a}": int(f()["num_local_optimizations"].sum()) for a, f in arms.items()})
        res[f"{name}_same_scenes_full_budget_{B}x{M}"] = row


if __name__ == "__main__":
    main()
