"""Batched GPU affine and similarity estimation (lightglue_b200.geometry.estimate_affine_2d and
estimate_affine_partial_2d) against OpenCV on the host.

Prints one JSON line:
  * the card's name and power limit, read in this run;
  * GPU ms per batch (CUDA events) at B pairs of M putative matches and 20 / 50 / 70 % outliers, for both models at
    cv2's defaults (3 px, 2000 iterations, 0.99, 10 refinement steps), with adaptive stopping ("adaptive") and with
    confidence 1 ("full", all 2000 samples);
  * cv2.estimateAffine2D and cv2.estimateAffinePartial2D (RANSAC) on the host for the same pairs, one after another
    and in a thread pool whose size is printed (null without cv2).
The scenes come from oracle/affine_oracle.scene (1 px noise, 640x480, no unmatched rows); nothing is written to disk.
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

from lightglue_b200.geometry import estimate_affine_2d, estimate_affine_partial_2d  # noqa: E402
from oracle import affine_oracle as ao  # noqa: E402
from tools.geometry_bench import gpu_info, time_gpu  # noqa: E402

MODELS = {"affine": (ao.AFFINE, estimate_affine_2d, "estimateAffine2D"),
          "partial": (ao.PARTIAL, estimate_affine_partial_2d, "estimateAffinePartial2D")}


def opencv_times(k0, k1, m0, name, threads):
    try:
        import cv2
    except ImportError:
        return None
    cv2.setNumThreads(1)
    fn = getattr(cv2, name)

    def one(b):
        v = m0[b] >= 0
        fn(k0[b][v], k1[b][m0[b][v]], method=cv2.RANSAC, ransacReprojThreshold=3.0, maxIters=2000, confidence=0.99,
           refineIters=10)

    t = time.perf_counter()
    for b in range(len(m0)):
        one(b)
    seq = (time.perf_counter() - t) * 1e3
    with ThreadPoolExecutor(threads) as ex:
        t = time.perf_counter()
        list(ex.map(one, range(len(m0))))
        pool = (time.perf_counter() - t) * 1e3
    return {"sequential_ms": round(seq, 2), "pool_ms": round(pool, 2), "threads": threads}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--matches", type=int, default=2048)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--threads", type=int, default=16)
    args = ap.parse_args()
    torch.set_grad_enabled(False)
    res = {"tool": "affine_bench", **gpu_info(), "B": args.batch, "matches": args.matches}
    for model, (kind, fn, cv_name) in MODELS.items():
        res[model] = {}
        for o in (0.2, 0.5, 0.7):
            scenes = [ao.scene(kind, args.matches, o, 1000 + b, noise=1.0, unmatched=0.0) for b in range(args.batch)]
            k0, k1, m0 = (np.stack([sc[i] for sc in scenes]) for i in range(3))
            t0, t1, tm = (torch.from_numpy(x).cuda() for x in (k0, k1, m0))
            row = {}
            for mode, c in (("adaptive", 0.99), ("full", 1.0)):
                out = fn(t0, t1, tm, confidence=c)
                row[mode] = {"gpu_ms": round(time_gpu(lambda: fn(t0, t1, tm, confidence=c), args.reps), 3),
                             "mean_samples": float(out["num_hypotheses"].float().mean()),
                             "mean_inliers": float(out["num_inliers"].float().mean())}
            row["opencv"] = opencv_times(k0, k1, m0, cv_name, args.threads)
            res[model][f"outliers{o}"] = row
    print(json.dumps(res))


if __name__ == "__main__":
    main()
