"""Batched GPU absolute pose (lightglue_b200.geometry.estimate_absolute_pose and estimate_absolute_pose_lo) against
OpenCV on the host, and its cost behind the matcher.

Prints one JSON line:
  * the card's name and power limit, read in this run;
  * GPU ms per batch (CUDA events) at B pairs of M putative 2D-3D matches and 20 / 50 / 70 % outliers, with OpenCV's
    adaptive stopping ("adaptive") and with confidence 1 ("full", every sample), at cv2.solvePnPRansac's defaults
    (8 px, 0.99) and a budget of 100 samples (1000 at 70 %), for the plain estimator and ("lo_adaptive", "lo_full")
    the LO-RANSAC one;
  * cv2.solvePnPRansac on the host for the same pairs, one after another and in a 16-thread pool (null without cv2),
    with its RANSAC ("opencv") and with UsacParams of MSAC, inner + iterative LO and the LSQ polisher ("opencv_usac");
  * pairs/s of LightGlue (bf16x3, N = 2048, synthetic weights) alone and followed by estimate_absolute_pose on one
    stream, alternated.
The scenes come from oracle/pnp_oracle.localization_scene (0.5 px noise, 640x480, f = 500); nothing is written to disk.
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

from lightglue_b200 import LightGlue, synth  # noqa: E402
from lightglue_b200.geometry import estimate_absolute_pose, estimate_absolute_pose_lo  # noqa: E402
from oracle import pnp_oracle as pp  # noqa: E402
from tools.geometry_bench import gpu_info, time_gpu  # noqa: E402


def opencv_times(k0, p3, m0, K, iters, threads, usac=False):
    try:
        import cv2
    except ImportError:
        return None
    cv2.setNumThreads(1)
    if usac:
        params = cv2.UsacParams()
        params.confidence, params.maxIterations, params.threshold = 0.99, iters, 8.0
        params.score, params.loMethod = cv2.SCORE_METHOD_MSAC, cv2.LOCAL_OPTIM_INNER_AND_ITER_LO
        params.final_polisher = cv2.LSQ_POLISHER

    def one(b):
        _, pix, wld = pp.compact(k0[b], p3[b], m0[b])
        if usac:
            cv2.solvePnPRansac(wld.astype(np.float64), pix.astype(np.float64), K, None, params=params)
        else:
            cv2.solvePnPRansac(wld.astype(np.float64), pix.astype(np.float64), K, None, iterationsCount=iters,
                               reprojectionError=8.0, confidence=0.99)

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
    ap.add_argument("--steps", type=int, default=20, help="matcher steps per pairs/s measurement")
    ap.add_argument("--threads", type=int, default=16)
    args = ap.parse_args()
    torch.set_grad_enabled(False)
    res = {"tool": "pnp_bench", **gpu_info(), "B": args.batch, "matches": args.matches, "pnp": {}}
    for o in (0.2, 0.5, 0.7):
        iters = 1000 if o > 0.6 else 100
        pairs = [pp.localization_scene(args.matches, o, 1000 + b, unmatched=0.0) for b in range(args.batch)]
        k0, p3, m0, _, K, _, _ = (np.stack([p[i] for p in pairs]) for i in range(7))
        t0, t3, tm, tk = (torch.from_numpy(x).cuda() for x in (k0, p3, m0, K[0]))
        row = {"max_iters": iters}
        for prefix, fn in (("", estimate_absolute_pose), ("lo_", estimate_absolute_pose_lo)):
            for mode, c in (("adaptive", 0.99), ("full", 1.0)):
                out = fn(t0, t3, tm, tk, max_iters=iters, confidence=c)
                row[prefix + mode] = {
                    "gpu_ms": round(time_gpu(lambda: fn(t0, t3, tm, tk, max_iters=iters, confidence=c), args.reps), 3),
                    "mean_samples": float(out["num_hypotheses"].float().mean()),
                    "mean_inliers": float(out["num_inliers"].float().mean())}
        row["opencv"] = opencv_times(k0, p3, m0, K[0], iters, args.threads)
        row["opencv_usac"] = opencv_times(k0, p3, m0, K[0], iters, args.threads, usac=True)
        res["pnp"][f"outliers{o}"] = row
    # the matcher alone, and followed by the absolute pose on its device output (no host read-back in between)
    data, _ = synth.make_pair(2048, b=args.batch, seed=7)
    cuda = {k: {kk: vv.cuda() for kk, vv in v.items()} for k, v in data.items()}
    m = LightGlue(features=None, depth_confidence=-1, width_confidence=-1, precision="bf16x3")
    m.load_state_dict(synth.make_state_dict(), strict=False)
    m = m.eval().cuda()
    Kc = torch.tensor([[800.0, 0.0, 512.0], [0.0, 800.0, 384.0], [0.0, 0.0, 1.0]], dtype=torch.float64, device="cuda")
    k1 = cuda["image1"]["keypoints"].double()
    d = torch.rand(k1.shape[:2], generator=torch.Generator().manual_seed(3), dtype=torch.float64).cuda() * 8.0 + 4.0
    p3 = torch.stack([(k1[..., 0] - 512.0) / 800.0 * d, (k1[..., 1] - 384.0) / 800.0 * d, d], -1).float()

    def matcher_only():
        return m.forward_async(cuda).tensors["matches0"]

    def matcher_pnp():
        m0 = m.forward_async(cuda).tensors["matches0"]
        return estimate_absolute_pose(cuda["image0"]["keypoints"], p3, m0, Kc)

    for name, f in (("lightglue", matcher_only), ("lightglue_plus_pnp", matcher_pnp), ("lightglue_again", matcher_only),
                    ("lightglue_plus_pnp_again", matcher_pnp)):
        ms = time_gpu(f, args.steps)
        res[f"{name}_pairs_per_s"] = round(args.batch / ms * 1e3, 1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
