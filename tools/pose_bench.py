"""Batched GPU relative pose (lightglue_b200.geometry.estimate_relative_pose and its LO-RANSAC arm,
estimate_relative_pose_lo) against OpenCV on the host, and its cost behind the matcher.

Prints one JSON line:
  * the card's name and power limit, read in this run;
  * GPU ms per batch (CUDA events) at B pairs of M putative matches and 20 / 50 / 70 % outliers, with OpenCV's
    adaptive stopping ("adaptive") and with confidence 1 ("full", every sample);
  * the same for estimate_relative_pose_lo ("lo"), and both estimators' median pose error against the ground truth
    (the larger of the rotation and translation-direction errors, degrees);
  * cv2.findEssentialMat(RANSAC) + cv2.recoverPose on the host for the same pairs, one after another and in a thread
    pool, and cv2.findEssentialMat(USAC_ACCURATE) in the pool (null without cv2);
  * pairs/s of LightGlue (bf16x3, N = 2048, synthetic weights) alone and followed by estimate_relative_pose or
    estimate_relative_pose_lo on one stream.
The scenes come from oracle/pose_oracle.calibrated_two_view (0.5 px noise, 640x480, f = 500); nothing is written to disk.
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
from lightglue_b200.geometry import estimate_relative_pose, estimate_relative_pose_lo  # noqa: E402
from oracle import pose_oracle as po  # noqa: E402
from tools.geometry_bench import gpu_info, time_gpu  # noqa: E402


def pose_error(R, t, Rg, tg):
    """Median over the pairs of the larger of the rotation and translation-direction errors, degrees."""
    e = []
    for b in range(len(Rg)):
        c = np.clip((np.trace(R[b].T @ Rg[b]) - 1.0) / 2.0, -1.0, 1.0)
        ct = min(1.0, abs(float(t[b] @ tg[b])) / max(np.linalg.norm(t[b]), 1e-300))
        e.append(max(np.degrees(np.arccos(c)), np.degrees(np.arccos(ct))))
    return round(float(np.median(e)), 3)


def opencv_times(k0, k1, m0, K, threads, method="RANSAC", sequential=True):
    try:
        import cv2
    except ImportError:
        return None
    cv2.setNumThreads(1)
    flag = getattr(cv2, method)

    def one(b):
        v = m0[b] >= 0
        a, c = k0[b][v].astype(np.float64), k1[b][m0[b][v]].astype(np.float64)
        E, mask = cv2.findEssentialMat(a, c, K, flag, 0.999, 1.0, maxIters=1000)
        cv2.recoverPose(E[:3], a, c, K, mask=mask)

    if not sequential:
        with ThreadPoolExecutor(threads) as ex:
            t = time.perf_counter()
            list(ex.map(one, range(len(m0))))
            pool = (time.perf_counter() - t) * 1e3
        return {"pool_ms": round(pool, 2), "threads": threads}

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
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--steps", type=int, default=20, help="matcher steps per pairs/s measurement")
    args = ap.parse_args()
    torch.set_grad_enabled(False)
    res = {"tool": "pose_bench", **gpu_info(), "B": args.batch, "matches": args.matches, "pose": {}}
    threads = os.cpu_count() or 1
    for o in (0.2, 0.5, 0.7):
        pairs = [po.calibrated_two_view(args.matches, o, 1000 + b, unmatched=0.0) for b in range(args.batch)]
        k0, k1, m0, _, K, _, Rg, tg = (np.stack([p[i] for p in pairs]) for i in range(8))
        t0, t1, tm, tk = (torch.from_numpy(x).cuda() for x in (k0, k1, m0, K[0]))
        row = {}
        for arm, f in (("ransac", estimate_relative_pose), ("lo", estimate_relative_pose_lo)):
            for mode, c in (("adaptive", 0.999), ("full", 1.0)):
                out = f(t0, t1, tm, tk, confidence=c)
                row[f"{arm}_{mode}" if arm == "lo" else mode] = {
                    "gpu_ms": round(time_gpu(lambda: f(t0, t1, tm, tk, confidence=c), args.reps), 3),
                    "mean_samples": float(out["num_hypotheses"].float().mean()),
                    "mean_inliers": float(out["num_inliers"].float().mean()),
                    "median_pose_error_deg": pose_error(out["R"].cpu().numpy(), out["t"].cpu().numpy(), Rg, tg)}
        row["opencv"] = opencv_times(k0, k1, m0, K[0], threads)
        row["opencv_usac_accurate"] = opencv_times(k0, k1, m0, K[0], threads, "USAC_ACCURATE", sequential=False)
        res["pose"][f"outliers{o}"] = row
    # the matcher alone, and followed by the relative pose on its device output (no host read-back in between)
    data, _ = synth.make_pair(2048, b=args.batch, seed=7)
    cuda = {k: {kk: vv.cuda() for kk, vv in v.items()} for k, v in data.items()}
    m = LightGlue(features=None, depth_confidence=-1, width_confidence=-1, precision="bf16x3")
    m.load_state_dict(synth.make_state_dict(), strict=False)
    m = m.eval().cuda()
    Kc = torch.tensor([[800.0, 0.0, 512.0], [0.0, 800.0, 384.0], [0.0, 0.0, 1.0]], dtype=torch.float64, device="cuda")

    def matcher_only():
        return m.forward_async(cuda).tensors["matches0"]

    def matcher_pose():
        m0 = m.forward_async(cuda).tensors["matches0"]
        return estimate_relative_pose(cuda["image0"]["keypoints"], cuda["image1"]["keypoints"], m0, Kc)

    def matcher_lo_pose():
        m0 = m.forward_async(cuda).tensors["matches0"]
        return estimate_relative_pose_lo(cuda["image0"]["keypoints"], cuda["image1"]["keypoints"], m0, Kc)

    for name, f in (("lightglue", matcher_only), ("lightglue_plus_pose", matcher_pose),
                    ("lightglue_again", matcher_only), ("lightglue_plus_lo_pose", matcher_lo_pose),
                    ("lightglue_again2", matcher_only)):
        ms = time_gpu(f, args.steps)
        res[f"{name}_pairs_per_s"] = round(args.batch / ms * 1e3, 1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
