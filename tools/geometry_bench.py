"""Batched GPU RANSAC (lightglue_b200.geometry) against OpenCV on the host, and its cost behind the matcher.

Prints one JSON line:
  * the card's name and power limit, read in this run;
  * GPU ms per batch (CUDA events) for find_homography and find_fundamental, and for their LO-RANSAC variants
    find_homography_lo and find_fundamental_lo ("lo_adaptive", "lo_full") and their MAGSAC++ variants
    find_homography_magsac and find_fundamental_magsac ("magsac_adaptive", "magsac_full"), at B pairs of M putative matches, inlier
    ratios 0.8 / 0.5 / 0.3, with OpenCV's adaptive stopping ("adaptive") and with confidence 1 ("full", every
    hypothesis);
  * OpenCV on the host for the same pairs, one after another and in a thread pool (null without cv2), and
    cv2.findHomography / cv2.findFundamentalMat(USAC_ACCURATE), the LO-RANSAC the LO variants are compared with
    ("opencv_usac_accurate"), and USAC_MAGSAC, which the MAGSAC++ variants follow ("opencv_usac_magsac");
  * pairs/s of LightGlue (bf16x3, N = 2048, synthetic weights) alone and followed by find_fundamental,
    find_homography_lo or find_fundamental_lo on one stream, the runs alternated.
The scenes come from oracle/geometry_synth.py (0.5 px noise, 640x480); nothing is written to disk.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from lightglue_b200 import LightGlue, synth  # noqa: E402
from lightglue_b200.geometry import (find_fundamental, find_fundamental_lo,  # noqa: E402
                                     find_fundamental_magsac, find_homography, find_homography_lo,
                                     find_homography_magsac)
from oracle import geometry_synth as gs  # noqa: E402

DEFAULTS = {"H": (find_homography, 2000, 0.995), "F": (find_fundamental, 1000, 0.99)}
LO = {"H": find_homography_lo, "F": find_fundamental_lo}
MAGSAC = {"H": find_homography_magsac, "F": find_fundamental_magsac}


def gpu_info() -> dict:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (x.strip() for x in q.split(","))
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # the numbers still stand with torch's device name
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": None, "nvidia_smi_error": str(e)}


def time_gpu(fn, reps: int) -> float:
    for _ in range(3):
        fn()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(reps):
        fn()
    stop.record()
    torch.cuda.synchronize()
    return start.elapsed_time(stop) / reps


def opencv_times(key, k0, k1, m0, threads, usac=None):
    try:
        import cv2
    except ImportError:
        return None
    cv2.setNumThreads(1)
    iters, conf = DEFAULTS[key][1:]
    method = {None: cv2.RANSAC if key == "H" else cv2.FM_RANSAC, "accurate": cv2.USAC_ACCURATE,
              "magsac": cv2.USAC_MAGSAC}[usac]

    def one(b):
        v = m0[b] >= 0
        a, c = k0[b][v], k1[b][m0[b][v]]
        if key == "H":
            cv2.findHomography(a, c, method, 3.0, maxIters=iters, confidence=conf)
        else:
            cv2.findFundamentalMat(a, c, method, 3.0, conf, iters)

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
    args = ap.parse_args()
    torch.set_grad_enabled(False)
    res = {"tool": "geometry_bench", **gpu_info(), "B": args.batch, "matches": args.matches, "ransac": {}}
    threads = os.cpu_count() or 1
    for key in ("H", "F"):
        fn, iters, conf = DEFAULTS[key]
        for inl in (0.8, 0.5, 0.3):
            k0, k1, m0, _, _ = gs.batch(key, args.matches, 1.0 - inl, list(range(1000, 1000 + args.batch)),
                                        unmatched=0.0)
            t0, t1, tm = (torch.from_numpy(x).cuda() for x in (k0, k1, m0))
            row = {}
            for mode, c in (("adaptive", conf), ("full", 1.0)):
                out = fn(t0, t1, tm, confidence=c)
                row[mode] = {"gpu_ms": round(time_gpu(lambda: fn(t0, t1, tm, confidence=c), args.reps), 3),
                             "mean_hypotheses": float(out["num_hypotheses"].float().mean()),
                             "mean_inliers": float(out["num_inliers"].float().mean())}
                for name, lo in (("lo_", LO[key]), ("magsac_", MAGSAC[key])):
                    out = lo(t0, t1, tm, confidence=c)
                    row[name + mode] = {
                        "gpu_ms": round(time_gpu(lambda: lo(t0, t1, tm, confidence=c), args.reps), 3),
                        "mean_hypotheses": float(out["num_hypotheses"].float().mean()),
                        "mean_inliers": float(out["num_inliers"].float().mean()),
                        "mean_local_optimizations": float(out["num_local_optimizations"].float().mean())}
            row["opencv"] = opencv_times(key, k0, k1, m0, threads)
            row["opencv_usac_accurate"] = opencv_times(key, k0, k1, m0, threads, usac="accurate")
            row["opencv_usac_magsac"] = opencv_times(key, k0, k1, m0, threads, usac="magsac")
            res["ransac"][f"{key}_inliers{inl}"] = row
    # the matcher alone, and followed by find_fundamental on its device output (no host read-back in between)
    data, _ = synth.make_pair(2048, b=args.batch, seed=7)
    cuda = {k: {kk: vv.cuda() for kk, vv in v.items()} for k, v in data.items()}
    m = LightGlue(features=None, depth_confidence=-1, width_confidence=-1, precision="bf16x3")
    m.load_state_dict(synth.make_state_dict(), strict=False)
    m = m.eval().cuda()

    def matcher_only():
        return m.forward_async(cuda).tensors["matches0"]

    def matcher_ransac():
        m0 = m.forward_async(cuda).tensors["matches0"]
        return find_fundamental(cuda["image0"]["keypoints"], cuda["image1"]["keypoints"], m0)

    def matcher_lo_homography():
        m0 = m.forward_async(cuda).tensors["matches0"]
        return find_homography_lo(cuda["image0"]["keypoints"], cuda["image1"]["keypoints"], m0)

    def matcher_lo_fundamental():
        m0 = m.forward_async(cuda).tensors["matches0"]
        return find_fundamental_lo(cuda["image0"]["keypoints"], cuda["image1"]["keypoints"], m0)

    for name, f in (("lightglue", matcher_only), ("lightglue_plus_fundamental", matcher_ransac),
                    ("lightglue_again", matcher_only), ("lightglue_plus_homography_lo", matcher_lo_homography),
                    ("lightglue_again2", matcher_only), ("lightglue_plus_fundamental_lo", matcher_lo_fundamental),
                    ("lightglue_again3", matcher_only)):
        ms = time_gpu(f, args.steps)
        res[f"{name}_pairs_per_s"] = round(args.batch / ms * 1e3, 1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
