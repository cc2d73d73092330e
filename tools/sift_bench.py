"""Per-image time of the SIFT extractor (lightglue_b200.SIFT, default conf) at 768x1024, B = 1 and B = 4, against the
reference arm: the unmodified reference sift.py (oracle/_ref/sift_ref.py) with cv2 on the host, fed from the GPU as
its users do.  The reference arm is skipped where cv2 or the copy is missing.  Prints the card name and power limit,
one JSON line per configuration, and with --stages the CUDA time per kernel class (torch.profiler, separate run)."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from lightglue_b200.sift import SIFT  # noqa: E402
from oracle import sift_ref_loader as loader  # noqa: E402
from oracle import sift_synth  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def time_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        out = fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters, out


def stages(model, data, out_dir):
    from torch.profiler import ProfilerActivity, profile

    model(data)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        model(data)
        torch.cuda.synchronize()
    acc = {}
    for e in prof.key_averages():
        name = e.key
        for tag in ("SiftGray", "SiftUpsample", "SiftRowBlur", "SiftColBlur", "SiftDecimate", "SiftDetect", "SiftOrient",
                    "SiftSortLex", "SiftRetain", "SiftDogFilter", "SiftNms", "SiftSelect", "SiftDescribe"):
            if tag in name:
                acc[tag] = acc.get(tag, 0.0) + e.device_time_total / 1000.0
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        prof.export_chrome_trace(os.path.join(out_dir, "sift_trace.pt.trace.json"))
    return acc


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--h", type=int, default=768)
    ap.add_argument("--w", type=int, default=1024)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--stages", action="store_true")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    torch.set_grad_enabled(False)
    name, power = card()
    print(f"card: {name}, power limit {power}")
    ref_ok = loader.available()
    if not ref_ok:
        print("reference arm skipped: oracle/_ref/sift_ref.py or cv2 is missing")
    ours = SIFT()
    for b in (1, 4):
        img = sift_synth.make_image(args.h, args.w, b, 100).cuda()
        data = {"image": img}
        if b > 1:  # equal counts across the batch: the same image b times
            data = {"image": img[:1].expand(b, -1, -1, -1).contiguous()}
        ms, out = time_ms(lambda: ours(data), args.iters, args.warmup)
        row = {"impl": "cuda", "B": b, "h": args.h, "w": args.w, "ms_per_image": ms / b,
               "keypoints": int(out["keypoints"].shape[1]), "card": name, "power_limit": power}
        if ref_ok:
            ref = loader.build_model()
            t = time.perf_counter()
            n_ref = 3
            for _ in range(n_ref):
                r = ref(data)
                torch.cuda.synchronize()
            row["ref_ms_per_image"] = (time.perf_counter() - t) * 1000 / n_ref / b
            row["ref_keypoints"] = int(r["keypoints"].shape[1])
            import cv2

            row["cv2"] = cv2.__version__
            row["ref_threads"] = cv2.getNumThreads()
        print(json.dumps(row))
        if args.stages and b == 1:
            print(json.dumps({"stages_ms": stages(ours, data, args.out)}))


if __name__ == "__main__":
    main()
