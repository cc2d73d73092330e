"""ALIKED extractor timings: ms per image with CUDA events after warm-up, at 1024 x 768 (W x H), B = 1 and B = 4, for
the default conf and for max_num_keypoints = 2048, on synthetic weights (oracle/aliked_synth.py; the cost does not
depend on the weight values, only on the keypoint count, which is printed).

    python tools/aliked_bench.py [--iters 20] [--warmup 5] [--model aliked-n16]

If oracle/_ref/aliked_ref.py (``make -C oracle -f aliked_ref.mk``) and torchvision are present, the unmodified reference runs on
the same GPU (eager fp32, TF32 off) for the same inputs and the largest output differences are reported; otherwise that leg is
skipped with a message.  Prints the card name and power limit of the run, and one JSON line per configuration."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from lightglue_b200.aliked import ALIKED  # noqa: E402
from oracle import aliked_ref_loader as loader  # noqa: E402
from oracle import aliked_synth as als  # noqa: E402


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--model", default="aliked-n16")
    args = ap.parse_args()
    torch.set_grad_enabled(False)
    # the reference leg is eager fp32: no TF32 in cuDNN convolutions (PyTorch's default) or matmuls
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    name, power = card()
    print(f"card: {name}, power limit {power}")
    sd = als.make_aliked_state_dict(args.model, 0)
    ref_ok = loader.available()
    if not ref_ok:
        print("reference leg skipped: oracle/_ref/aliked_ref.py or torchvision is missing (make -C oracle -f aliked_ref.mk)")
    for conf in ({}, {"max_num_keypoints": 2048}):
        ours = ALIKED(weights=None, model_name=args.model, **conf)
        ours.load_state_dict(sd)
        ours = ours.cuda()
        ref = loader.build_model(sd, model_name=args.model, **conf).cuda() if ref_ok else None
        for b in (1, 4):
            image = als.make_image(768, 1024, b, 7).cuda()
            try:
                ms, out = time_ms(lambda: ours({"image": image}), args.iters, args.warmup)
            except ValueError:  # threshold mode on a batch: images end with different counts
                ms, out = time_ms(lambda: [ours({"image": image[i:i + 1]}) for i in range(b)], args.iters, args.warmup)
                out = out[0]
            row = {"model": args.model, "conf": conf or "default", "B": b, "H": 768, "W": 1024,
                   "ms_per_image": round(ms / b, 3), "keypoints_img0": int(out["keypoints"].shape[1]),
                   "card": name, "power_limit": power}
            if ref is not None:
                try:
                    rms, rout = time_ms(lambda: ref({"image": image}), max(2, args.iters // 4), 2)
                except RuntimeError:  # torch.stack of unequal per-image counts
                    rms, rout = time_ms(lambda: [ref({"image": image[i:i + 1]}) for i in range(b)], max(2, args.iters // 4), 2)
                    rout = rout[0]
                row["reference_ms_per_image"] = round(rms / b, 3)
                if rout["keypoints"].shape == out["keypoints"].shape:
                    row["max_diff"] = {k: float((out[k][0] - rout[k][0]).abs().max()) for k in ("keypoints", "keypoint_scores", "descriptors")}
                else:
                    row["max_diff"] = f"keypoint counts differ: {tuple(out['keypoints'].shape)} vs {tuple(rout['keypoints'].shape)}"
            print(json.dumps(row))


if __name__ == "__main__":
    main()
