"""Per-image time of the DISK extractor (lightglue_b200.DISK, synthetic weights) at 768x1024, B = 1 and B = 4, with the
default conf and with max_num_keypoints=2048, against the comparison arm "oracle (kornia's DISK restated)":
oracle/disk_oracle.py in fp32 on the same GPU (cuDNN), once with TF32 off and once with torch's default (cuDNN TF32 on).
Prints the card name and power limit, one JSON line per configuration, and with --stages the CUDA time per stage
(torch.profiler, a separate run)."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from lightglue_b200.disk import DISK  # noqa: E402
from oracle import disk_oracle as do  # noqa: E402
from oracle import disk_synth as ds  # noqa: E402

STAGES = {  # kernel-name fragment -> stage
    "disk_stats": "instance-norm statistics",
    "disk_apply": "prepare (pool / upsample, normalise, PReLU)",
    "disk_down0": "down0 (CUDA cores)",
    "tc_linear_kernel": "tensor-core convolutions + descriptor GEMM",
    "disk_heatmap": "heatmap channel (CUDA cores)",
    "disk_nms": "NMS",
    "sp_row": "candidate compaction",
    "kp_select": "top-k",
    "disk_gather": "descriptor im2col gather",
    "disk_finish": "descriptor normalisation",
}


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
        for frag, stage in STAGES.items():
            if frag in e.key:
                acc[stage] = acc.get(stage, 0.0) + e.device_time_total / 1000.0
    # the tensor-core launches in issue order: down1 .. down4, up0 .. up2, descriptor head
    tc = sorted((e for e in prof.events() if "tc_linear_kernel" in e.name), key=lambda e: e.time_range.start)
    acc["tensor-core launches, in order"] = [round(e.time_range.elapsed_us() / 1000.0, 4) for e in tc]
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        prof.export_chrome_trace(os.path.join(out_dir, "disk_trace.pt.trace.json"))
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
    sd = ds.make_disk_state_dict(0)
    sd_cuda = {k: v.cuda() for k, v in sd.items()}
    img = ds.make_image(args.h, args.w, 1, 100).cuda()
    for conf in ({}, {"max_num_keypoints": 2048}):
        ours = DISK(weights=None, **conf)
        ours.model.load_state_dict(sd, strict=True)
        ours = ours.cuda()
        for b in (1, 4):
            data = {"image": img.expand(b, -1, -1, -1).contiguous()}  # equal counts across the batch
            ms, out = time_ms(lambda: ours(data), args.iters, args.warmup)
            row = {"impl": "cuda", "conf": conf, "B": b, "h": args.h, "w": args.w, "ms_per_image": ms / b,
                   "keypoints": int(out["keypoints"].shape[1]), "card": name, "power_limit": power}
            for label, tf32 in (("tf32_off", False), ("tf32_default", torch.backends.cudnn.allow_tf32)):
                prev = torch.backends.cudnn.allow_tf32
                torch.backends.cudnn.allow_tf32 = tf32
                try:
                    oms, _ = time_ms(lambda: do.forward(sd_cuda, data["image"], conf), max(3, args.iters // 4), 2)
                finally:
                    torch.backends.cudnn.allow_tf32 = prev
                row[f"oracle_ms_per_image_{label}"] = oms / b
            row["oracle"] = "oracle (kornia's DISK restated), fp32, cuDNN"
            print(json.dumps(row))
            if args.stages and b == 1:
                print(json.dumps({"conf": conf, "stages_ms": stages(ours, data, args.out)}))


if __name__ == "__main__":
    main()
