"""Per-image time of the DoG-HardNet extractor (lightglue_b200.DoGHardNet, synthetic HardNet weights) at 768x1024,
B = 1 and B = 4, with the default conf and with max_num_keypoints=2048, against two arms:
  * "sift": this project's SIFT alone (lightglue_b200.SIFT, same conf), so the difference is the descriptor head;
  * "reference": the unmodified reference sift.py with cv2 on the host (oracle/sift_ref_loader.py), as the reference's
    DoGHardNet runs it per image, plus oracle/doghardnet_oracle.py's patch extraction and HardNet in fp32 on the same
    GPU (cuDNN), once with TF32 off and once with it on.  Skipped where cv2 or the reference copy is missing.
Prints the card name and power limit, the executed against algorithmic multiply-adds per patch (from the layer shapes),
one JSON line per configuration, and with --stages the CUDA time per stage and per HardNet layer (torch.profiler, a
separate run)."""
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
from lightglue_b200 import SIFT, DoGHardNet  # noqa: E402
from oracle import doghardnet_oracle as dho  # noqa: E402
from oracle import doghardnet_synth as dhs  # noqa: E402
from oracle import sift_ref_loader, sift_synth  # noqa: E402

# per patch: (layer, algorithmic MAC, executed MAC).  Executed: conv 0 on CUDA cores over the 32 x 32 pixels; the tensor-
# core layers over every padded row of their output frame (34^2, 18^2, 10^2), MMA columns rounded up to 64 / 128, input
# channels to 64, and the stride-2 layers computing only the strided outputs (phase split); conv 6 one row per patch.
MACS = [
    ("conv0 1->32", 32 * 32 * 32 * 9, 32 * 32 * 32 * 9),
    ("conv1 32->32", 32 * 32 * 32 * 32 * 9, 34 * 34 * 64 * 9 * 64),
    ("conv2 32->64 s2", 16 * 16 * 64 * 32 * 9, 18 * 18 * 64 * 9 * 64),
    ("conv3 64->64", 16 * 16 * 64 * 64 * 9, 18 * 18 * 64 * 9 * 64),
    ("conv4 64->128 s2", 8 * 8 * 128 * 64 * 9, 10 * 10 * 128 * 9 * 64),
    ("conv5 128->128", 8 * 8 * 128 * 128 * 9, 10 * 10 * 128 * 9 * 128),
    ("conv6 128->128 8x8", 128 * 128 * 64, 128 * 8192),
]
STAGES = {  # kernel-name fragment -> stage
    "sift_stage": "SIFT detection (functors)",
    "sift_count": "SIFT detection (functors)",
    "dhn_gray": "gray crop + pyramid",
    "dhn_pyrdown": "gray crop + pyramid",
    "dhn_state": "row counts",
    "dhn_patch": "patch sampling + normalisation + conv0",
    "dhn_phase": "polyphase repack",
    "tc_linear_kernel": "tensor-core convolutions (conv1..conv6)",
    "dhn_gather": "conv6 row gather",
    "dhn_finish": "L2 normalisation",
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
    # tensor-core launches in issue order: conv1 .. conv5 per chunk of keypoints, then conv6 once
    tc = sorted((e for e in prof.events() if "tc_linear_kernel" in e.name), key=lambda e: e.time_range.start)
    per_layer = [0.0] * 6
    for i, e in enumerate(tc[:-1]):
        per_layer[i % 5] += e.time_range.elapsed_us() / 1000.0
    if tc:
        per_layer[5] = tc[-1].time_range.elapsed_us() / 1000.0
    acc["tensor-core ms per layer (conv1..conv6)"] = [round(v, 4) for v in per_layer]
    if sum(per_layer) > 0:
        acc["conv1 share of tensor-core time"] = round(per_layer[0] / sum(per_layer), 4)
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        prof.export_chrome_trace(os.path.join(out_dir, "doghardnet_trace.pt.trace.json"))
    return {k: (round(v, 4) if isinstance(v, float) else v) for k, v in acc.items()}


def reference_ms(conf, sd_cuda, data, tf32, n):
    """cv2 SIFT on the host per image (the reference's SIFT.extract_single_image), then the oracle's patches and HardNet
    in fp32 on the GPU."""
    sift = sift_ref_loader.build_model(**conf)
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = tf32
    try:
        for i in range(n + 1):  # the first pass is not timed (cv2 and cuDNN set-up)
            if i == 1:
                torch.cuda.synchronize()
                t = time.perf_counter()
            g = dho.gray(data["image"])
            for k in range(g.shape[0]):
                p = sift.extract_single_image(g[k])
                dho.describe_one(sd_cuda, g[k], p["keypoints"].cuda(), p["scales"].cuda(), p["oris"].cuda())
            torch.cuda.synchronize()
        return (time.perf_counter() - t) * 1000 / n / g.shape[0]
    finally:
        torch.backends.cudnn.allow_tf32 = prev


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
    alg, exe = sum(m[1] for m in MACS), sum(m[2] for m in MACS)
    print(json.dumps({"mac_per_patch": {m[0]: {"algorithmic": m[1], "executed": m[2]} for m in MACS},
                      "algorithmic_total": alg, "executed_total": exe, "executed_over_algorithmic": round(exe / alg, 3)}))
    ref_ok = sift_ref_loader.available()
    if not ref_ok:
        print("reference arm skipped: oracle/_ref/sift_ref.py or cv2 is missing")
    sd = dhs.make_state_dict(0)
    sd_cuda = {k: v.cuda() for k, v in sd.items()}
    img = sift_synth.make_image(args.h, args.w, 1, 100).cuda()
    for conf in ({}, {"max_num_keypoints": 2048}):
        ours = DoGHardNet(weights=None, **conf)
        ours.laf_desc.descriptor.load_state_dict(sd, strict=True)
        ours = ours.cuda()
        sift = SIFT(**conf)
        for b in (1, 4):
            data = {"image": img.expand(b, -1, -1, -1).contiguous()}  # equal counts across the batch
            ms, out = time_ms(lambda: ours(data), args.iters, args.warmup)
            sms, _ = time_ms(lambda: sift(data), args.iters, args.warmup)
            n = int(out["keypoints"].shape[1])
            row = {"impl": "cuda", "conf": conf, "B": b, "h": args.h, "w": args.w, "ms_per_image": round(ms / b, 3),
                   "sift_alone_ms_per_image": round(sms / b, 3), "descriptor_head_ms_per_image": round((ms - sms) / b, 3),
                   "keypoints": n, "executed_gmac_per_image": round(n * exe / 1e9, 1), "card": name, "power_limit": power}
            if ref_ok:
                for label, tf32 in (("tf32_off", False), ("tf32_on", True)):
                    row[f"reference_ms_per_image_{label}"] = round(reference_ms(conf, sd_cuda, data, tf32, 2), 1)
                row["reference"] = "reference sift.py (cv2, host) + oracle patches and HardNet, fp32, cuDNN"
            print(json.dumps(row))
            if args.stages and b == 1:
                print(json.dumps({"conf": conf, "stages_ms": stages(ours, data, args.out)}))


if __name__ == "__main__":
    main()
