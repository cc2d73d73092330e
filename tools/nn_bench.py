"""The nearest-neighbour matcher (lightglue_b200.NearestNeighborMatcher, include/nn_b200.h) against the same rules in
torch on the same GPU.

Prints one JSON line per configuration, each with the card's name and power limit read in this run:
  * GPU ms per batch of nn_match (CUDA events around `--steps` calls on preallocated buffers, after `--warmup`);
  * the torch arm: fp32 einsum into the B x M x N similarity matrix, topk(2) along both axes and a gather for the
    mutual check, with TF32 off and on;
  * the peak device memory each arm allocates beyond its inputs;
  * the executed FLOP (3 split-bf16 passes x 2 directions x 2 M N D per pair) and the algorithmic FLOP (2 M N D per pair),
    and the executed rate;
  * the share of rows of image 0 on which matches0 agrees with the torch arm in fp32.
Configurations: B = 32 pairs of 2048 keypoints at D = 256 and D = 128 (SuperPoint / DISK-sized), and B = 8 pairs of
8192 at D = 256 and 128, each with ratio_thresh = 0.8 and the mutual check.  Descriptors come from
lightglue_b200.synth.make_pair; nothing is written to disk.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from lightglue_b200 import NearestNeighborMatcher, _cabi, synth  # noqa: E402
from tools.geometry_bench import gpu_info  # noqa: E402

CONFIGS = [(32, 2048, 256), (32, 2048, 128), (8, 8192, 256), (8, 8192, 128)]
RATIO = 0.8


def time_ms(fn, steps: int, warmup: int) -> float:
    for _ in range(warmup):
        fn()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(steps):
        fn()
    stop.record()
    torch.cuda.synchronize()
    return start.elapsed_time(stop) / steps


def peak_bytes(fn) -> int:
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    keep = fn()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    del keep
    return int(peak)


def torch_nn(d0, d1, ratio):
    """Mutual nearest neighbours with the ratio test on the materialised similarity matrix."""
    r2 = ratio * ratio
    s = torch.einsum("bmd,bnd->bmn", d0, d1)
    v0, i0 = s.topk(2, dim=2)
    v1, i1 = s.topk(2, dim=1)
    m0 = torch.where(2 * (1 - v0[..., 0]) <= r2 * 2 * (1 - v0[..., 1]), i0[..., 0], -1)
    m1 = torch.where(2 * (1 - v1[:, 0]) <= r2 * 2 * (1 - v1[:, 1]), i1[:, 0], -1)
    ar0 = torch.arange(d0.shape[1], device=d0.device)[None]
    mutual0 = (m0 >= 0) & (m1.gather(1, m0.clamp(min=0)) == ar0)
    return torch.where(mutual0, m0, -1), m1


def run(b: int, n: int, d: int, steps: int, warmup: int) -> dict:
    data, _ = synth.make_pair(n, d=d, b=b, seed=2024)
    d0 = data["image0"]["descriptors"].cuda()
    d1 = data["image1"]["descriptors"].cuda()
    lib = _cabi.load()
    m = n
    outs_t = [torch.empty(b, m, dtype=torch.int64, device="cuda"), torch.empty(b, n, dtype=torch.int64, device="cuda"),
              torch.empty(b, m, device="cuda"), torch.empty(b, n, device="cuda"),
              torch.empty(b, dtype=torch.int32, device="cuda"), torch.empty(b, m, 2, dtype=torch.int64, device="cuda"),
              torch.empty(b, m, device="cuda")]
    ws = torch.empty(lib.nn_workspace_bytes(b, m, n, d), dtype=torch.uint8, device="cuda")
    handle = NearestNeighborMatcher._handle(d0.device)
    cfg = _cabi.NnConfig(_cabi.NN_ABI_VERSION, d, 1, RATIO, 0.0)
    ins = _cabi.NnInputs(b, m, n, d0.data_ptr(), d1.data_ptr(), None, None)
    outs = _cabi.NnOutputs(*(t.data_ptr() for t in outs_t))

    def ours():
        stream = torch.cuda.current_stream().cuda_stream
        _cabi.check(lib.nn_match(handle, C.byref(cfg), C.byref(ins), C.byref(outs), ws.data_ptr(), ws.numel(), stream),
                    "nn_match")

    def ours_alloc():  # what a call needs beyond its inputs: the outputs and the workspace
        o = [torch.empty_like(t) for t in outs_t]
        w = torch.empty(ws.numel(), dtype=torch.uint8, device="cuda")
        return o, w

    ms = time_ms(ours, steps, warmup)
    mine = outs_t[0].clone()
    res = {"B": b, "M": m, "N": n, "D": d, "ratio_thresh": RATIO, "mutual_check": True, "nn_ms": round(ms, 3),
           "nn_peak_bytes": peak_bytes(ours_alloc), "nn_workspace_bytes": ws.numel()}
    for tf32 in (False, True):
        torch.backends.cuda.matmul.allow_tf32 = tf32
        key = "torch_tf32" if tf32 else "torch_fp32"
        res[key + "_ms"] = round(time_ms(lambda: torch_nn(d0, d1, RATIO), steps, warmup), 3)
        res[key + "_peak_bytes"] = peak_bytes(lambda: torch_nn(d0, d1, RATIO))
        if not tf32:
            ref = torch_nn(d0, d1, RATIO)[0]
            res["matches0_agree_fp32"] = round(float((ref == mine).double().mean()), 6)
    torch.backends.cuda.matmul.allow_tf32 = False
    algo = 2.0 * b * m * n * d
    res["algorithmic_flop"] = algo
    res["executed_flop"] = 6 * algo
    res["executed_tflops"] = round(6 * algo / (ms * 1e-3) / 1e12, 1)
    res["similarity_matrix_bytes"] = b * m * n * 4
    return res


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("nn_bench needs a CUDA device")
    info = gpu_info()
    for b, n, d in CONFIGS:
        print(json.dumps({**info, **run(b, n, d, args.steps, args.warmup)}), flush=True)


if __name__ == "__main__":
    main()
