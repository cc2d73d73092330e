"""Guided nearest-neighbour matching (NearestNeighborMatcher.forward(..., F= / H=), include/nn_b200.h) against the
unguided matcher and against the same guided rules restated in torch on the same GPU.

Prints one JSON line per configuration, each with the card's name and power limit read in this run:
  * GPU ms per call of the unguided forward, the guided forward under H and under F, and the torch arm under H and F
    (fp32 bmm into the B x M x N similarity matrix with TF32 off, the fp32 gate of include/geometry_b200.h step 5 as a
    B x M x N mask, topk(2) along both axes and the mutual check), medians over --reps rounds of --steps calls after
    --warmup, the arms alternating within each round;
  * find_fundamental_lo followed by the guided forward under its F, as one pipeline;
  * the share of decided rows (top-1 gap above 2e-4 and ratio margin above 4e-4 in the torch arm, on both sides of a
    mutual match) on which matches0 equals the torch arm's, per model.
Configurations: B = 32 pairs of 2048 keypoints at D = 128 and D = 256, and B = 8 pairs of 8192 at D = 128, ratio 0.8,
the mutual check, max_error 4 px.  Scenes: half of image 1 are noisy copies of image-0 descriptors placed where the
pair's model puts their keypoints (within about a pixel), the rest random; nothing is written to disk.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from lightglue_b200 import NearestNeighborMatcher  # noqa: E402
from lightglue_b200.geometry import find_fundamental_lo  # noqa: E402
from oracle import geometry_synth as gs  # noqa: E402
from tools.geometry_bench import gpu_info  # noqa: E402

CONFIGS = [(32, 2048, 128), (32, 2048, 256), (8, 8192, 128)]
RATIO, MAX_ERROR = 0.8, 4.0


def scene(b: int, n: int, d: int, seed: int):
    g = np.random.default_rng(seed)
    d0 = torch.randn(b, n, d, generator=torch.Generator().manual_seed(seed))
    d1 = torch.randn(b, n, d, generator=torch.Generator().manual_seed(seed + 1))
    k = n // 2
    d1[:, :k] = d0[:, :k] + 0.4 * torch.randn(b, k, d, generator=torch.Generator().manual_seed(seed + 2))
    d0, d1 = torch.nn.functional.normalize(d0, dim=-1), torch.nn.functional.normalize(d1, dim=-1)
    k0 = g.uniform([0, 0], [640, 480], (b, n, 2))
    k1 = g.uniform([0, 0], [640, 480], (b, n, 2))
    Hs = np.stack([gs.true_homography(g) for _ in range(b)])
    Fs = np.stack([gs.two_view(8, 0.0, int(s))[4] for s in g.integers(0, 1000, b)])
    k1h, k1f = k1.copy(), k1.copy()
    for p in range(b):  # the copies where each model puts their image-0 keypoints
        k1h[p, :k] = gs.apply_h(Hs[p], k0[p, :k]) + g.normal(0, 0.7, (k, 2))
        ln = np.concatenate([k0[p, :k], np.ones((k, 1))], 1) @ Fs[p].T
        r = (ln[:, :2] * k1[p, :k]).sum(1) + ln[:, 2]
        k1f[p, :k] = k1[p, :k] - (r / (ln[:, :2] ** 2).sum(1))[:, None] * ln[:, :2] + g.normal(0, 0.5, (k, 2))
    cuda = lambda x: torch.as_tensor(x).cuda()  # noqa: E731
    return (cuda(d0), cuda(d1), cuda(k0).float(), cuda(k1h).float(), cuda(k1f).float(), cuda(Hs), cuda(Fs))


def torch_gate(kind: str, model: torch.Tensor, k0: torch.Tensor, k1: torch.Tensor, t2: float) -> torch.Tensor:
    """[B, M, N] err < t2 in fp32, one eager operation per step of include/geometry_b200.h step 5."""
    h = model.float().reshape(-1, 9)
    g = [h[:, i, None, None] for i in range(9)]
    x0, y0 = k0[:, :, 0, None], k0[:, :, 1, None]
    x1, y1 = k1[:, None, :, 0], k1[:, None, :, 1]
    if kind == "H":
        w = 1.0 / ((g[6] * x0 + g[7] * y0) + g[8])
        dx = x1 - ((g[0] * x0 + g[1] * y0) + g[2]) * w
        dy = y1 - ((g[3] * x0 + g[4] * y0) + g[5]) * w
        return dx * dx + dy * dy < t2
    a, b, c = (g[0] * x0 + g[1] * y0) + g[2], (g[3] * x0 + g[4] * y0) + g[5], (g[6] * x0 + g[7] * y0) + g[8]
    d2, s2 = (x1 * a + y1 * b) + c, 1.0 / (a * a + b * b)
    a, b, c = (g[0] * x1 + g[3] * y1) + g[6], (g[1] * x1 + g[4] * y1) + g[7], (g[2] * x1 + g[5] * y1) + g[8]
    d1, s1 = (x0 * a + y0 * b) + c, 1.0 / (a * a + b * b)
    return torch.fmax(d1 * d1 * s1, d2 * d2 * s2) < t2


def torch_guided(d0, d1, k0, k1, model, kind):
    """The guided rules in torch: returns matches0 and the decided-row mask of image 0."""
    r2 = float(np.float32(float(np.float32(RATIO)) ** 2))
    t2 = float(np.float32(MAX_ERROR * MAX_ERROR))
    S = torch.bmm(d0, d1.transpose(1, 2)).masked_fill_(~torch_gate(kind, model, k0, k1, t2), -float("inf"))

    def side(S):
        v, j = S.topk(2, dim=2)
        s1, s2 = v[..., 0], v[..., 1]
        D1, D2 = 2 * (1 - s1), 2 * (1 - s2)
        keep = (s1 > -float("inf")) & (D1 <= r2 * D2)
        sure = ((s1 - s2) > 2e-4) & (((D1 - r2 * D2).abs() > 4e-4) | (s2 == -float("inf")))
        return torch.where(keep, j[..., 0], -1), sure | (s1 == -float("inf"))

    j0, sure0 = side(S)
    i1, sure1 = side(S.transpose(1, 2))
    ar = torch.arange(S.shape[1], device=S.device)
    back = torch.gather(i1, 1, j0.clamp(min=0))
    m0 = torch.where((j0 >= 0) & (back == ar), j0, -1)
    sure = sure0 & torch.where(j0 >= 0, torch.gather(sure1, 1, j0.clamp(min=0)), True)
    return m0, sure


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.set_grad_enabled(False)
    info = gpu_info()
    nnm = NearestNeighborMatcher(ratio_thresh=RATIO, mutual_check=True)
    for b, n, d in CONFIGS:
        d0, d1, k0, k1h, k1f, Hs, Fs = scene(b, n, d, seed=b * n + d)
        dh = {"image0": {"descriptors": d0, "keypoints": k0}, "image1": {"descriptors": d1, "keypoints": k1h}}
        df = {"image0": {"descriptors": d0, "keypoints": k0}, "image1": {"descriptors": d1, "keypoints": k1f}}
        m0_seed = nnm(df)["matches0"]

        def pipeline():
            geo = find_fundamental_lo(k0, k1f, m0_seed)
            return nnm(df, F=geo["F"], valid=geo["success"], max_error=MAX_ERROR)

        arms = {
            "unguided": lambda: nnm(df),
            "guided_H": lambda: nnm(dh, H=Hs, max_error=MAX_ERROR),
            "guided_F": lambda: nnm(df, F=Fs, max_error=MAX_ERROR),
            "torch_H": lambda: torch_guided(d0, d1, k0, k1h, Hs, "H"),
            "torch_F": lambda: torch_guided(d0, d1, k0, k1f, Fs, "F"),
            "fundamental_lo+guided_F": pipeline,
        }
        times = {k: [] for k in arms}
        for fn in arms.values():
            for _ in range(args.warmup):
                fn()
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(args.reps):
            for k, fn in arms.items():
                torch.cuda.synchronize()
                start.record()
                for _ in range(args.steps):
                    fn()
                stop.record()
                torch.cuda.synchronize()
                times[k].append(start.elapsed_time(stop) / args.steps)
        agree = {}
        for kind, data, kk1, model in (("H", dh, k1h, Hs), ("F", df, k1f, Fs)):
            got = nnm(data, **{kind: model}, max_error=MAX_ERROR)["matches0"]
            want, sure = torch_guided(d0, d1, k0, kk1, model, kind)
            agree[kind] = {"decided_rows": int(sure.sum()), "equal_on_decided": float((got == want)[sure].float().mean()),
                           "matches": int((got >= 0).sum())}
        torch.cuda.empty_cache()
        print(json.dumps({**info, "B": b, "M": n, "N": n, "D": d, "ratio": RATIO, "max_error": MAX_ERROR,
                          "ms": {k: round(statistics.median(v), 3) for k, v in times.items()},
                          "ms_spread": {k: [round(min(v), 3), round(max(v), 3)] for k, v in times.items()},
                          "agreement": agree}), flush=True)


if __name__ == "__main__":
    main()
