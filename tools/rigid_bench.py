"""Batched GPU 3D rigid and similarity estimation (lightglue_b200.geometry.estimate_rigid_3d and
estimate_similarity_3d) against a batched torch RANSAC on the same GPU.

Prints one JSON line:
  * the card's name and power limit, read in this run;
  * GPU ms per batch (CUDA events) at B pairs of M putative 3D-3D matches and 20 / 50 / 70 % outliers, for both models
    (1000 iterations, confidence 0.99, a 3 cm threshold on 1 cm noise), with adaptive stopping ("adaptive") and with
    confidence 1 ("full", all 1000 samples);
  * the same budget as a torch RANSAC a user would otherwise write: all samples of the batch at once, Kabsch or
    Umeyama by torch.linalg.svd in float64, inlier counts by one batched distance test, then the SVD fit on the best
    sample's inliers ("torch_full"; it has no adaptive stop);
  * whether the GPU outputs at the timed size equal the numpy oracle's (oracle/rigid_oracle.py) on the first pairs.
The scenes come from oracle/rigid_oracle.scene (depth-camera volume, no unmatched rows); nothing is written to disk.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from lightglue_b200.geometry import estimate_rigid_3d, estimate_similarity_3d  # noqa: E402
from oracle import rigid_oracle as ro  # noqa: E402
from tools.geometry_bench import gpu_info, time_gpu  # noqa: E402

MODELS = {"rigid": (ro.RIGID, estimate_rigid_3d), "similarity": (ro.SIMILARITY, estimate_similarity_3d)}
THR, ITERS = 0.03, 1000


def torch_fit(src, dst, w, with_scale):
    """Weighted Umeyama (Kabsch without scale) by torch.linalg.svd: src, dst [..., n, 3], w [..., n] -> R, t, s."""
    wn = w / w.sum(-1, keepdim=True).clamp_min(1)
    ms, md = (wn[..., None] * src).sum(-2), (wn[..., None] * dst).sum(-2)
    a, b = src - ms[..., None, :], dst - md[..., None, :]
    cov = (wn[..., None] * b).transpose(-1, -2) @ a
    U, D, Vt = torch.linalg.svd(cov)
    d = torch.sign(torch.linalg.det(U @ Vt))
    E = torch.ones_like(D)
    E[..., 2] = d
    R = (U * E[..., None, :]) @ Vt
    if with_scale:
        s = (D * E).sum(-1) / (wn * (a * a).sum(-1)).sum(-1)
    else:
        s = torch.ones_like(D[..., 0])
    t = md - s[..., None] * (R @ ms[..., None])[..., 0]
    return R, t, s


def torch_ransac(p0, p1, m0, with_scale, iters=ITERS, thr=THR, seed=0):
    """The RANSAC a user would write in torch: iters 3-point samples per pair, all fitted and scored at once."""
    B, M = m0.shape
    g = torch.Generator(device=p0.device).manual_seed(seed)
    valid = (m0 >= 0).double()
    src = p0.double()
    dst = torch.gather(p1.double(), 1, m0.clamp_min(0)[..., None].expand(-1, -1, 3))
    idx = torch.multinomial(valid.repeat_interleave(iters, 0), 3, generator=g).view(B, iters, 3)
    bi = torch.arange(B, device=p0.device)[:, None, None]
    R, t, s = torch_fit(src[bi, idx], dst[bi, idx], torch.ones(B, iters, 3, device=p0.device, dtype=torch.float64),
                        with_scale)
    pred = s[..., None, None] * torch.einsum("bhij,bnj->bhni", R, src) + t[:, :, None]
    inl = ((pred - dst[:, None]) ** 2).sum(-1).lt(thr * thr) & (valid[:, None] > 0)
    best = inl.sum(-1).argmax(-1)
    w = inl[torch.arange(B, device=p0.device), best].double()
    return torch_fit(src, dst, w, with_scale)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--matches", type=int, default=2048)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--check-pairs", type=int, default=4)
    args = ap.parse_args()
    torch.set_grad_enabled(False)
    res = {"tool": "rigid_bench", **gpu_info(), "B": args.batch, "matches": args.matches}
    for model, (kind, fn) in MODELS.items():
        res[model] = {}
        for o in (0.2, 0.5, 0.7):
            scenes = [ro.scene(kind, args.matches, o, 1000 + b, noise=0.01, unmatched=0.0) for b in range(args.batch)]
            p0, p1, m0 = (np.stack([sc[i] for sc in scenes]) for i in range(3))
            t0, t1, tm = (torch.from_numpy(x).cuda() for x in (p0, p1, m0))
            row = {}
            for mode, c in (("adaptive", 0.99), ("full", 1.0)):
                out = fn(t0, t1, tm, THR, max_iters=ITERS, confidence=c)
                got = {k: v.cpu().numpy() for k, v in out.items()}
                same = True
                for b in range(min(args.check_pairs, args.batch)):
                    r = ro.estimate_pair(kind, p0[b], p1[b], m0[b], THR, ITERS, c)
                    same &= all(got[k][b] == r[k] for k in ("best_hypothesis", "num_hypotheses", "num_inliers"))
                    same &= bool(np.array_equal(got["inliers"][b], r["inliers"]))
                    same &= all(np.abs(got[k][b] - r[k]).max() <= 1e-8 * max(np.abs(r[k]).max(), 1e-300)
                                for k in ("R", "t", "scale"))
                row[mode] = {"gpu_ms": round(time_gpu(lambda: fn(t0, t1, tm, THR, max_iters=ITERS, confidence=c),
                                                      args.reps), 3),
                             "mean_samples": float(out["num_hypotheses"].float().mean()),
                             "mean_inliers": float(out["num_inliers"].float().mean()),
                             "equals_oracle": bool(same)}
            row["torch_full"] = {"gpu_ms": round(time_gpu(lambda: torch_ransac(t0, t1, tm, kind == ro.SIMILARITY),
                                                          max(3, args.reps // 4)), 3)}
            res[model][f"outliers{o}"] = row
    print(json.dumps(res))


if __name__ == "__main__":
    main()
