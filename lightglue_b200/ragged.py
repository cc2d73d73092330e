"""Ragged batches: pairs with different keypoint counts matched in one launch sequence (SURVEY 8f2).

The reference can only batch pairs of equal size; its ``compile()`` path pads every image to a static
length with ones and threads boolean masks through ``masked_forward`` (lightglue.py:46-55, 256-262,
512-520).  The kernels here read each sequence's length from device memory, so padding rows are simply
never touched: ``pad_pairs`` stacks B single-pair feature dicts into one padded batch that carries
``num_keypoints``, ``LightGlue.forward`` passes the counts through the C ABI (``LgInputs.lens0/lens1``),
and ``split_outputs`` cuts the result back into per-pair dicts shaped like B=1 calls of the reference.
"""
from __future__ import annotations

from typing import Dict, List, Sequence

import torch

_PER_POINT = ("keypoints", "descriptors", "scales", "oris")


def _first(t: torch.Tensor) -> torch.Tensor:
    """[1, n, ...] or [n, ...] -> [n, ...] (the extractors return a leading batch dimension of 1)."""
    if t.dim() == 3:
        assert t.shape[0] == 1, "ragged batches are built from single pairs"
        return t[0]
    return t


def _stack_image(feats: Sequence[dict], device) -> dict:
    b = len(feats)
    kp = [_first(f["keypoints"]) for f in feats]
    counts = [int(k.shape[0]) for k in kp]
    width = max(counts) if counts else 0
    out = {"num_keypoints": torch.tensor(counts, dtype=torch.int32, device=device)}
    for key in _PER_POINT:
        if key not in feats[0]:
            continue
        rows = [_first(f[key]) if key in ("keypoints", "descriptors") else f[key].reshape(-1) for f in feats]
        tail = rows[0].shape[1:]
        slab = torch.zeros((b, width) + tuple(tail), dtype=torch.float32, device=device)
        for i, r in enumerate(rows):
            if r.shape[0]:
                slab[i, : r.shape[0]] = r.to(device=device, dtype=torch.float32)
        out[key] = slab
    has_size = ["image_size" in f and f["image_size"] is not None for f in feats]
    if any(has_size):
        if not all(has_size):
            raise ValueError("image_size must be given for every pair of a ragged batch or for none")
        out["image_size"] = torch.stack(
            [torch.as_tensor(f["image_size"], dtype=torch.float32).reshape(-1)[:2] for f in feats]
        ).to(device)
    return out


def pad_pairs(pairs: Sequence[dict], device=None) -> dict:
    """``[{"image0": feats0, "image1": feats1}, ...]`` (each a single pair, keypoints ``[n,2]`` or
    ``[1,n,2]``) -> one batched ``data`` dict with zero padding and ``num_keypoints`` per image."""
    if not pairs:
        raise ValueError("pad_pairs needs at least one pair")
    if device is None:
        device = pairs[0]["image0"]["keypoints"].device
    return {
        "image0": _stack_image([p["image0"] for p in pairs], device),
        "image1": _stack_image([p["image1"] for p in pairs], device),
    }


def split_outputs(out: dict, lens0, lens1) -> List[Dict]:
    """Cut a ragged batch's result into per-pair dicts with the reference's B=1 shapes
    (``matches0 [1, m_b]`` ..., ``matches``/``scores`` one-element lists)."""
    lens0 = [int(v) for v in (lens0.tolist() if torch.is_tensor(lens0) else lens0)]
    lens1 = [int(v) for v in (lens1.tolist() if torch.is_tensor(lens1) else lens1)]
    res = []
    lists = isinstance(out["matches"], (list, tuple))
    for b, (m, n) in enumerate(zip(lens0, lens1)):
        pair = {
            "matches0": out["matches0"][b : b + 1, :m],
            "matches1": out["matches1"][b : b + 1, :n],
            "matching_scores0": out["matching_scores0"][b : b + 1, :m],
            "matching_scores1": out["matching_scores1"][b : b + 1, :n],
            "matches": [out["matches"][b]] if lists else out["matches"][b : b + 1],
            "scores": [out["scores"][b]] if lists else out["scores"][b : b + 1],
        }
        if "prune0" in out:  # LightGlue's adaptive-depth keys; a matcher without layers has none
            pair["prune0"] = out["prune0"][b : b + 1, :m]
            pair["prune1"] = out["prune1"][b : b + 1, :n]
        if "stops" in out or "stop" in out:
            pair["stop"] = int(out["stops"][b]) if "stops" in out else out["stop"]
        res.append(pair)
    return res


def match_ragged(matcher, pairs: Sequence[dict]) -> List[Dict]:
    """Match a list of single pairs of arbitrary sizes with one forward call."""
    data = pad_pairs(pairs)
    out = matcher(data)
    return split_outputs(out, data["image0"]["num_keypoints"], data["image1"]["num_keypoints"])
