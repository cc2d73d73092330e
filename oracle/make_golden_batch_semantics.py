"""Generate tests/golden/batch_semantics/ref_batch_semantics.pt: what the UNMODIFIED reference matcher does with adaptive depth on
batches of more than one pair (tests/test_reference_batch_semantics.py).

    python oracle/make_golden_batch_semantics.py      # needs the reference project (see make_golden.py); CPU, fp32

Inputs and weights are regenerated from their seeds (``lightglue_b200.synth``); the fixture keeps the recipe, checksums
of the regenerated inputs / weights and the reference's outputs for pair 41 alone, pair 42 alone, pair 41 twice in one
batch and the batch [41, 42].
"""
from __future__ import annotations

import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from lightglue_b200 import synth  # noqa: E402
from oracle.make_golden import load_reference  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "batch_semantics", "ref_batch_semantics.pt")
RECIPE = dict(weight_seed=2, n=192, seeds=(41, 42), depth_confidence=0.95, width_confidence=-1)


def checksum(t: torch.Tensor) -> float:
    return float(t.double().abs().sum())


def cat(pairs):
    return {k: {kk: torch.cat([p[k][kk] for p in pairs]) for kk in pairs[0][k]} for k in ("image0", "image1")}


def main():
    torch.set_grad_enabled(False)
    mod = load_reference()
    sd = synth.make_state_dict(adaptive=True, seed=RECIPE["weight_seed"])
    ref = mod.LightGlue(features=None, depth_confidence=RECIPE["depth_confidence"], width_confidence=RECIPE["width_confidence"])
    missing, unexpected = ref.load_state_dict(sd, strict=False)
    assert not unexpected and all(k == "confidence_thresholds" for k in missing)
    ref = ref.eval()
    p41, p42 = (synth.make_pair(RECIPE["n"], b=1, seed=s)[0] for s in RECIPE["seeds"])
    runs = {"alone41": [p41], "alone42": [p42], "twice41": [p41, p41], "mixed41_42": [p41, p42]}
    out = {"recipe": RECIPE,
           "checksums": {"weights": sum(checksum(v) for v in sd.values()),
                         "kpts41": checksum(p41["image0"]["keypoints"]), "kpts42": checksum(p42["image0"]["keypoints"])}}
    for name, pairs in runs.items():
        r = ref(cat(pairs))
        out[name] = {"stop": int(r["stop"]), "matches0": r["matches0"].clone(), "matching_scores0": r["matching_scores0"].clone()}
    torch.save(out, OUT)
    print("wrote", OUT, {k: v["stop"] for k, v in out.items() if isinstance(v, dict) and "stop" in v})


if __name__ == "__main__":
    main()
