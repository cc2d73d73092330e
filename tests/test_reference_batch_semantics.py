"""What the reference does with adaptive depth on a batch of more than one pair -- results of the UNMODIFIED reference
file stored in tests/golden/batch_semantics/ref_batch_semantics.pt (oracle/make_golden_batch_semantics.py, CPU) -- and therefore why
lightglue_b200 decides per pair (documented deviation, LightGlue.forward docstring, INTEGRATION.md).

lightglue.py:645-656 (`check_if_stop`): the low-confidence count is summed over the WHOLE batch and divided by ONE pair's
m + n, and one decision is taken for all pairs.  So a pair's result depends on its batch-mates -- even on being duplicated:
two copies of a pair that stops early alone run all nine layers together, with different matches.  (With point pruning on,
`torch.where(mask)[1]` at 554 / 562 additionally concatenates the kept columns of all rows: not defined for B > 1.)"""
import os

import torch

from lightglue_b200 import synth
from oracle import lightglue_oracle as oracle
from oracle.make_golden_batch_semantics import RECIPE, checksum


def _golden(golden_dir):
    g = torch.load(os.path.join(golden_dir, "batch_semantics", "ref_batch_semantics.pt"), weights_only=False)
    assert g["recipe"] == RECIPE
    return g


def test_reference_batched_early_exit_depends_on_batch_mates(golden_dir):
    g = _golden(golden_dir)
    alone41, alone42, twice, mixed = g["alone41"], g["alone42"], g["twice41"], g["mixed41_42"]
    assert alone41["stop"] < alone42["stop"] == 9  # one pair exits early, the other never
    assert twice["stop"] == 9 > alone41["stop"]    # the SAME pair twice no longer exits: count summed over the batch
    assert not torch.equal(twice["matches0"][0], alone41["matches0"][0])  # and its matches changed with it
    assert torch.equal(twice["matches0"][0], twice["matches0"][1])
    assert mixed["stop"] == 9  # one batch-global decision: pair 41 is dragged along


def test_per_pair_decision_matches_reference_on_each_pair_alone(golden_dir):
    """The project's rule (every pair decides for itself) is the reference's answer for that pair run alone."""
    torch.set_grad_enabled(False)
    g = _golden(golden_dir)
    sd = synth.make_state_dict(adaptive=True, seed=RECIPE["weight_seed"])
    assert abs(sum(checksum(v) for v in sd.values()) - g["checksums"]["weights"]) <= 1e-6 * g["checksums"]["weights"]
    for seed in RECIPE["seeds"]:
        data = synth.make_pair(RECIPE["n"], b=1, seed=seed)[0]
        assert checksum(data["image0"]["keypoints"]) == g["checksums"][f"kpts{seed}"]
        out = oracle.forward(sd, data, depth_confidence=RECIPE["depth_confidence"], width_confidence=RECIPE["width_confidence"])
        ref = g[f"alone{seed}"]
        assert int(out["stop"]) == ref["stop"]
        assert torch.equal(out["matches0"], ref["matches0"])
        assert float((out["matching_scores0"] - ref["matching_scores0"]).abs().max()) < 1e-4
