"""Certificates for the adaptive cases of tests/test_gpu_adaptive_batches.py (CPU only).

Early exit and point pruning are threshold decisions: a token confidence against thr_i, a matchability against
1 - width_confidence, a count of low-confidence points against (1 - depth_confidence)(m + n).  A kernel whose
arithmetic differs from float64 in the last bits may take a decision the other way when a value sits on its threshold,
and then stop, prune0/1 and the matches differ for reasons that say nothing about the kernel being right.  So the GPU
test compares with the oracle only on pairs whose every decision is at least DELTA from its threshold and whose
count is at least one point from the stop boundary.  This file pins those pairs and shows that the margin is enough:

* every pinned case certifies in float64, and the fp32 oracle takes the same decisions and matches;
* the oracle with the tensor-core rounding emulated (split-bf16 linears, fp16 q, k, v and P; oracle/tc_emulation.py)
  takes the same decisions and matches, and moves no token confidence or matchability by more than a quarter of its
  own float64 distance from the threshold.

Recorded on the pinned cases: smallest margin 1.01e-4 (w3_th-1 256x257), smallest count slack 1.0 point (w2_th256
65x255); the emulated rounding uses at most 0.16 of a margin (w2_th256 2x127) and 0.08 elsewhere.
"""
import functools
import math

import pytest
import torch

from lightglue_b200 import synth
from oracle import lightglue_oracle as oracle
from oracle.tc_emulation import BF16X3, emulated

DEPTH, WIDTH = 0.95, 0.99
DELTA = 1e-4

# name -> (weight seed of make_state_dict(adaptive=True), pruning threshold, [(m, n, pair seed), ...]).
# w2_th256: sizes on both sides of the 64- and 128-row edges and of the threshold, an empty image, pairs that stop
# after 6 layers beside pairs that run all 9, and 256 x 300 (one image never prunes, the other does).
# w3_th-1: 2 x 300 prunes image 0 to zero points and ends after layer 4 while the rest of the batch runs to 6
# (1 x 64 loses its point at layer 4 and ends with them); neither is the batch's first pair.
RAGGED = {
    "w2_th256": (2, 256, [(0, 65, 1), (1, 63, 6), (2, 127, 4), (64, 128, 1), (65, 255, 5), (129, 257, 4),
                          (257, 129, 1), (256, 300, 1), (256, 300, 16), (383, 640, 1), (640, 383, 6)]),
    "w3_th-1": (3, -1, [(128, 383, 6), (2, 300, 692), (1, 64, 3), (300, 2, 7), (256, 257, 1)]),
}
# one dense batch of four 512 x 512 pairs, pruning from the first layer
DENSE = (2, -1, [(512, 512, s) for s in (2, 5, 7, 14)])

CASES = sorted({(ws, th) + c for ws, th, cs in list(RAGGED.values()) + [DENSE] for c in cs if c[0] and c[1]})


@functools.lru_cache(maxsize=None)
def state_dict(ws):
    return synth.make_state_dict(seed=ws, adaptive=True)


def single_pair(m, n, seed):
    """One pair of m and n points as make_pair draws it (batch dimension 1)."""
    return synth.make_pair(n, m=m, seed=seed)[0]


def run(ws, th, m, n, seed, dtype=torch.float64):
    return oracle.forward(state_dict(ws), single_pair(m, n, seed), depth_confidence=DEPTH, width_confidence=WIDTH,
                          pruning_threshold=th, dtype=dtype, return_decisions=True)


@functools.lru_cache(maxsize=None)
def reference(ws, th, m, n, seed):
    """The float64 oracle's result for one pinned pair alone (cached: the GPU tests compare several forwards with it)."""
    return run(ws, th, m, n, seed)


def pruned_to_zero(ref) -> bool:
    """Some pruning step of this pair kept no point of one image."""
    for d in ref.get("decisions", []):
        for k, t in (("mat0", "tok0"), ("mat1", "tok1")):
            if k in d and not bool(((d[k] > 1 - WIDTH) | (d[t] <= d["thr"])).any()):
                return True
    return False


def assert_same_result(a, b, what):
    assert a["stop"] == b["stop"], (what, a["stop"], b["stop"])
    for k in ("prune0", "prune1", "matches0", "matches1"):
        assert torch.equal(a[k], b[k]), (what, k)
    assert all(torch.equal(x, y) for x, y in zip(a["matches"], b["matches"])), (what, "matches")
    assert [d.get("below") for d in a["decisions"]] == [d.get("below") for d in b["decisions"]], (what, "below")


def decision_deviation(a, b):
    """Two runs that took the same decisions: (largest |difference| of a token confidence or matchability, largest
    ratio of a decision value's difference to its own distance from the threshold in ``b``, over the values
    ``certificate`` takes into account)."""
    dev = ratio = 0.0
    for da, db in zip(a["decisions"], b["decisions"]):
        assert da.keys() == db.keys()
        for k, tok in (("tok0", None), ("tok1", None), ("mat0", "tok0"), ("mat1", "tok1")):
            if k not in db or not db[k].numel():
                continue
            thr = db["thr"] if tok is None else 1.0 - WIDTH
            v, d = db[k].double(), (da[k].double() - db[k].double()).abs()
            dev = max(dev, float(d.max()))
            if tok in db:  # points with confidence <= thr are kept whatever their matchability
                v, d = v[db[tok] > db["thr"]], d[db[tok] > db["thr"]]
            if v.numel():
                ratio = max(ratio, float((d / (v - thr).abs()).max()))
    return dev, ratio


@pytest.mark.parametrize("case", CASES, ids=lambda c: "w{}_th{}_{}x{}_s{}".format(*c))
def test_pinned_case_is_certified(case):
    torch.set_grad_enabled(False)
    ref = reference(*case)
    margin, slack = oracle.certificate(ref["decisions"], depth_confidence=DEPTH, width_confidence=WIDTH)
    print(f"{case}: stop {ref['stop']}  margin {margin:.2e}  count slack {slack:.2f}")
    assert margin >= DELTA and slack >= 1.0
    assert_same_result(run(*case, dtype=torch.float32), ref, "fp32")


@pytest.mark.parametrize("case", CASES, ids=lambda c: "w{}_th{}_{}x{}_s{}".format(*c))
def test_emulated_tensor_core_rounding_stays_inside_the_margin(case):
    """The calibration of the certificate: with the bf16x3 path's rounding emulated, every pinned case takes
    float64's decisions and matches, and no decision value moves by more than a quarter of its own distance from the
    threshold.  (The largest absolute move is not below DELTA / 4: 1.1e-4 at 512 points, 4.0e-4 in 1- and 2-point
    images, in values far from their thresholds where the sigmoid is steepest.)"""
    torch.set_grad_enabled(False)
    ref = reference(*case)
    with emulated(state_dict(case[0]), BF16X3):
        em = run(*case, dtype=torch.float32)
    assert_same_result(em, ref, "emulated bf16x3")
    dev, ratio = decision_deviation(em, ref)
    print(f"{case}: emulated bf16x3 deviation {dev:.2e}, at most {ratio:.3f} of a margin")
    assert ratio <= 0.25


def test_batches_hold_the_cases_they_are_pinned_for():
    torch.set_grad_enabled(False)
    ws, th, cases = RAGGED["w2_th256"]
    stops = {reference(ws, th, *c)["stop"] for c in cases if c[0] and c[1]}
    assert stops == {6, 9}
    ws, th, cases = RAGGED["w3_th-1"]
    assert [reference(ws, th, *c)["stop"] for c in cases] == [6, 4, 6, 6, 6]
    assert [pruned_to_zero(reference(ws, th, *c)) for c in cases] == [False, True, True, False, False]


def test_certificate_counts_and_margins():
    """certificate() on hand-made decisions: a count on the stop boundary has no slack, the matchability of a point
    that is never pruned (confidence <= thr) does not count."""
    tok = torch.tensor([0.5, 0.9], dtype=torch.float64)
    d = {"thr": 0.8, "size": 400, "tok0": tok, "tok1": tok[:0], "below": 20,
         "mat0": torch.tensor([0.01 + 1e-9, 0.5], dtype=torch.float64)}
    margin, slack = oracle.certificate([d], depth_confidence=DEPTH, width_confidence=WIDTH)
    assert slack < 1e-9 and math.isclose(margin, 0.1, rel_tol=1e-9)
    d["below"], d["tok0"] = 17, torch.tensor([0.9, 0.5], dtype=torch.float64)
    margin, slack = oracle.certificate([d], depth_confidence=DEPTH, width_confidence=WIDTH)
    assert math.isclose(slack, 3.0) and margin < 2e-9
    assert oracle.certificate([], depth_confidence=DEPTH, width_confidence=WIDTH) == (math.inf, math.inf)
