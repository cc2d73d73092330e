"""Early exit and point pruning in batches: the configuration LightGlue() runs by default (adaptive, batched, on the
tensor cores) against the oracle and against each pair run alone.

In a batch whose pairs stop at different layers and whose images prune to different lengths, the kernels skip the
tiles of stopped pairs and dead rows, attend to each partner's compacted keys, decide pruning per image, end a pair
whose image was pruned to zero while the others continue, refresh the bf16 shadows after each compaction and select
each pair's own assignment head.  None of that runs at B = 1 or with adaptivity off.

A. Certified pairs (tests/test_adaptive_margins.py: every decision >= 1e-4 from its threshold, every count >= 1 point
   from the stop boundary) in ragged and dense batches, bf16x3 and fp32: each pair equals the float64 oracle alone.
B. The default threshold (1536) at 1400 .. 2048 points, bf16x3 / bf16 / fp32: each pair equals its own B = 1 call bit
   for bit; the bf16x3 bench-shaped batch stays within a bound of the fp32 oracle.
C. CUDA-graph replay and NaN padding rows with adaptivity on.
"""
import pytest
import torch

from lightglue_b200 import LightGlue, synth
from lightglue_b200.ragged import pad_pairs, split_outputs
from oracle import lightglue_oracle as oracle
from tests.test_adaptive_margins import DENSE, DEPTH, RAGGED, WIDTH, reference, single_pair, state_dict

pytestmark = pytest.mark.gpu

TOL = {"bf16x3": 1e-3, "fp32": 1e-4}


def make_matcher(precision, ws, threshold=None, **conf):
    m = LightGlue(features=None, precision=precision, depth_confidence=DEPTH, width_confidence=WIDTH, **conf)
    m.load_state_dict(state_dict(ws), strict=False)
    m = m.eval().cuda()
    if threshold is not None:
        m.pruning_keypoint_thresholds = dict(LightGlue.pruning_keypoint_thresholds, flash=threshold)
    return m


def to_cuda(data):
    return {k: {kk: vv.cuda() for kk, vv in v.items()} for k, v in data.items()}


def ragged_batch(cases):
    return pad_pairs([to_cuda(single_pair(m, n, s)) for m, n, s in cases])


def dense_batch(cases):
    pairs = [single_pair(m, n, s) for m, n, s in cases]
    return to_cuda({k: {kk: torch.cat([p[k][kk] for p in pairs]) for kk in pairs[0][k]} for k in ("image0", "image1")})


def pair_of(out, b):
    """Pair b of a dense batch's output, shaped like a B = 1 call."""
    res = {k: out[k][b : b + 1] for k in ("matches0", "matches1", "matching_scores0", "matching_scores1", "prune0", "prune1")}
    res.update(matches=[out["matches"][b]], scores=[out["scores"][b]], stop=out["stops"][b])
    return res


def check_against_oracle(got, ref, tol, what):
    """Identical stop, prune counters and matches; scores within tol.  Returns the largest score difference."""
    assert int(got["stop"]) == int(ref["stop"]), (what, got["stop"], ref["stop"])
    for k in ("prune0", "prune1", "matches0", "matches1"):
        assert torch.equal(got[k].cpu().to(torch.int64), ref[k].to(torch.int64)), (what, k)
    assert torch.equal(got["matches"][0].cpu().to(torch.int64).reshape(-1, 2), ref["matches"][0].reshape(-1, 2)), (what, "matches")
    dmax = 0.0
    for k in ("matching_scores0", "matching_scores1"):
        if ref[k].numel():
            dmax = max(dmax, float((got[k].cpu().double() - ref[k].double()).abs().max()))
    assert dmax <= tol, (what, dmax)
    return dmax


def check_equal(got, alone, what):
    """A pair of a batch against the same pair alone: everything bit for bit."""
    assert int(got["stop"]) == int(alone["stop"]), (what, got["stop"], alone["stop"])
    for k in ("prune0", "prune1", "matches0", "matches1", "matching_scores0", "matching_scores1"):
        assert torch.equal(got[k], alone[k]), (what, k)
    assert torch.equal(got["matches"][0], alone["matches"][0]) and torch.equal(got["scores"][0], alone["scores"][0]), what


# ---------------------------------------------------------------------------------------------------- A: the oracle
@pytest.mark.parametrize("precision", ["bf16x3", "fp32"])
@pytest.mark.parametrize("batch", sorted(RAGGED))
def test_ragged_adaptive_batch_equals_certified_oracle(batch, precision):
    torch.set_grad_enabled(False)
    ws, th, cases = RAGGED[batch]
    m = make_matcher(precision, ws, th)
    data = ragged_batch(cases)
    out = m(data)
    results = split_outputs(out, data["image0"]["num_keypoints"], data["image1"]["num_keypoints"])
    dmax, stops = 0.0, []
    for case, got in zip(cases, results):
        ref = reference(ws, th, *case)
        dmax = max(dmax, check_against_oracle(got, ref, TOL[precision], case))
        stops.append(int(ref["stop"]))
    assert out["stops"] == stops and out["stop"] == max(stops)
    print(f"{batch} {precision}: stops {stops}, max |dscore| {dmax:.2e}")


@pytest.mark.parametrize("precision", ["bf16x3", "fp32"])
def test_dense_adaptive_batch_equals_certified_oracle(precision):
    torch.set_grad_enabled(False)
    ws, th, cases = DENSE
    out = make_matcher(precision, ws, th)(dense_batch(cases))
    refs = [reference(ws, th, *c) for c in cases]
    dmax = max(check_against_oracle(pair_of(out, b), r, TOL[precision], c) for b, (c, r) in enumerate(zip(cases, refs)))
    assert out["stops"] == [int(r["stop"]) for r in refs]
    print(f"dense B=4 {precision}: stops {out['stops']}, max |dscore| {dmax:.2e}")


# ------------------------------------------------------------------------------- B: each pair alone, default threshold
_BENCH = {}


def bench_shaped(precision):
    """B = 32 pairs of 2048 points with adaptivity on at the module's own threshold: (batch output, data, matcher)."""
    if precision not in _BENCH:
        data = to_cuda(synth.make_pair(2048, b=32, seed=1000)[0])
        m = make_matcher(precision, 0)
        _BENCH[precision] = (m(data), data, m)
    return _BENCH[precision]


@pytest.mark.parametrize("precision", ["bf16x3", "bf16", "fp32"])
def test_bench_shaped_adaptive_batch_equals_single_pairs(precision):
    torch.set_grad_enabled(False)
    out, data, m = bench_shaped(precision)
    for b in range(32):
        alone = m({k: {kk: vv[b : b + 1] for kk, vv in v.items()} for k, v in data.items()})
        check_equal(pair_of(out, b), alone, b)
    stops = torch.tensor(out["stops"], device=out["prune0"].device)[:, None]
    pruned = int((out["prune0"] < stops).sum() + (out["prune1"] < stops).sum())
    print(f"B=32 n=2048 {precision}: stops {sorted(set(out['stops']))}, {pruned} of {2 * 32 * 2048} points pruned")


# image sizes on both sides of the default threshold (1536), beside smaller and larger images
DEFAULT_SIZES = [(1535, 1400, 11), (1536, 2048, 12), (1537, 1600, 13), (1600, 1536, 14), (2048, 1537, 15), (1400, 2048, 16)]


@pytest.mark.parametrize("precision", ["bf16x3", "bf16", "fp32"])
def test_ragged_adaptive_batch_at_default_threshold_equals_single_pairs(precision):
    torch.set_grad_enabled(False)
    m = make_matcher(precision, 0)
    data = ragged_batch(DEFAULT_SIZES)
    out = m(data)
    results = split_outputs(out, data["image0"]["num_keypoints"], data["image1"]["num_keypoints"])
    for (mm, nn, s), got in zip(DEFAULT_SIZES, results):
        alone = m(to_cuda(single_pair(mm, nn, s)))
        check_equal(got, alone, (mm, nn))
    print(f"default threshold {precision}: stops {out['stops']}")


def test_bench_shaped_bf16x3_batch_stays_near_the_fp32_oracle():
    """Not certified (margins at 2048 points are 3e-6 .. 3e-5), so bounded: identical stop (the count slack is hundreds
    of points), prune counters on at most 0.5 % of the points."""
    torch.set_grad_enabled(False)
    out, data, m = bench_shaped("bf16x3")
    sd = state_dict(0)
    for b in (0, 13, 31):
        one = {k: {kk: vv[b : b + 1].cpu() for kk, vv in v.items()} for k, v in data.items()}
        ref = oracle.forward(sd, one, depth_confidence=DEPTH, width_confidence=WIDTH, pruning_threshold=1536)
        got = pair_of(out, b)
        assert int(got["stop"]) == int(ref["stop"]), (b, got["stop"], ref["stop"])
        diff = [int((got[k].cpu() != ref[k]).sum()) for k in ("prune0", "prune1")]
        flips = sum(int((got[k].cpu() != ref[k]).sum()) for k in ("matches0", "matches1"))
        print(f"pair {b}: stop {ref['stop']}, prune counters differ on {diff} of 2048 + 2048 points, {flips} index flips")
        assert sum(diff) <= 0.005 * 4096, (b, diff)


# ------------------------------------------------------------------------------------ C: graph replay, inert padding
def test_ragged_adaptive_cuda_graph_replay_equals_eager():
    """Captured on one set of lengths and replayed on another of the same padded shape: stops and prune patterns
    differ between the two, and each replay equals the eager forward bit for bit."""
    torch.set_grad_enabled(False)
    g = make_matcher("bf16x3", 2, 256, cuda_graph=True)
    e = make_matcher("bf16x3", 2, 256)
    stops = []
    for cases in ([(383, 640, 1), (256, 300, 16), (64, 128, 1)], [(300, 640, 2), (383, 129, 1), (1, 63, 6)]):
        data = ragged_batch(cases)
        a, b = g(data), e(data)
        assert a["stops"] == b["stops"]
        for k in ("matches0", "matches1", "matching_scores0", "matching_scores1", "prune0", "prune1"):
            assert torch.equal(a[k], b[k]), k
        stops.append(a["stops"])
    assert len(g._graphs) == 1 and stops[0] != stops[1], stops


def test_ragged_adaptive_padding_rows_are_inert():
    """NaN in the padding rows of a ragged adaptive batch changes no output; padding rows come back -1 / 0."""
    torch.set_grad_enabled(False)
    ws, th, cases = RAGGED["w2_th256"]
    m = make_matcher("bf16x3", ws, th)
    data = ragged_batch(cases)
    clean = m(data)
    lens0, lens1 = data["image0"]["num_keypoints"].tolist(), data["image1"]["num_keypoints"].tolist()
    for key, lens in (("image0", lens0), ("image1", lens1)):
        for b, n in enumerate(lens):
            data[key]["keypoints"][b, n:] = float("nan")
            data[key]["descriptors"][b, n:] = float("nan")
    dirty = m(data)
    for k in ("matches0", "matches1", "matching_scores0", "matching_scores1", "prune0", "prune1"):
        assert torch.equal(clean[k], dirty[k]), k
    assert dirty["stops"] == clean["stops"]
    for b, (n0, n1) in enumerate(zip(lens0, lens1)):
        assert int((dirty["matches0"][b, n0:] != -1).sum()) == 0 and int((dirty["matches1"][b, n1:] != -1).sum()) == 0
        assert float(dirty["matching_scores0"][b, n0:].abs().sum()) == 0 and int(dirty["prune0"][b, n0:].abs().sum()) == 0
