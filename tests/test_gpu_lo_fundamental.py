"""GPU LO-RANSAC fundamental matrix (lightglue_b200.geometry.find_fundamental_lo over include/geometry_b200.h, steps
LF1-LF8) against its numpy oracle, pair by pair: the same seeding hypothesis, samples drawn, local optimisations, MSAC
cost, counts and inliers, and F within 1e-8; failures, batch composition, CUDA graphs and the matcher's device output
as input; and the launch-shape and value bounds of tests/test_gpu_geometry_bounds.py, run through that module's
helpers."""
import math

import numpy as np
import pytest
import torch

from lightglue_b200 import LightGlue, synth
from lightglue_b200.geometry import find_fundamental, find_fundamental_lo
from oracle import geometry_oracle as go
from oracle import geometry_synth as gs
from oracle import lo_fundamental_oracle as lf
from tests import test_gpu_geometry_bounds as gb

pytestmark = pytest.mark.gpu

EXACT = ("best_hypothesis", "num_hypotheses", "num_local_optimizations", "cost", "num_inliers", "success")


def _run(k0, k1, m0, fn=find_fundamental_lo, **kw):
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()  # noqa: E731
    out = fn(t(k0), t(k1), t(m0), **kw)
    return {k: v.cpu().numpy() for k, v in out.items()}


def _oracle(k0, k1, m0, ransac_reproj_threshold=3.0, max_iters=1000, confidence=0.99, seed=0, pairs=None):
    pairs = range(len(m0)) if pairs is None else pairs
    return [lf.lo_fundamental_pair(k0[b], k1[b], m0[b], ransac_reproj_threshold, max_iters, confidence, seed)
            for b in pairs]


def _assert_equal(got, refs, pairs=None):
    pairs = range(len(refs)) if pairs is None else pairs
    for r, b in zip(refs, pairs):
        for k in EXACT:
            assert got[k][b] == r[k], (b, k, got[k][b], r[k])
        assert np.array_equal(got["inliers"][b], r["inliers"]), (b, int((got["inliers"][b] != r["inliers"]).sum()))
        assert np.isfinite(got["F"][b]).all(), b
        assert np.abs(got["F"][b] - r["F"]).max() <= 1e-8 * max(np.abs(r["F"]).max(), 1e-300), (b, got["F"][b], r["F"])


@pytest.mark.parametrize("outliers", [0.2, 0.5, 0.7])
@pytest.mark.parametrize("confidence", [0.99, 1.0])
def test_matches_the_oracle(outliers, confidence):
    # B = 4 pairs with 5 .. 50 % unmatched rows, so each pair has its own match count
    pairs = [gs.two_view(1024, outliers, 100 + b, noise=1.0, unmatched=u) for b, u in enumerate((0.05, 0.2, 0.35, 0.5))]
    k0, k1, m0 = (np.stack([p[i] for p in pairs]) for i in range(3))
    got = _run(k0, k1, m0, confidence=confidence)
    _assert_equal(got, _oracle(k0, k1, m0, confidence=confidence))
    assert got["success"].all() and (got["num_local_optimizations"] >= 1).all()
    if confidence == 1.0:
        assert (got["num_hypotheses"] == 1000).all()


def test_matches_the_oracle_at_scale():
    k0, k1, m0, _, _ = gs.batch("F", 4096, [0.2, 0.5, 0.7, 0.6] * 8, list(range(200, 232)))
    got = _run(k0, k1, m0, max_iters=5000, confidence=1.0)
    assert (got["num_hypotheses"] == 5000).all() and got["success"].all()
    _assert_equal(got, _oracle(k0, k1, m0, max_iters=5000, confidence=1.0, pairs=[2, 29]), pairs=[2, 29])


def test_draws_the_same_samples_as_plain_ransac():
    # one sample per pair: both estimators solve hypothesis 0 of the same hash and keep it
    k0, k1, m0, _, _ = gs.batch("F", 1024, [0.0, 0.3], [105, 106], unmatched=0.0)
    a = _run(k0, k1, m0, fn=find_fundamental, max_iters=1)
    b = _run(k0, k1, m0, max_iters=1)
    assert (a["best_hypothesis"] == 0).all() and (b["best_hypothesis"] == 0).all()
    assert np.array_equal(a["num_hypotheses"], b["num_hypotheses"])
    # and over a chunk the plain estimator equals its oracle and the LO one equals its own, both on go.hypotheses
    a = _run(k0, k1, m0, fn=find_fundamental, max_iters=256, confidence=1.0)
    b = _run(k0, k1, m0, max_iters=256, confidence=1.0)
    for i, r in enumerate(go.estimate_pair(go.FUNDAMENTAL, k0[i], k1[i], m0[i], 3.0, 256, 1.0, 0) for i in range(2)):
        assert a["best_hypothesis"][i] == r["best_hypothesis"]
    _assert_equal(b, _oracle(k0, k1, m0, max_iters=256, confidence=1.0))


@pytest.mark.parametrize("valid", [0, 7])
def test_too_few_matches_fail(valid):
    k0, k1, m0, _, _ = gs.two_view(256, 0.0, 7, unmatched=0.0)
    m0 = m0.copy()
    m0[valid:] = -1
    got = _run(k0[None], k1[None], m0[None])
    assert not got["success"][0] and got["num_inliers"][0] == 0 and not got["inliers"].any()
    assert not got["F"].any() and got["best_hypothesis"][0] == -1 and got["num_hypotheses"][0] == 0
    assert got["num_local_optimizations"][0] == 0 and got["cost"][0] == 0


def test_all_degenerate_samples_fail():
    # one line in both images: every eight-point system is rank-deficient
    line = np.stack([np.linspace(0, 600, 300), np.linspace(10, 400, 300)], 1).astype(np.float32)
    m0 = np.arange(300, dtype=np.int64)
    got = _run(line[None], line[None].copy(), m0[None], max_iters=512)
    assert not got["success"][0] and not got["inliers"].any() and got["num_inliers"][0] == 0
    assert got["num_hypotheses"][0] == 512 and got["cost"][0] == 0 and got["num_local_optimizations"][0] == 0
    _assert_equal(got, _oracle(line[None], line[None], m0[None], max_iters=512))


def test_out_of_range_indices_are_unmatched():
    k0, k1, m0, _, _ = gs.two_view(512, 0.3, 8)
    bad = m0.copy()
    bad[::7] = 512 + np.arange(bad[::7].size)  # past N
    bad[3::11] = -5
    clean = np.where((bad >= 0) & (bad < 512), bad, -1)
    a = _run(k0[None], k1[None], bad[None])
    b = _run(k0[None], k1[None], clean[None])
    for k in a:
        assert np.array_equal(a[k], b[k]), k
    _assert_equal(a, _oracle(k0[None], k1[None], clean[None]))


def test_batch_equals_single_pairs_and_repeats():
    k0, k1, m0, _, _ = gs.batch("F", 777, [0.3, 0.6, 0.1], [31, 32, 33], unmatched=[0.1, 0.4, 0.0])
    full = _run(k0, k1, m0)
    again = _run(k0, k1, m0)
    for k in full:
        assert np.array_equal(full[k], again[k]), k
    for b in range(3):
        one = _run(k0[b:b + 1], k1[b:b + 1], m0[b:b + 1])
        for k in full:
            assert np.array_equal(full[k][b], one[k][0]), (b, k)


def test_another_seed_recovers_the_truth():
    k0, k1, m0, truth, Ft = gs.two_view(2048, 0.5, 9)
    a = _run(k0[None], k1[None], m0[None], seed=0)
    b = _run(k0[None], k1[None], m0[None], seed=987654321)
    assert a["best_hypothesis"][0] != b["best_hypothesis"][0]
    assert (b["inliers"][0] & truth).sum() / truth.sum() >= 0.98
    plain = _run(k0[None], k1[None], m0[None], fn=find_fundamental, seed=987654321)
    assert lf.fundamental_error(b["F"][0], Ft) < min(lf.fundamental_error(plain["F"][0], Ft), 4.0)
    _assert_equal(b, _oracle(k0[None], k1[None], m0[None], seed=987654321))


def test_composes_with_the_matcher():
    # image 1's keypoints are image 0's seen by a second camera, so the matcher's matches0 carries an epipolar geometry
    torch.manual_seed(0)
    data, perm = synth.make_pair(1024, seed=2024)
    rng = np.random.default_rng(5)
    k0 = data["image0"]["keypoints"][0].numpy().astype(np.float64)
    K = np.array([[800.0, 0.0, 512.0], [0.0, 800.0, 384.0], [0.0, 0.0, 1.0]])
    X = np.concatenate([k0, np.ones((1024, 1))], 1) @ np.linalg.inv(K).T * rng.uniform(4.0, 12.0, (1024, 1))
    R = gs._rot(rng)
    t = np.array([1.0, 0.1, -0.1])
    p1 = (X @ R.T + t) @ K.T
    k1 = p1[:, :2] / p1[:, 2:3] + rng.normal(0.0, 0.5, (1024, 2))
    data["image1"]["keypoints"] = torch.from_numpy(k1[perm[0].numpy()].astype(np.float32))[None]
    matcher = LightGlue(features=None, depth_confidence=-1, width_confidence=-1, precision="bf16x3")
    matcher.load_state_dict(synth.make_state_dict(), strict=False)
    matcher = matcher.eval().cuda()
    cuda = {k: {kk: vv.cuda() for kk, vv in v.items()} for k, v in data.items()}
    with torch.no_grad():
        pending = matcher.forward_async(cuda)
        m0 = pending.tensors["matches0"]
        r = find_fundamental_lo(cuda["image0"]["keypoints"], cuda["image1"]["keypoints"], m0)
    got = {k: v.cpu().numpy() for k, v in r.items()}
    m0 = m0.cpu().numpy()
    assert (m0 >= 0).sum() >= 100 and got["success"][0]
    kk0 = data["image0"]["keypoints"].numpy()
    kk1 = data["image1"]["keypoints"].numpy()
    _assert_equal(got, _oracle(kk0, kk1, m0))


def test_cuda_graph_replay_equals_eager():
    k0, k1, m0, _, _ = gs.batch("F", 1024, [0.3, 0.5], [41, 42])
    k0, k1, m0 = (torch.from_numpy(x).cuda() for x in (k0, k1, m0))
    eager = find_fundamental_lo(k0, k1, m0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        find_fundamental_lo(k0, k1, m0)  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        captured = find_fundamental_lo(k0, k1, m0)
    for v in captured.values():
        v.zero_()
    g.replay()
    torch.cuda.synchronize()
    for k in eager:
        assert torch.equal(eager[k], captured[k]), k


# --------------------------------------------------------------------- the bounds of tests/test_gpu_geometry_bounds.py

LO_F = gb.Est("LO-F", lambda a, b, m0, K, **kw: find_fundamental_lo(gb._t(a), gb._t(b), gb._t(m0), **kw),
              lambda a, b, m0, K, thr, it, conf, seed: lf.lo_fundamental_pair(a, b, m0, thr, it, conf, seed),
              gb._H_EXACT + gb._LO, ("inliers",), {"F": "F"}, gb._two_view, 3.0, False, 1024,
              "geo_lo_fundamental_workspace_bytes", lo=True)


@pytest.fixture
def lo_f(monkeypatch):
    """The bound cases look their estimator up by name in gb.ESTIMATORS: add LO-F for the test's duration."""
    monkeypatch.setitem(gb.ESTIMATORS, LO_F.name, LO_F)
    return LO_F.name


def test_bounds_one_split_of_several_tiles(lo_f):
    gb.test_one_split_of_several_tiles(lo_f)


def test_bounds_most_splits(lo_f):
    gb.test_most_splits(lo_f, (1 << 17) + 37, 0.1)


def test_bounds_more_pairs_than_a_grid_column(lo_f):
    gb.test_more_pairs_than_a_grid_column(lo_f)


@pytest.mark.parametrize("max_iters", [1, 255, 257, 513])
def test_bounds_chunk_edges(lo_f, max_iters):
    gb.test_chunk_edges(lo_f, max_iters)


def test_bounds_adaptive_stop_mid_budget(lo_f):
    gb.test_adaptive_stop_mid_budget(lo_f)


def test_bounds_empty_pairs(lo_f):
    gb.test_empty_pairs(lo_f)


def test_bounds_lo_bound_with_every_point_an_outlier(lo_f):
    gb.test_lo_bound_with_every_point_an_outlier(lo_f)


@pytest.mark.parametrize("thr2", [0.0, gb.SUBNORMAL, gb.FLT_MIN, math.inf], ids=["zero", "subnormal", "flt_min", "inf"])
def test_bounds_threshold_extremes(lo_f, thr2):
    gb.test_threshold_extremes(lo_f, thr2)
    if thr2 == math.inf:  # every finite error is an inlier, so every point scores 0
        a, b, m0, K = gb._batch(LO_F, 500, [71, 72], outliers=[0.2, 0.5])
        got = gb._run(LO_F, a, b, m0, K, **gb._kw(LO_F, threshold=1e20))
        assert (got["num_inliers"] == gb._valid(LO_F, a, b, m0)).all() and not got["cost"].any()


@pytest.mark.parametrize("case", ["8192x6144", "offset", "integer"])
def test_bounds_coordinates(lo_f, case):
    gb.test_coordinates(lo_f, case)


def test_bounds_non_finite_keypoints_are_invalid(lo_f):
    gb.test_non_finite_keypoints_are_invalid(lo_f)


def test_bounds_duplicate_points_and_matches(lo_f):
    gb.test_duplicate_points_and_matches(lo_f)
