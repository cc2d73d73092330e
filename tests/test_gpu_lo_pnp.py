"""GPU LO-RANSAC absolute pose (lightglue_b200.geometry.estimate_absolute_pose_lo over include/geometry_b200.h, steps
LA1-LA8) against its numpy oracle, pair by pair: the same seeding solution, samples drawn, local optimisations, MSAC
cost, counts and inliers, and R, t within 1e-8; failures, intrinsics, batch composition, CUDA graphs and the matcher's
device output as input; and the launch-shape and value bounds of tests/test_gpu_geometry_bounds.py, run through that
module's helpers."""
import math

import numpy as np
import pytest
import torch

from lightglue_b200 import LightGlue, synth
from lightglue_b200.geometry import estimate_absolute_pose, estimate_absolute_pose_lo
from oracle import lo_pnp_oracle as la
from oracle import pnp_oracle as pp
from tests import test_gpu_geometry_bounds as gb

pytestmark = pytest.mark.gpu

EXACT = ("best_hypothesis", "best_solution", "num_hypotheses", "num_local_optimizations", "cost", "num_inliers",
         "success")
K_A = np.array([[500.0, 0.0, 320.0], [0.0, 500.0, 240.0], [0.0, 0.0, 1.0]])
K_B = np.array([[620.0, 0.5, 300.0], [0.0, 580.0, 250.0], [0.0, 0.0, 1.0]])
K_C = np.array([[450.0, 0.0, 330.0], [0.0, 470.0, 230.0], [0.0, 0.0, 1.0]])


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _run(k0, p3, m0, K0, fn=estimate_absolute_pose_lo, **kw):
    out = fn(_t(k0), _t(p3), _t(m0), _t(K0), **kw)
    return {k: v.cpu().numpy() for k, v in out.items()}


def _oracle(k0, p3, m0, K0, ransac_reproj_threshold=8.0, max_iters=100, confidence=0.99, seed=0, pairs=None):
    K0 = np.asarray(K0, dtype=np.float64)
    K0 = np.broadcast_to(K0, (len(m0), 3, 3)) if K0.shape == (3, 3) else K0
    pairs = range(len(m0)) if pairs is None else pairs
    return [la.lo_absolute_pose_pair(k0[b], p3[b], m0[b], K0[b], ransac_reproj_threshold, max_iters, confidence, seed)
            for b in pairs]


def _assert_equal(got, refs, pairs=None):
    pairs = range(len(refs)) if pairs is None else pairs
    for r, b in zip(refs, pairs):
        for k in EXACT:
            assert got[k][b] == r[k], (b, k, got[k][b], r[k])
        assert np.array_equal(got["inliers"][b], r["inliers"]), (b, int((got["inliers"][b] != r["inliers"]).sum()))
        for k in ("R", "t"):
            assert np.isfinite(got[k][b]).all(), (b, k)
            assert np.abs(got[k][b] - r[k]).max() <= 1e-8, (b, k, got[k][b], r[k])


def _scenes(m, outliers, seeds, unmatched, missing3d=0.05, K=None, planar=False):
    pairs = [pp.localization_scene(m, outliers, s, unmatched=u, missing3d=missing3d, K=K, planar=planar)
             for s, u in zip(seeds, unmatched)]
    return tuple(np.stack([p[i] for p in pairs]) for i in range(7))


@pytest.mark.parametrize("outliers", [0.2, 0.5, 0.7])
@pytest.mark.parametrize("confidence", [0.99, 1.0])
def test_matches_the_oracle(outliers, confidence):
    # B = 4 pairs with 5 .. 50 % unmatched rows and 5 % NaN 3D rows, so each pair has its own match count
    k0, p3, m0, _, K, _, _ = _scenes(1024, outliers, [100, 101, 102, 103], (0.05, 0.2, 0.35, 0.5))
    iters = 1000 if outliers > 0.6 else 300
    got = _run(k0, p3, m0, K, max_iters=iters, confidence=confidence)
    _assert_equal(got, _oracle(k0, p3, m0, K, max_iters=iters, confidence=confidence))
    assert got["success"].all() and (got["num_local_optimizations"] >= 1).all()
    if confidence == 1.0:
        assert (got["num_hypotheses"] == iters).all()


def test_per_pair_intrinsics():
    pairs = [pp.localization_scene(1024, 0.3, 110 + b, K=K) for b, K in enumerate([K_A, K_B, K_C])]
    k0, p3, m0, _, K, _, _ = (np.stack([p[i] for p in pairs]) for i in range(7))
    got = _run(k0, p3, m0, K)
    _assert_equal(got, _oracle(k0, p3, m0, K))
    assert got["success"].all()


def test_one_k_equals_the_expanded_k():
    k0, p3, m0, _, _, _, _ = _scenes(1024, 0.4, [120, 121], (0.1, 0.1), K=K_B)
    one = _run(k0, p3, m0, K_B)
    full = _run(k0, p3, m0, np.broadcast_to(K_B, (2, 3, 3)).copy())
    for k in one:
        assert np.array_equal(one[k], full[k]), k
    _assert_equal(one, _oracle(k0, p3, m0, K_B))


def test_matches_the_oracle_at_scale():
    pairs = [pp.localization_scene(4096, o, 200 + b) for b, o in enumerate([0.2, 0.5, 0.7, 0.6] * 8)]
    k0, p3, m0 = (np.stack([p[i] for p in pairs]) for i in range(3))
    got = _run(k0, p3, m0, K_A, max_iters=5000, confidence=1.0)
    assert (got["num_hypotheses"] == 5000).all() and got["success"].all()
    _assert_equal(got, _oracle(k0, p3, m0, K_A, max_iters=5000, confidence=1.0, pairs=[2, 29]), pairs=[2, 29])


def test_planar_scene():
    k0, p3, m0, _, K, _, _ = _scenes(1024, 0.4, [140, 141], (0.1, 0.2), planar=True)
    got = _run(k0, p3, m0, K)
    _assert_equal(got, _oracle(k0, p3, m0, K))
    assert got["success"].all()


def test_draws_the_same_samples_as_plain_ransac():
    # one sample per pair: both estimators solve sample 0 of the same hash and keep one of its solutions
    k0, p3, m0, _, K, _, _ = _scenes(1024, 0.3, [105, 106], (0.0, 0.0))
    a = _run(k0, p3, m0, K, fn=estimate_absolute_pose, max_iters=1)
    b = _run(k0, p3, m0, K, max_iters=1)
    assert (a["best_hypothesis"] == 0).all() and (b["best_hypothesis"] == 0).all()
    assert np.array_equal(a["num_hypotheses"], b["num_hypotheses"])
    _assert_equal(b, _oracle(k0, p3, m0, K, max_iters=1))


def _assert_failed(got, b=0, drawn=0):
    assert not got["success"][b] and got["num_inliers"][b] == 0 and not got["inliers"][b].any()
    assert not got["R"][b].any() and not got["t"][b].any()
    assert got["best_hypothesis"][b] == -1 and got["best_solution"][b] == -1 and got["num_hypotheses"][b] == drawn
    assert got["num_local_optimizations"][b] == 0 and got["cost"][b] == 0


@pytest.mark.parametrize("valid", [0, 2])
def test_too_few_matches_fail(valid):
    k0, p3, m0, *_ = pp.localization_scene(256, 0.0, 7, unmatched=0.0, missing3d=0.0)
    m0 = m0.copy()
    m0[valid:] = -1
    got = _run(k0[None], p3[None], m0[None], K_A)
    _assert_failed(got)


def test_nan_points_leave_too_few_matches():
    k0, p3, m0, *_ = pp.localization_scene(256, 0.0, 7, unmatched=0.0, missing3d=0.0)
    p3 = p3.copy()
    p3[m0[2:]] = np.nan  # every match but two loses its 3D point
    p3[m0[2:10], 1] = 1.0  # a single NaN coordinate is enough
    got = _run(k0[None], p3[None], m0[None], K_A)
    _assert_failed(got)


def test_collinear_points_fail():
    # on one line, exactly in float (dyadic coordinates), and some coincident
    s = np.random.default_rng(4).integers(-96, 97, 300) / 32.0
    X = np.stack([s, 0.5 * s, 8.0 + 0.25 * s], 1).astype(np.float32)
    p = X.astype(np.float64) @ K_A.T
    k0 = (p[:, :2] / p[:, 2:]).astype(np.float32)
    m0 = np.arange(300, dtype=np.int64)
    got = _run(k0[None], X[None], m0[None], K_A, max_iters=512)
    _assert_failed(got, drawn=512)
    _assert_equal(got, _oracle(k0[None], X[None], m0[None], K_A, max_iters=512))


def test_points_behind_the_camera_are_never_inliers():
    # the scene mirrored through the camera centre: every point keeps its pixel at the negated depth, so the true pose
    # sees every point behind the camera and no proper rotation sees them all in front
    k0, p3, m0, _, K, R, t = pp.localization_scene(512, 0.0, 9, missing3d=0.0, unmatched=0.0)
    behind = ((-(p3.astype(np.float64) @ R.T + t) - t) @ R).astype(np.float32)
    P = pp.projection(R.reshape(9), t, K)[None]
    assert not pp.reproj_inliers(P, k0, behind[m0], np.float32(64.0)).any()
    assert np.isinf(la.errors(P, k0, behind[m0])).all()  # and each scores as an outlier
    got = _run(k0[None], behind[None], m0[None], K)
    assert got["num_inliers"][0] <= 0.25 * 512
    _assert_equal(got, _oracle(k0[None], behind[None], m0[None], K))
    # every inlier of the result is in front of its camera
    Xc = behind.astype(np.float64)[m0] @ got["R"][0].T + got["t"][0]
    assert (Xc[got["inliers"][0], 2] > 0.0).all()


@pytest.mark.parametrize("bad", ["nan", "fx", "bottom"])
def test_an_invalid_k_fails_only_its_pair(bad):
    k0, p3, m0, _, _, _, _ = _scenes(1024, 0.3, [130, 131, 132], (0.1, 0.2, 0.0))
    K = np.broadcast_to(K_A, (3, 3, 3)).copy()
    good = _run(k0, p3, m0, K)
    if bad == "nan":
        K[1, 0, 2] = np.nan
    elif bad == "fx":
        K[1, 0, 0] = 0.0
    else:
        K[1, 2, 2] = 2.0
    got = _run(k0, p3, m0, K)
    _assert_failed(got, b=1)
    for k in got:
        for b in (0, 2):
            assert np.array_equal(got[k][b], good[k][b]), (k, b)


def test_out_of_range_indices_are_unmatched():
    k0, p3, m0, *_ = pp.localization_scene(512, 0.3, 8)
    bad = m0.copy()
    bad[::7] = 512 + np.arange(bad[::7].size)  # past N
    bad[3::11] = -5
    clean = np.where((bad >= 0) & (bad < 512), bad, -1)
    a = _run(k0[None], p3[None], bad[None], K_A)
    b = _run(k0[None], p3[None], clean[None], K_A)
    for k in a:
        assert np.array_equal(a[k], b[k]), k
    _assert_equal(a, _oracle(k0[None], p3[None], clean[None], K_A))


def test_batch_equals_single_pairs_and_repeats():
    k0, p3, m0, _, _, _, _ = _scenes(777, 0.3, [31, 32, 33], (0.1, 0.4, 0.0))
    full = _run(k0, p3, m0, K_A)
    again = _run(k0, p3, m0, K_A)
    for k in full:
        assert np.array_equal(full[k], again[k]), k
    for b in range(3):
        one = _run(k0[b:b + 1], p3[b:b + 1], m0[b:b + 1], K_A)
        for k in full:
            assert np.array_equal(full[k][b], one[k][0]), (b, k)


def test_another_seed_recovers_the_truth():
    k0, p3, m0, truth, K, R, t = pp.localization_scene(2048, 0.5, 9)
    a = _run(k0[None], p3[None], m0[None], K, seed=0)
    b = _run(k0[None], p3[None], m0[None], K, seed=987654321)
    assert a["best_hypothesis"][0] != b["best_hypothesis"][0]
    assert la.rotation_error(b["R"][0], R) <= 0.1
    assert np.linalg.norm(b["t"][0] - t) <= 0.02
    assert (b["inliers"][0] & truth).sum() / truth.sum() >= 0.98
    _assert_equal(b, _oracle(k0[None], p3[None], m0[None], K, seed=987654321))


def test_composes_with_the_matcher():
    torch.manual_seed(0)
    data, perm = synth.make_pair(1024, seed=2024)
    k1 = data["image1"]["keypoints"][0].numpy().astype(np.float64)
    # image 1's keypoints lifted to depths 4..12 through its own K, then seen by the query camera
    rng = np.random.default_rng(5)
    K = np.array([[800.0, 0.0, 512.0], [0.0, 800.0, 384.0], [0.0, 0.0, 1.0]])
    d = rng.uniform(4, 12, 1024)
    X = np.c_[(k1[:, 0] - 512.0) / 800.0 * d, (k1[:, 1] - 384.0) / 800.0 * d, d]
    X[rng.random(1024) < 0.1] = np.nan  # depth holes
    p3 = torch.from_numpy(X.astype(np.float32))[None].cuda()
    matcher = LightGlue(features=None, depth_confidence=-1, width_confidence=-1, precision="bf16x3")
    matcher.load_state_dict(synth.make_state_dict(), strict=False)
    matcher = matcher.eval().cuda()
    cuda = {k: {kk: vv.cuda() for kk, vv in v.items()} for k, v in data.items()}
    with torch.no_grad():
        pending = matcher.forward_async(cuda)
        m0 = pending.tensors["matches0"]
        r = estimate_absolute_pose_lo(cuda["image0"]["keypoints"], p3, m0, torch.from_numpy(K).cuda())
    got = {k: v.cpu().numpy() for k, v in r.items()}
    m0 = m0.cpu().numpy()
    assert (m0 >= 0).sum() >= 100
    kk0 = data["image0"]["keypoints"].numpy()
    _assert_equal(got, _oracle(kk0, X.astype(np.float32)[None], m0, K))


def test_cuda_graph_replay_equals_eager():
    k0, p3, m0, _, _, _, _ = _scenes(1024, 0.3, [41, 42], (0.1, 0.1))
    K = np.stack([K_A, K_B])
    k0, p3, m0, K = (_t(x) for x in (k0, p3, m0, K))
    eager = estimate_absolute_pose_lo(k0, p3, m0, K)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        estimate_absolute_pose_lo(k0, p3, m0, K)  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        captured = estimate_absolute_pose_lo(k0, p3, m0, K)
    for v in captured.values():
        v.zero_()
    g.replay()
    torch.cuda.synchronize()
    for k in eager:
        assert torch.equal(eager[k], captured[k]), k


# --------------------------------------------------------------------- the bounds of tests/test_gpu_geometry_bounds.py

LO_PNP = gb.Est("LO-PnP", lambda a, b, m0, K, **kw: estimate_absolute_pose_lo(gb._t(a), gb._t(b), gb._t(m0), gb._t(K),
                                                                              **kw),
                lambda a, b, m0, K, thr, it, conf, seed: la.lo_absolute_pose_pair(a, b, m0, K, thr, it, conf, seed),
                ("best_hypothesis", "best_solution", "num_hypotheses", "num_inliers", "success") + gb._LO,
                ("inliers",), {"R": "R", "t": "t"}, gb._localization, 8.0, False, 512, "geo_lo_pnp_workspace_bytes",
                lo=True, relative=False)


@pytest.fixture
def lo_pnp(monkeypatch):
    """The bound cases look their estimator up by name in gb.ESTIMATORS: add LO-PnP for the test's duration."""
    monkeypatch.setitem(gb.ESTIMATORS, LO_PNP.name, LO_PNP)
    return LO_PNP.name


def test_bounds_one_split_of_several_tiles(lo_pnp):
    gb.test_one_split_of_several_tiles(lo_pnp)


@pytest.mark.parametrize("m,unmatched", [((1 << 17) + 37, 0.1), (300_000, 0.0)])
def test_bounds_most_splits(lo_pnp, m, unmatched):
    gb.test_most_splits(lo_pnp, m, unmatched)


def test_bounds_more_pairs_than_a_grid_column(lo_pnp):
    gb.test_more_pairs_than_a_grid_column(lo_pnp)


@pytest.mark.parametrize("max_iters", [1, 255, 257, 513])
def test_bounds_chunk_edges(lo_pnp, max_iters):
    gb.test_chunk_edges(lo_pnp, max_iters)


def test_bounds_adaptive_stop_mid_budget(lo_pnp):
    gb.test_adaptive_stop_mid_budget(lo_pnp)


def test_bounds_empty_pairs(lo_pnp):
    gb.test_empty_pairs(lo_pnp)


def test_bounds_lo_bound_with_every_point_an_outlier(lo_pnp):
    # gb's case, with n in place of M: the localization scene leaves 5 % of the 3D points NaN, so n < M
    e = gb.ESTIMATORS[lo_pnp]
    M = gb._cabi.GEO_LO_MAX_MATCHES
    a, b, m0, K = gb._batch(e, M, [61], outliers=0.3, unmatched=0.0)
    threshold = 1e-30
    assert gb._thr2(e, threshold, K) == 0.0
    got = gb._check(e, a, b, m0, K, **gb._kw(e, threshold=threshold, max_iters=8))
    n = int(gb._valid(e, a, b, m0)[0])
    assert got["success"][0] and got["num_inliers"][0] == 0 and n > 0.9 * M
    assert got["cost"][0] == la.QSCALE * n


@pytest.mark.parametrize("thr2", [0.0, gb.SUBNORMAL, gb.FLT_MIN, math.inf], ids=["zero", "subnormal", "flt_min", "inf"])
def test_bounds_threshold_extremes(lo_pnp, thr2):
    gb.test_threshold_extremes(lo_pnp, thr2)


@pytest.mark.parametrize("case", ["8192x6144", "offset", "integer"])
def test_bounds_coordinates(lo_pnp, case):
    gb.test_coordinates(lo_pnp, case)


def test_bounds_non_finite_keypoints_are_invalid(lo_pnp):
    gb.test_non_finite_keypoints_are_invalid(lo_pnp)


def test_bounds_duplicate_points_and_matches(lo_pnp):
    gb.test_duplicate_points_and_matches(lo_pnp)
