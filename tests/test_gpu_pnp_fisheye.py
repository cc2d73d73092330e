"""The fisheye absolute pose on the GPU (estimate_absolute_pose_fisheye and estimate_absolute_pose_lo_fisheye;
include/geometry_b200.h steps AE1-AE4) against oracle/fisheye_oracle.py: every output bit for bit (R
and t within 1e-8) at 20/50/70 % outliers, adaptive and full budgets, per-pair K and D, failing bearings inside a
pair, invalid coefficients, B = 32 x 4096, the matcher's output fed without read-back, and the launch-shape and value
bounds of test_gpu_geometry_bounds.py."""
from __future__ import annotations

import numpy as np
import pytest
import torch

from lightglue_b200.geometry import estimate_absolute_pose_fisheye, estimate_absolute_pose_lo_fisheye
from oracle import fisheye_oracle as fo
from tests import test_gpu_geometry_bounds as gb

pytestmark = pytest.mark.gpu

D = fo.D_SCENE
D_RIM = np.array([-0.02, -0.01, 0.0, 0.0])  # FE3 fails beyond theta_d = 1.52 (437 px at f = 280)
EXACT = ("best_hypothesis", "best_solution", "num_hypotheses", "num_inliers", "success")
LO_EXACT = EXACT + ("num_local_optimizations", "cost")


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _scenes(M, seeds, outliers, dists, **kw):
    sc = [fo.scene(M, o, s, d, **kw) for s, o, d in zip(seeds, outliers, dists)]
    return tuple(np.stack([s[i] for s in sc]) for i in range(3)) + (sc[0][4],)


def _compare(lo, got, ref, pairs=None):
    pairs = range(len(ref["success"])) if pairs is None else pairs
    for i, p in enumerate(pairs):
        for k in (LO_EXACT if lo else EXACT):
            assert got[k][p] == ref[k][i], (p, k, got[k][p], ref[k][i])
        flips = int((got["inliers"][p] != ref["inliers"][i]).sum())
        assert flips == 0, (p, flips)
        for k in ("R", "t"):
            assert np.abs(got[k][p] - ref[k][i]).max() <= 1e-8, (p, k)


def _run(lo, k0, p3, m0, K, dist, **kw):
    fn = estimate_absolute_pose_lo_fisheye if lo else estimate_absolute_pose_fisheye
    return {k: v.cpu().numpy() for k, v in fn(_t(k0), _t(p3), _t(m0), _t(K), _t(dist), **kw).items()}


def _oracle(lo, k0, p3, m0, K, dist, pairs, threshold=8.0, max_iters=100, confidence=0.99, seed=0):
    f = fo.lo_absolute_pose_pair if lo else fo.absolute_pose_pair
    K = np.broadcast_to(K, (len(k0), 3, 3))
    outs = [f(k0[p], p3[p], m0[p], K[p], threshold, max_iters, confidence, seed, dist[p]) for p in pairs]
    return {k: np.stack([np.asarray(o[k]) for o in outs]) for k in outs[0]}


@pytest.mark.parametrize("lo", [False, True], ids=["plain", "lo"])
@pytest.mark.parametrize("budget", ["adaptive", "full"])
def test_matches_oracle_at_outlier_shares(lo, budget):
    k0, p3, m0, K = _scenes(1024, [11, 12, 13], [0.2, 0.5, 0.7], [D] * 3)
    dist = np.stack([D] * 3)
    kw = dict(max_iters=1000, confidence=0.99) if budget == "adaptive" else dict(max_iters=512, confidence=1.0)
    got = _run(lo, k0, p3, m0, K, dist, **kw)
    _compare(lo, got, _oracle(lo, k0, p3, m0, K, dist, range(3), **kw))
    assert got["success"].all()


@pytest.mark.parametrize("lo", [False, True], ids=["plain", "lo"])
def test_per_pair_cameras_failing_bearings_and_failures(lo):
    dists = [D, D * 0.5, D_RIM, D, D, D, D]
    k0, p3, m0, K = _scenes(600, list(range(31, 38)), [0.3] * 7, dists)
    dist = np.stack(dists)
    k0, p3, m0 = k0.copy(), p3.copy(), m0.copy()
    Kb = np.stack([K] * 7)
    Kb[1, 0, 0] = 300.0                           # per-pair K
    Kb[1, 0, 1] = 0.4
    k0[2, ::7] = Kb[2, :2, 2] + np.array([450.0, 0.0], dtype=np.float32)  # bearings that fail FE3 in pair 2
    dist[3, 2] = np.nan                           # invalid coefficients
    m0[4, 2:] = -1                                # fewer than 3 valid matches
    k0[5, ::3] = np.nan                           # NaN keypoints
    Kb[6, 0, 0] = -1.0                            # invalid K0
    assert not fo.usable(Kb[2], D_RIM, k0[2, ::7][:5]).any()
    fn = estimate_absolute_pose_lo_fisheye if lo else estimate_absolute_pose_fisheye
    got = {k: v.cpu().numpy() for k, v in fn(_t(k0), _t(p3), _t(m0), _t(Kb), _t(dist)).items()}
    f = fo.lo_absolute_pose_pair if lo else fo.absolute_pose_pair
    outs = [f(k0[p], p3[p], m0[p], Kb[p], 8.0, 100, 0.99, 0, dist[p]) for p in range(7)]
    _compare(lo, got, {k: np.stack([np.asarray(o[k]) for o in outs]) for k in outs[0]})
    assert got["success"][[0, 2, 5]].all() and not got["success"][[3, 4, 6]].any()
    assert not got["inliers"][2, ::7].any()
    assert got["num_hypotheses"][3] == 0 and got["best_hypothesis"][3] == -1


@pytest.mark.parametrize("lo", [False, True], ids=["plain", "lo"])
def test_scale_batch(lo):
    B, M = 32, 4096
    k0, p3, m0, K = _scenes(M, [100 + i for i in range(B)], [0.2, 0.5, 0.7, 0.4] * 8, [D] * B)
    dist = np.stack([D] * B)
    got = _run(lo, k0, p3, m0, K, dist, max_iters=256, confidence=1.0)
    pairs = [0, 13, 31]
    _compare(lo, got, _oracle(lo, k0, p3, m0, K, dist, pairs, max_iters=256, confidence=1.0), pairs)
    again = _run(lo, k0, p3, m0, K, dist, max_iters=256, confidence=1.0)
    for k in got:
        assert np.array_equal(got[k], again[k]), k


@pytest.mark.parametrize("lo", [False, True], ids=["plain", "lo"])
def test_matcher_output_without_read_back(lo):
    # matches0 from the nearest-neighbour matcher on descriptors that encode the scene's correspondences, fed straight
    # into the estimator on the device
    from lightglue_b200.nn_matcher import NearestNeighborMatcher
    M = 512
    k0, p3, m0, K = _scenes(M, [51], [0.3], [D])
    N = p3.shape[1]
    g = torch.Generator().manual_seed(5)
    desc1 = torch.nn.functional.normalize(torch.randn(1, N, 128, generator=g), dim=-1)
    idx = torch.from_numpy(np.where(m0[0] >= 0, m0[0], 0))
    desc0 = desc1[0, idx].clone()[None]
    desc0[0, torch.from_numpy(m0[0] < 0)] = torch.nn.functional.normalize(torch.randn(int((m0[0] < 0).sum()), 128,
                                                                                       generator=g), dim=-1)
    mt = NearestNeighborMatcher()({"image0": {"descriptors": desc0.cuda()},
                                   "image1": {"descriptors": desc1.cuda()}})["matches0"]
    fn = estimate_absolute_pose_lo_fisheye if lo else estimate_absolute_pose_fisheye
    got = {k: v.cpu().numpy() for k, v in fn(_t(k0), _t(p3), mt, _t(K), _t(D)).items()}
    _compare(lo, got, _oracle(lo, k0, p3, mt.cpu().numpy(), K, D[None], [0]))
    assert got["success"][0]


# ---- the bound cases of test_gpu_geometry_bounds.py, with the fisheye lens ----

def _localization_fisheye(m, outliers, seed, unmatched):
    k0, p3, m0, _, K, _, _, _ = fo.scene(m, outliers, seed, D, unmatched=unmatched)
    return k0, p3, m0, K


gb.ESTIMATORS.update({e.name: e for e in (
    gb.Est("PnP-fisheye", lambda a, b, m0, K, **kw: estimate_absolute_pose_fisheye(_t(a), _t(b), _t(m0), _t(K),
                                                                                   _t(D), **kw),
           lambda a, b, m0, K, thr, it, conf, seed: fo.absolute_pose_pair(a, b, m0, K, thr, it, conf, seed, D),
           EXACT, ("inliers",), {"R": "R", "t": "t"}, _localization_fisheye, 8.0, False, 512,
           "geo_pnp_workspace_bytes", relative=False),
    gb.Est("LO-PnP-fisheye", lambda a, b, m0, K, **kw: estimate_absolute_pose_lo_fisheye(_t(a), _t(b), _t(m0),
                                                                                         _t(K), _t(D), **kw),
           lambda a, b, m0, K, thr, it, conf, seed: fo.lo_absolute_pose_pair(a, b, m0, K, thr, it, conf, seed, D),
           LO_EXACT, ("inliers",), {"R": "R", "t": "t"}, _localization_fisheye, 8.0, False, 512,
           "geo_lo_pnp_workspace_bytes", lo=True, relative=False),
)})
NAMES = ["PnP-fisheye", "LO-PnP-fisheye"]


@pytest.mark.parametrize("name", NAMES)
def test_bound_one_split_of_several_tiles(name):
    gb.test_one_split_of_several_tiles(name)


@pytest.mark.parametrize("name", NAMES)
def test_bound_most_splits(name):
    gb.test_most_splits(name, (1 << 17) + 37, 0.1)


@pytest.mark.parametrize("name", NAMES)
def test_bound_more_pairs_than_a_grid_column(name):
    gb.test_more_pairs_than_a_grid_column(name)


@pytest.mark.parametrize("max_iters", [1, 255, 257, 513])
@pytest.mark.parametrize("name", NAMES)
def test_bound_chunk_edges(name, max_iters):
    gb.test_chunk_edges(name, max_iters)


@pytest.mark.parametrize("name", NAMES)
def test_bound_adaptive_stop_mid_budget(name):
    gb.test_adaptive_stop_mid_budget(name)


@pytest.mark.parametrize("name", NAMES)
def test_bound_empty_pairs(name):
    gb.test_empty_pairs(name)


@pytest.mark.parametrize("thr2", [0.0, gb.SUBNORMAL, gb.FLT_MIN, float("inf")],
                         ids=["zero", "subnormal", "flt_min", "inf"])
@pytest.mark.parametrize("name", NAMES)
def test_bound_threshold_extremes(name, thr2):
    gb.test_threshold_extremes(name, thr2)


@pytest.mark.parametrize("case", ["8192x6144", "offset", "integer"])
@pytest.mark.parametrize("name", NAMES)
def test_bound_coordinates(name, case):
    gb.test_coordinates(name, case)


@pytest.mark.parametrize("name", NAMES)
def test_bound_non_finite_keypoints_are_invalid(name):
    gb.test_non_finite_keypoints_are_invalid(name)


@pytest.mark.parametrize("name", NAMES)
def test_bound_duplicate_points_and_matches(name):
    gb.test_duplicate_points_and_matches(name)
