"""GPU LO-RANSAC relative pose (lightglue_b200.geometry.estimate_relative_pose_lo over include/geometry_b200.h, steps
L1-L8) against its numpy oracle, pair by pair: the same seeding solution, samples drawn, local optimisations, MSAC cost,
counts and masks, and E, R, t within 1e-8; failures, intrinsics, batch composition, CUDA graphs and the matcher's
device output as input.  The cases mirror tests/test_gpu_pose.py."""
import numpy as np
import pytest
import torch

from lightglue_b200 import LightGlue, synth
from lightglue_b200.geometry import estimate_relative_pose, estimate_relative_pose_lo
from oracle import lo_pose_oracle as lo
from oracle import pose_oracle as po

pytestmark = pytest.mark.gpu

K_A = np.array([[500.0, 0.0, 320.0], [0.0, 500.0, 240.0], [0.0, 0.0, 1.0]])
K_B = np.array([[620.0, 0.5, 300.0], [0.0, 580.0, 250.0], [0.0, 0.0, 1.0]])
K_C = np.array([[450.0, 0.0, 330.0], [0.0, 470.0, 230.0], [0.0, 0.0, 1.0]])
EXACT = ("best_hypothesis", "best_solution", "num_hypotheses", "num_local_optimizations", "cost", "num_inliers",
         "num_pose_inliers", "success")


def _run(k0, k1, m0, K0, K1=None, **kw):
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()  # noqa: E731
    out = estimate_relative_pose_lo(t(k0), t(k1), t(m0), t(K0), None if K1 is None else t(K1), **kw)
    return {k: v.cpu().numpy() for k, v in out.items()}


def _batched(K, b):
    K = np.asarray(K, dtype=np.float64)
    return np.broadcast_to(K, (b, 3, 3)) if K.shape == (3, 3) else K


def _oracle(k0, k1, m0, K0, K1=None, ransac_reproj_threshold=1.0, max_iters=1000, confidence=0.999,
            distance_threshold=50.0, seed=0, pairs=None):
    K0 = _batched(K0, len(m0))
    K1 = K0 if K1 is None else _batched(K1, len(m0))
    pairs = range(len(m0)) if pairs is None else pairs
    return [lo.lo_relative_pose_pair(k0[b], k1[b], m0[b], K0[b], K1[b], ransac_reproj_threshold, max_iters, confidence,
                                     distance_threshold, seed) for b in pairs]


def _assert_equal(got, refs, pairs=None):
    pairs = range(len(refs)) if pairs is None else pairs
    for r, b in zip(refs, pairs):
        for k in EXACT:
            assert got[k][b] == r[k], (b, k, got[k][b], r[k])
        for k in ("inliers", "pose_inliers"):
            assert np.array_equal(got[k][b], r[k]), (b, k, int((got[k][b] != r[k]).sum()))
        for k in ("E", "R", "t"):
            assert np.isfinite(got[k][b]).all(), (b, k)
            assert np.abs(got[k][b] - r[k]).max() <= 1e-8, (b, k, got[k][b], r[k])


def _scenes(m, outliers, seeds, unmatched, K0=None, K1=None):
    pairs = [po.calibrated_two_view(m, outliers, s, unmatched=u, K0=K0, K1=K1) for s, u in zip(seeds, unmatched)]
    return tuple(np.stack([p[i] for p in pairs]) for i in range(8))


@pytest.mark.parametrize("outliers", [0.2, 0.5, 0.7])
@pytest.mark.parametrize("confidence", [0.999, 1.0])
def test_matches_the_oracle(outliers, confidence):
    k0, k1, m0, _, K0, _, _, _ = _scenes(1024, outliers, [100, 101, 102, 103], (0.05, 0.2, 0.35, 0.5))
    got = _run(k0, k1, m0, K0, confidence=confidence)
    _assert_equal(got, _oracle(k0, k1, m0, K0, confidence=confidence))
    assert got["success"].all() and (got["num_local_optimizations"] >= 1).all()
    if confidence == 1.0:
        assert (got["num_hypotheses"] == 1000).all()


def test_draws_the_same_samples_as_plain_ransac():
    # with the same seed the first chunk's best-scoring sample is drawn by both estimators: same hash, same solver
    k0, k1, m0, _, K0, _, _, _ = _scenes(1024, 0.3, [105, 106], (0.1, 0.1))
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()  # noqa: E731
    a = estimate_relative_pose(t(k0), t(k1), t(m0), t(K0), confidence=1.0, max_iters=256)
    b = estimate_relative_pose_lo(t(k0), t(k1), t(m0), t(K0), confidence=1.0, max_iters=256)
    assert torch.equal(a["num_hypotheses"], b["num_hypotheses"])
    assert (b["best_hypothesis"] < 256).all() and b["success"].all()


def test_per_pair_intrinsics():
    pairs = [po.calibrated_two_view(1024, 0.3, 110 + b, K0=K0, K1=K1)
             for b, (K0, K1) in enumerate([(K_A, K_B), (K_B, K_C), (K_C, K_A)])]
    k0, k1, m0, _, K0, K1, _, _ = (np.stack([p[i] for p in pairs]) for i in range(8))
    got = _run(k0, k1, m0, K0, K1)
    _assert_equal(got, _oracle(k0, k1, m0, K0, K1))
    assert got["success"].all()


def test_one_k_equals_the_expanded_k():
    k0, k1, m0, _, _, _, _, _ = _scenes(1024, 0.4, [120, 121], (0.1, 0.1), K0=K_B)
    one = _run(k0, k1, m0, K_B)
    full = _run(k0, k1, m0, np.broadcast_to(K_B, (2, 3, 3)).copy(), np.broadcast_to(K_B, (2, 3, 3)).copy())
    for k in one:
        assert np.array_equal(one[k], full[k]), k
    _assert_equal(one, _oracle(k0, k1, m0, K_B))


def test_matches_the_oracle_at_scale():
    pairs = [po.calibrated_two_view(4096, o, 200 + b) for b, o in enumerate([0.2, 0.5, 0.7, 0.6] * 8)]
    k0, k1, m0 = (np.stack([p[i] for p in pairs]) for i in range(3))
    got = _run(k0, k1, m0, K_A, max_iters=5000, confidence=1.0)
    assert (got["num_hypotheses"] == 5000).all() and got["success"].all()
    _assert_equal(got, _oracle(k0, k1, m0, K_A, max_iters=5000, confidence=1.0, pairs=[2, 29]), pairs=[2, 29])


@pytest.mark.parametrize("valid", [0, 4])
def test_too_few_matches_fail(valid):
    k0, k1, m0, *_ = po.calibrated_two_view(256, 0.0, 7, unmatched=0.0)
    m0 = m0.copy()
    m0[valid:] = -1
    got = _run(k0[None], k1[None], m0[None], K_A)
    assert not got["success"][0] and got["num_inliers"][0] == 0 and not got["inliers"].any()
    assert not got["pose_inliers"].any() and got["num_pose_inliers"][0] == 0
    assert not got["E"].any() and not got["R"].any() and not got["t"].any()
    assert got["best_hypothesis"][0] == -1 and got["best_solution"][0] == -1 and got["num_hypotheses"][0] == 0
    assert got["num_local_optimizations"][0] == 0 and got["cost"][0] == 0


@pytest.mark.parametrize("bad", ["nan", "fx", "bottom"])
def test_an_invalid_k_fails_only_its_pair(bad):
    k0, k1, m0, _, _, _, _, _ = _scenes(1024, 0.3, [130, 131, 132], (0.1, 0.2, 0.0))
    K = np.broadcast_to(K_A, (3, 3, 3)).copy()
    good = _run(k0, k1, m0, K)
    if bad == "nan":
        K[1, 0, 2] = np.nan
    elif bad == "fx":
        K[1, 0, 0] = 0.0
    else:
        K[1, 2, 2] = 2.0
    got = _run(k0, k1, m0, K)
    assert not got["success"][1] and not got["E"][1].any() and got["best_hypothesis"][1] == -1
    assert not got["inliers"][1].any() and got["num_hypotheses"][1] == 0 and got["cost"][1] == 0
    for k in got:
        for b in (0, 2):
            assert np.array_equal(got[k][b], good[k][b]), (k, b)


def test_coincident_points_fail():
    p = np.full((300, 2), 100.0, dtype=np.float32)
    m0 = np.arange(300, dtype=np.int64)
    got = _run(p[None], p[None].copy(), m0[None], K_A, max_iters=512)
    assert not got["success"][0] and not got["inliers"].any() and got["num_inliers"][0] == 0
    _assert_equal(got, _oracle(p[None], p[None], m0[None], K_A, max_iters=512))


def test_pure_rotation_is_finite_and_equals_the_oracle():
    rng = np.random.default_rng(3)
    X = np.stack([rng.uniform(-4, 4, 800), rng.uniform(-3, 3, 800), rng.uniform(4, 12, 800)], 1)
    a = 0.1
    R = np.array([[np.cos(a), 0.0, np.sin(a)], [0.0, 1.0, 0.0], [-np.sin(a), 0.0, np.cos(a)]])
    p0 = X @ K_A.T
    p1 = (X @ R.T) @ K_A.T
    k0 = (p0[:, :2] / p0[:, 2:]).astype(np.float32)
    k1 = (p1[:, :2] / p1[:, 2:] + rng.normal(0, 0.3, (800, 2))).astype(np.float32)
    m0 = np.arange(800, dtype=np.int64)
    got = _run(k0[None], k1[None], m0[None], K_A)
    for k in ("E", "R", "t"):
        assert np.isfinite(got[k]).all(), k
    _assert_equal(got, _oracle(k0[None], k1[None], m0[None], K_A))


def test_out_of_range_indices_are_unmatched():
    k0, k1, m0, *_ = po.calibrated_two_view(512, 0.3, 8)
    bad = m0.copy()
    bad[::7] = 512 + np.arange(bad[::7].size)  # past N
    bad[3::11] = -5
    clean = np.where((bad >= 0) & (bad < 512), bad, -1)
    a = _run(k0[None], k1[None], bad[None], K_A)
    b = _run(k0[None], k1[None], clean[None], K_A)
    for k in a:
        assert np.array_equal(a[k], b[k]), k
    _assert_equal(a, _oracle(k0[None], k1[None], clean[None], K_A))


def test_batch_equals_single_pairs_and_repeats():
    k0, k1, m0, _, _, _, _, _ = _scenes(777, 0.3, [31, 32, 33], (0.1, 0.4, 0.0))
    full = _run(k0, k1, m0, K_A)
    again = _run(k0, k1, m0, K_A)
    for k in full:
        assert np.array_equal(full[k], again[k]), k
    for b in range(3):
        one = _run(k0[b:b + 1], k1[b:b + 1], m0[b:b + 1], K_A)
        for k in full:
            assert np.array_equal(full[k][b], one[k][0]), (b, k)


def test_another_seed_recovers_the_truth():
    k0, k1, m0, truth, _, _, R, t = po.calibrated_two_view(2048, 0.5, 9)
    a = _run(k0[None], k1[None], m0[None], K_A, seed=0)
    b = _run(k0[None], k1[None], m0[None], K_A, seed=987654321)
    assert a["best_hypothesis"][0] != b["best_hypothesis"][0]
    cos = (np.trace(b["R"][0].T @ R) - 1.0) / 2.0
    assert np.degrees(np.arccos(min(1.0, cos))) <= 0.3
    assert np.degrees(np.arccos(min(1.0, float(b["t"][0] @ t)))) <= 2.0
    _assert_equal(b, _oracle(k0[None], k1[None], m0[None], K_A, seed=987654321))


def test_composes_with_the_matcher():
    torch.manual_seed(0)
    data, perm = synth.make_pair(1024, seed=2024)
    k0 = data["image0"]["keypoints"][0].numpy().astype(np.float64)
    # the matcher's own image-0 keypoints, lifted to depths 4..12 and seen by a second camera
    rng = np.random.default_rng(5)
    K = np.array([[800.0, 0.0, 512.0], [0.0, 800.0, 384.0], [0.0, 0.0, 1.0]])
    d = rng.uniform(4, 12, 1024)
    X = np.c_[(k0[:, 0] - 512.0) / 800.0 * d, (k0[:, 1] - 384.0) / 800.0 * d, d]
    a = 0.05
    R = np.array([[np.cos(a), 0.0, np.sin(a)], [0.0, 1.0, 0.0], [-np.sin(a), 0.0, np.cos(a)]])
    p1 = (X[perm[0].numpy()] @ R.T + np.array([0.5, 0.0, 0.0])) @ K.T
    k1 = p1[:, :2] / p1[:, 2:] + rng.normal(0.0, 0.5, (1024, 2))
    data["image1"]["keypoints"] = torch.from_numpy(k1.astype(np.float32))[None]
    matcher = LightGlue(features=None, depth_confidence=-1, width_confidence=-1, precision="bf16x3")
    matcher.load_state_dict(synth.make_state_dict(), strict=False)
    matcher = matcher.eval().cuda()
    cuda = {k: {kk: vv.cuda() for kk, vv in v.items()} for k, v in data.items()}
    with torch.no_grad():
        pending = matcher.forward_async(cuda)
        m0 = pending.tensors["matches0"]
        r = estimate_relative_pose_lo(cuda["image0"]["keypoints"], cuda["image1"]["keypoints"], m0,
                                      torch.from_numpy(K).cuda())
    got = {k: v.cpu().numpy() for k, v in r.items()}
    m0 = m0.cpu().numpy()
    assert (m0 >= 0).sum() >= 100
    assert got["success"][0]
    kk0 = data["image0"]["keypoints"].numpy()
    kk1 = data["image1"]["keypoints"].numpy()
    _assert_equal(got, _oracle(kk0, kk1, m0, K))


def test_cuda_graph_replay_equals_eager():
    k0, k1, m0, _, K0, K1, _, _ = _scenes(1024, 0.3, [41, 42], (0.1, 0.1), K0=K_A, K1=K_B)
    k0, k1, m0, K0, K1 = (torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in (k0, k1, m0, K0, K1))
    eager = estimate_relative_pose_lo(k0, k1, m0, K0, K1)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        estimate_relative_pose_lo(k0, k1, m0, K0, K1)  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        captured = estimate_relative_pose_lo(k0, k1, m0, K0, K1)
    for v in captured.values():
        v.zero_()
    g.replay()
    torch.cuda.synchronize()
    for k in eager:
        assert torch.equal(eager[k], captured[k]), k
