"""GPU affine and partial affine RANSAC (lightglue_b200.geometry.estimate_affine_2d and estimate_affine_partial_2d over
include/geometry_b200.h, steps AF1-AF7) against the numpy oracle, pair by pair: the same best hypothesis, samples
drawn, counts and inliers, and A within 1e-8; budgets, refinement lengths, failures, batch composition, CUDA graphs,
the matchers' device output as input, and guided matching under the estimated model."""
import numpy as np
import pytest
import torch

from lightglue_b200 import LightGlue, NearestNeighborMatcher, synth
from lightglue_b200.geometry import estimate_affine_2d, estimate_affine_partial_2d
from oracle import affine_oracle as ao
from oracle import geometry_oracle as go

pytestmark = pytest.mark.gpu

EXACT = ("best_hypothesis", "num_hypotheses", "num_inliers", "success")
FN = {ao.AFFINE: estimate_affine_2d, ao.PARTIAL: estimate_affine_partial_2d}
KINDS = [ao.AFFINE, ao.PARTIAL]


def _dev(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _run(kind, k0, k1, m0, **kw):
    out = FN[kind](_dev(k0), _dev(k1), _dev(m0), **kw)
    return {k: v.cpu().numpy() for k, v in out.items()}


def _oracle(kind, k0, k1, m0, ransac_reproj_threshold=3.0, max_iters=2000, confidence=0.99, refine_iters=10, seed=0,
            pairs=None):
    pairs = range(len(m0)) if pairs is None else pairs
    return [ao.estimate_pair(kind, k0[b], k1[b], m0[b], ransac_reproj_threshold, max_iters, confidence, refine_iters,
                             seed) for b in pairs]


def _assert_equal(kind, got, refs, pairs=None):
    pairs = range(len(refs)) if pairs is None else pairs
    for r, b in zip(refs, pairs):
        for k in EXACT:
            assert got[k][b] == r[k], (b, k, got[k][b], r[k])
        assert np.array_equal(got["inliers"][b], r["inliers"]), (b, int((got["inliers"][b] != r["inliers"]).sum()))
        want = r["model"][:2]
        assert np.isfinite(got["A"][b]).all(), b
        assert np.abs(got["A"][b] - want).max() <= 1e-8 * max(np.abs(want).max(), 1e-300), (b, got["A"][b], want)
    _assert_structure(kind, got)


def _assert_structure(kind, got):
    A, ok = got["A"], got["success"]
    assert (A[~ok] == 0).all()
    if kind == ao.PARTIAL:
        assert np.array_equal(A[ok, 0, 0], A[ok, 1, 1]) and np.array_equal(A[ok, 0, 1], -A[ok, 1, 0])


def _batch(kind, m, outliers, seeds, noise=1.0, unmatched=(0.05, 0.2, 0.35, 0.5)):
    scenes = [ao.scene(kind, m, o, s, noise=noise, unmatched=unmatched[i % len(unmatched)])
              for i, (o, s) in enumerate(zip(outliers, seeds))]
    return tuple(np.stack([sc[i] for sc in scenes]) for i in range(5))


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("outliers", [0.2, 0.5, 0.7])
@pytest.mark.parametrize("confidence", [0.99, 1.0])
def test_matches_the_oracle(kind, outliers, confidence):
    k0, k1, m0, _, _ = _batch(kind, 1024, [outliers] * 4, [100 + kind * 10 + b for b in range(4)])
    got = _run(kind, k0, k1, m0, confidence=confidence)
    _assert_equal(kind, got, _oracle(kind, k0, k1, m0, confidence=confidence))
    assert got["success"].all()
    if confidence == 1.0:
        assert (got["num_hypotheses"] == 2000).all()


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("max_iters", [1, 255, 257, 513])
@pytest.mark.parametrize("refine_iters", [0, 1, 10])
def test_budgets_and_refinement_lengths(kind, max_iters, refine_iters):
    k0, k1, m0, _, _ = _batch(kind, 600, [0.3, 0.6], [7, 8], noise=1.5)
    kw = dict(max_iters=max_iters, refine_iters=refine_iters, confidence=1.0)
    got = _run(kind, k0, k1, m0, **kw)
    assert (got["num_hypotheses"] == max_iters).all()
    _assert_equal(kind, got, _oracle(kind, k0, k1, m0, **kw))


@pytest.mark.parametrize("kind", KINDS)
def test_more_pairs_than_sms_and_batch_invariance(kind):
    b = 2 * torch.cuda.get_device_properties(0).multi_processor_count + 1
    k0, k1, m0, _, _ = _batch(kind, 300, [0.2, 0.5, 0.7] * b, list(range(500, 500 + b)))
    m0[::3, ::7] = 300 + np.arange(m0[::3, ::7].shape[1])  # indices >= N are unmatched, like -1
    got = _run(kind, k0, k1, m0)
    pairs = [0, 1, 2, b // 2, b - 1]
    _assert_equal(kind, got, _oracle(kind, k0, k1, m0, pairs=pairs), pairs)
    for p in pairs:  # a pair alone gives what it gives in the batch, bit for bit
        alone = _run(kind, k0[p:p + 1], k1[p:p + 1], m0[p:p + 1])
        for k in got:
            assert np.array_equal(alone[k][0], got[k][p]), (p, k)


@pytest.mark.parametrize("kind", KINDS)
def test_one_large_pair(kind):
    k0, k1, m0, _, _ = _batch(kind, (1 << 17) + 37, [0.5], [31], unmatched=(0.1,))
    got = _run(kind, k0, k1, m0)
    _assert_equal(kind, got, _oracle(kind, k0, k1, m0))


@pytest.mark.parametrize("kind", KINDS)
def test_batch_of_32_by_2048(kind):
    k0, k1, m0, A, _ = _batch(kind, 2048, [0.2, 0.5, 0.7, 0.4] * 8, list(range(900, 932)))
    got = _run(kind, k0, k1, m0)
    assert got["success"].all()
    _assert_equal(kind, got, _oracle(kind, k0, k1, m0))
    corners = np.array([[0.0, 0.0, 1.0], [640.0, 0.0, 1.0], [640.0, 480.0, 1.0], [0.0, 480.0, 1.0]])
    err = np.linalg.norm(np.einsum("bij,kj->bki", got["A"] - A, corners), axis=-1).mean(1)
    assert err.max() < 2.0, err


def _failure_batch(kind, m=64):
    """Pairs that fail, or whose samples are partly degenerate, by AF3 and AF7, next to a normal pair."""
    g = np.random.default_rng(4)
    k0 = g.uniform(0, 640, (7, m, 2)).astype(np.float32)
    k1 = (k0 * 0.9 + 5.0).astype(np.float32)
    m0 = np.tile(np.arange(m), (7, 1))
    m0[1, 2:] = -1                                     # 2 valid matches: n < 3 for the affine
    m0[2, 1:] = -1                                     # 1 valid match: n < s for both
    k0[3, :, 0] = np.nan                               # every match invalid
    k0[4] = k0[4, :1]                                  # coincident in image 0: the normalisation fails
    k0[5, :, 1] = 2.0 * k0[5, :, 0] + 1.0              # collinear in image 0: every affine sample is degenerate
    k1[6, : m // 2] = k1[6, :1]                        # half the points coincident in image 1
    k1[6, :, 1] = 100.0 if kind == ao.AFFINE else k1[6, :, 1]  # collinear in image 1 (affine)
    return k0, k1, m0


@pytest.mark.parametrize("kind", KINDS)
def test_failures_and_nan_keypoints(kind):
    k0, k1, m0 = _failure_batch(kind)
    got = _run(kind, k0, k1, m0, max_iters=300)
    _assert_equal(kind, got, _oracle(kind, k0, k1, m0, max_iters=300))
    want_fail = [1, 2, 3, 4, 5, 6] if kind == ao.AFFINE else [2, 3, 4]
    assert [b for b in range(7) if not got["success"][b]] == want_fail
    assert (got["best_hypothesis"][want_fail] == -1).all() and (got["num_inliers"][want_fail] == 0).all()
    assert not got["inliers"][want_fail].any()
    empty = _run(kind, k0[:, :0], k1, m0[:, :0])
    assert not empty["success"].any() and empty["A"].shape == (7, 2, 3) and (empty["A"] == 0).all()


@pytest.mark.parametrize("kind", KINDS)
def test_repeats_and_cuda_graph_replay_are_bit_identical(kind):
    k0, k1, m0, _, _ = _batch(kind, 1500, [0.3, 0.5, 0.6], [61, 62, 63])
    a, b, c = _dev(k0), _dev(k1), _dev(m0)
    first = FN[kind](a, b, c)
    for _ in range(2):
        again = FN[kind](a, b, c)
        for k in first:
            assert torch.equal(first[k], again[k]), k
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        FN[kind](a, b, c)  # warm-up on the capture stream
    torch.cuda.current_stream().wait_stream(stream)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = FN[kind](a, b, c)
    for k in captured.values():
        k.zero_()
    graph.replay()
    torch.cuda.synchronize()
    for k in first:
        assert torch.equal(first[k], captured[k]), k


def _affine_scene_keypoints(kind, perm, k0, seed, noise=0.5):
    """image-1 keypoints: image 0's, permuted by perm, moved by a random transform of the kind plus noise"""
    _, _, _, A, _ = ao.scene(kind, 8, 0.0, seed)
    rng = np.random.default_rng(seed)
    x1 = k0[perm] @ A[:, :2].T + A[:, 2] + rng.normal(0.0, noise, (len(perm), 2))
    return x1.astype(np.float32), A


@pytest.mark.parametrize("kind", KINDS)
def test_composes_with_the_matcher(kind):
    torch.manual_seed(0)
    data, perm = synth.make_pair(1024, seed=2024)
    k0 = data["image0"]["keypoints"][0].numpy().astype(np.float64)
    k1, A = _affine_scene_keypoints(kind, perm[0].numpy(), k0, 77)
    data["image1"]["keypoints"] = torch.from_numpy(k1)[None]
    matcher = LightGlue(features=None, depth_confidence=-1, width_confidence=-1, precision="bf16x3")
    matcher.load_state_dict(synth.make_state_dict(), strict=False)
    matcher = matcher.eval().cuda()
    cuda = {k: {kk: vv.cuda() for kk, vv in v.items()} for k, v in data.items()}
    with torch.no_grad():
        pending = matcher.forward_async(cuda)
        m0 = pending.tensors["matches0"]
        r = FN[kind](cuda["image0"]["keypoints"], cuda["image1"]["keypoints"], m0)
    got = {k: v.cpu().numpy() for k, v in r.items()}
    m0 = m0.cpu().numpy()
    assert (m0 >= 0).sum() >= 100 and got["success"][0]
    corners = np.array([[0.0, 0.0, 1.0], [1024.0, 0.0, 1.0], [1024.0, 768.0, 1.0], [0.0, 768.0, 1.0]])
    assert np.abs((got["A"][0] - A) @ corners.T).max() <= 1.0
    kk0, kk1 = data["image0"]["keypoints"].numpy(), data["image1"]["keypoints"].numpy()
    _assert_equal(kind, got, _oracle(kind, kk0, kk1, m0))


def _nn_scene(kind, seed, b=3, m=700, n=800, d=128, count=300):
    """Unit descriptors where the first `count` rows of image 1 are noisy copies of image 0's, placed by a transform
    of the kind within about a pixel; the other keypoints are random."""
    g = np.random.default_rng(seed)
    d0 = g.normal(size=(b, m, d))
    d1 = g.normal(size=(b, n, d))
    d1[:, :count] = d0[:, :count] + 0.4 * g.normal(size=(b, count, d))
    d0 /= np.linalg.norm(d0, axis=-1, keepdims=True)
    d1 /= np.linalg.norm(d1, axis=-1, keepdims=True)
    k0 = g.uniform(0, 640, (b, m, 2))
    k1 = g.uniform(0, 640, (b, n, 2))
    for i in range(b):
        _, _, _, A, _ = ao.scene(kind, 8, 0.0, seed + i)
        k1[i, :count] = k0[i, :count] @ A[:, :2].T + A[:, 2] + g.normal(0.0, 0.7, (count, 2))
    f = lambda x: torch.from_numpy(x.astype(np.float32)).cuda()  # noqa: E731
    return {"image0": {"descriptors": f(d0), "keypoints": f(k0)}, "image1": {"descriptors": f(d1), "keypoints": f(k1)}}


@pytest.mark.parametrize("kind", KINDS)
def test_nearest_neighbour_matches_then_guided_matching_under_the_estimate(kind):
    t = 3.0
    data = _nn_scene(kind, 40 + kind)
    nn = NearestNeighborMatcher(ratio_thresh=0.9, mutual_check=True)
    plain = nn(data)
    r = FN[kind](data["image0"]["keypoints"], data["image1"]["keypoints"], plain["matches0"],
                 ransac_reproj_threshold=t)
    assert bool(r["success"].all())
    row = torch.tensor([0.0, 0.0, 1.0], dtype=torch.float64, device="cuda").expand(len(r["A"]), 1, 3)
    guided = nn(data, H=torch.cat([r["A"], row], 1), max_error=t)
    k0 = data["image0"]["keypoints"].cpu().numpy()
    k1 = data["image1"]["keypoints"].cpu().numpy()
    pm, ps = plain["matches0"].cpu().numpy(), plain["matching_scores0"].cpu().numpy()
    gm, gsc = guided["matches0"].cpu().numpy(), guided["matching_scores0"].cpu().numpy()
    inl = r["inliers"].cpu().numpy()
    A = r["A"].cpu().numpy()
    assert inl.sum() > 200
    # every unguided match the estimator marked as an inlier is kept by the guided call, with the identical score
    np.testing.assert_array_equal(gm[inl], pm[inl])
    np.testing.assert_array_equal(gsc[inl], ps[inl])
    for b in range(len(gm)):  # every guided match passes the affine inlier test
        i = np.flatnonzero(gm[b] >= 0)
        pts = np.concatenate([k0[b, i], k1[b, gm[b, i]]], 1).astype(np.float32)
        assert (ao.errors(A[b].reshape(1, 6), pts)[0] < np.float32(t * t)).all()
    # and the estimator's own mask is that test on the unguided matches
    want = [ao.estimate_pair(kind, k0[b], k1[b], pm[b], t) for b in range(len(pm))]
    _assert_equal(kind, {k: v.cpu().numpy() for k, v in r.items()}, want)
    for b in range(len(pm)):
        i = np.flatnonzero(pm[b] >= 0)
        pts = np.concatenate([k0[b, i], k1[b, pm[b, i]]], 1).astype(np.float32)
        e = go.errors(go.HOMOGRAPHY, ao.as_h(A[b].reshape(1, 6)), pts)[0]
        np.testing.assert_array_equal(inl[b, i], e < np.float32(t * t))
