"""GPU 3D rigid and similarity RANSAC (lightglue_b200.geometry.estimate_rigid_3d and estimate_similarity_3d over
include/geometry_b200.h, steps RG1-RG7) against the numpy oracle, pair by pair: the same best hypothesis, samples
drawn, counts and inliers, and R, t and scale within 1e-8; outlier fractions, budgets, failures, launch-shape bounds,
batch composition, CUDA graphs, the matchers' device output as input, and keypoints lifted from depth maps."""
import numpy as np
import pytest
import torch

from lightglue_b200 import LightGlue, NearestNeighborMatcher, synth
from lightglue_b200.geometry import estimate_rigid_3d, estimate_similarity_3d
from oracle import rigid_oracle as ro

pytestmark = pytest.mark.gpu

EXACT = ("best_hypothesis", "num_hypotheses", "num_inliers", "success")
FN = {ro.RIGID: estimate_rigid_3d, ro.SIMILARITY: estimate_similarity_3d}
KINDS = [ro.RIGID, ro.SIMILARITY]
THR = 0.03


def _dev(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _run(kind, p0, p1, m0, thr=THR, **kw):
    out = FN[kind](_dev(p0), _dev(p1), _dev(m0), thr, **kw)
    return {k: v.cpu().numpy() for k, v in out.items()}


def _oracle(kind, p0, p1, m0, thr=THR, max_iters=1000, confidence=0.99, seed=0, pairs=None):
    pairs = range(len(m0)) if pairs is None else pairs
    return [ro.estimate_pair(kind, p0[b], p1[b], m0[b], thr, max_iters, confidence, seed) for b in pairs]


def _close(got, want):
    return np.abs(got - want).max() <= 1e-8 * max(np.abs(want).max(), 1e-300)


def _assert_equal(kind, got, refs, pairs=None):
    pairs = range(len(refs)) if pairs is None else pairs
    for r, b in zip(refs, pairs):
        for k in EXACT:
            assert got[k][b] == r[k], (b, k, got[k][b], r[k])
        assert np.array_equal(got["inliers"][b], r["inliers"]), (b, int((got["inliers"][b] != r["inliers"]).sum()))
        for k in ("R", "t", "scale"):
            assert np.isfinite(got[k][b]).all(), (b, k)
            assert _close(got[k][b], np.asarray(r[k])), (b, k, got[k][b], r[k])
    ok = got["success"]
    assert (got["R"][~ok] == 0).all() and (got["t"][~ok] == 0).all() and (got["scale"][~ok] == 0).all()
    if kind == ro.RIGID:
        assert (got["scale"][ok] == 1.0).all()
    R = got["R"][ok]
    assert np.abs(R @ R.transpose(0, 2, 1) - np.eye(3)).max(initial=0) < 1e-12
    assert np.abs(np.linalg.det(R) - 1.0).max(initial=0) < 1e-12


def _batch(kind, m, outliers, seeds, noise=0.01, unmatched=(0.05, 0.2, 0.35, 0.5)):
    scenes = [ro.scene(kind, m, o, s, noise=noise, unmatched=unmatched[i % len(unmatched)])
              for i, (o, s) in enumerate(zip(outliers, seeds))]
    return tuple(np.stack([sc[i] for sc in scenes]) for i in (0, 1, 2, 4)) + ([sc[3] for sc in scenes],)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("outliers", [0.2, 0.5, 0.7])
@pytest.mark.parametrize("confidence", [0.99, 1.0])
def test_matches_the_oracle(kind, outliers, confidence):
    p0, p1, m0, _, truth = _batch(kind, 1024, [outliers] * 4, [100 + kind * 10 + b for b in range(4)])
    got = _run(kind, p0, p1, m0, confidence=confidence)
    _assert_equal(kind, got, _oracle(kind, p0, p1, m0, confidence=confidence))
    assert got["success"].all()
    if confidence == 1.0:
        assert (got["num_hypotheses"] == 1000).all()
    for b, (R, t, sc) in enumerate(truth):
        assert np.abs(got["R"][b] - R).max() < 0.01 and np.abs(got["t"][b] - t).max() < 0.02
        assert abs(got["scale"][b] / sc - 1) < 0.01


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("max_iters", [1, 255, 257, 513])
def test_budgets(kind, max_iters):
    p0, p1, m0, _, _ = _batch(kind, 600, [0.3, 0.6], [7, 8], noise=0.015)
    got = _run(kind, p0, p1, m0, max_iters=max_iters, confidence=1.0)
    assert (got["num_hypotheses"] == max_iters).all()
    _assert_equal(kind, got, _oracle(kind, p0, p1, m0, max_iters=max_iters, confidence=1.0))


@pytest.mark.parametrize("kind", KINDS)
def test_float64_inputs_and_seeds(kind):
    p0, p1, m0, _, _ = _batch(kind, 800, [0.4, 0.6, 0.2], [21, 22, 23])
    a, b = p0.astype(np.float64) + 1e-9, p1.astype(np.float64)  # read as float32, as the oracle reads them
    for seed in (0, 12345):
        got = _run(kind, a, b, m0, seed=seed)
        _assert_equal(kind, got, _oracle(kind, a, b, m0, seed=seed))


@pytest.mark.parametrize("kind", KINDS)
def test_more_pairs_than_sms_and_batch_invariance(kind):
    b = 2 * torch.cuda.get_device_properties(0).multi_processor_count + 1
    p0, p1, m0, _, _ = _batch(kind, 300, [0.2, 0.5, 0.7] * b, list(range(500, 500 + b)))
    m0[::3, ::7] = 300 + np.arange(m0[::3, ::7].shape[1])  # indices >= N are unmatched, like -1
    got = _run(kind, p0, p1, m0)
    pairs = [0, 1, 2, b // 2, b - 1]
    _assert_equal(kind, got, _oracle(kind, p0, p1, m0, pairs=pairs), pairs)
    for p in pairs:  # a pair alone gives what it gives in the batch, bit for bit
        alone = _run(kind, p0[p:p + 1], p1[p:p + 1], m0[p:p + 1])
        for k in got:
            assert np.array_equal(alone[k][0], got[k][p]), (p, k)


@pytest.mark.parametrize("kind", KINDS)
def test_one_large_pair(kind):
    p0, p1, m0, _, _ = _batch(kind, (1 << 17) + 37, [0.5], [31], unmatched=(0.1,))
    got = _run(kind, p0, p1, m0)
    _assert_equal(kind, got, _oracle(kind, p0, p1, m0))


@pytest.mark.parametrize("kind", KINDS)
def test_batch_of_32_by_2048(kind):
    p0, p1, m0, _, _ = _batch(kind, 2048, [0.2, 0.5, 0.7, 0.4] * 8, list(range(900, 932)))
    got = _run(kind, p0, p1, m0)
    assert got["success"].all()
    _assert_equal(kind, got, _oracle(kind, p0, p1, m0))


def _failure_batch(m=64):
    """Pairs that fail, or whose samples are partly degenerate, by RG3 and RG7, next to a normal pair."""
    g = np.random.default_rng(4)
    p0 = g.uniform(-1, 1, (6, m, 3)).astype(np.float32)
    p1 = (p0 * 0.9 + 0.5).astype(np.float32)
    m0 = np.tile(np.arange(m), (6, 1))
    m0[1, 2:] = -1                                     # 2 valid matches: n < 3
    p0[2, :, 0] = np.nan                               # every row NaN
    p0[3] = np.outer(np.linspace(-1, 1, m), [1.0, 2.0, 0.5])  # collinear in set 0: every sample degenerate
    p1[4, :, 1:] = 0.25                                # collinear in set 1
    p1[5, : m // 2] = p1[5, :1]                        # half the points coincident in set 1
    return p0, p1, m0


@pytest.mark.parametrize("kind", KINDS)
def test_failures_and_nan_rows(kind):
    p0, p1, m0 = _failure_batch()
    got = _run(kind, p0, p1, m0, max_iters=300)
    _assert_equal(kind, got, _oracle(kind, p0, p1, m0, max_iters=300))
    want_fail = [1, 2, 3, 4]
    assert [b for b in range(6) if not got["success"][b]] == want_fail
    assert (got["best_hypothesis"][want_fail] == -1).all() and (got["num_inliers"][want_fail] == 0).all()
    assert not got["inliers"][want_fail].any()
    assert got["num_hypotheses"][1] == got["num_hypotheses"][2] == 0 and got["num_hypotheses"][3] == 300


@pytest.mark.parametrize("kind", KINDS)
def test_empty_shapes(kind):
    p0, p1, m0, _, _ = _batch(kind, 50, [0.3, 0.3, 0.3], [1, 2, 3])
    for a, b, m in ((p0[:, :0], p1, m0[:, :0]), (p0, p1[:, :0], m0), (p0[:0], p1[:0], m0[:0])):
        got = _run(kind, a, b, m)
        assert got["R"].shape == (len(m), 3, 3) and got["inliers"].shape == m.shape
        assert not got["success"].any() and (got["R"] == 0).all() and (got["scale"] == 0).all()
        assert (got["best_hypothesis"] == -1).all() and (got["num_hypotheses"] == 0).all()


@pytest.mark.parametrize("kind", KINDS)
def test_repeats_and_cuda_graph_replay_are_bit_identical(kind):
    p0, p1, m0, _, _ = _batch(kind, 1500, [0.3, 0.5, 0.6], [61, 62, 63])
    a, b, c = _dev(p0), _dev(p1), _dev(m0)
    first = FN[kind](a, b, c, THR)
    for _ in range(2):
        again = FN[kind](a, b, c, THR)
        for k in first:
            assert torch.equal(first[k], again[k]), k
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        FN[kind](a, b, c, THR)  # warm-up on the capture stream
    torch.cuda.current_stream().wait_stream(stream)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = FN[kind](a, b, c, THR)
    for k in captured.values():
        k.zero_()
    graph.replay()
    torch.cuda.synchronize()
    for k in first:
        assert torch.equal(first[k], captured[k]), k


def _lift(kpts, depth, K):
    """INTEGRATION.md's recipe: keypoints [B, N, 2] of a depth map [B, H, W] to camera-frame points, NaN without
    depth."""
    b_idx = torch.arange(kpts.shape[0], device=kpts.device)[:, None]
    u, v = kpts[..., 0], kpts[..., 1]
    d = depth[b_idx, v.round().long(), u.round().long()]
    d = torch.where(d > 0, d, torch.nan)
    y = (v - K[1, 2]) / K[1, 1]
    x = (u - K[0, 2] - K[0, 1] * y) / K[0, 0]
    return torch.stack([x * d, y * d, d], -1)


def _plane_depth(K, n, c, h, w):
    """Analytic depth of the plane n.X = c seen by a camera with intrinsics K: d = c / (n . K^-1 [u, v, 1])."""
    v, u = np.mgrid[0:h, 0:w].astype(np.float64)
    ray = np.stack([(u - K[0, 2]) / K[0, 0], (v - K[1, 2]) / K[1, 1], np.ones_like(u)], -1)
    return c / (ray @ n)


def test_depth_lifting_recovers_a_known_motion():
    """Two views of one scene (a slanted plane): keypoints on integer pixels of view 0 and their projections in view
    1, both lifted from the views' analytic depth maps, give the known (R, t) of view 0 to view 1."""
    h, w = 480, 640
    K = np.array([[525.0, 0.0, 319.5], [0.0, 525.0, 239.5], [0.0, 0.0, 1.0]])
    R, t = ro.random_rotation(np.random.default_rng(5)), np.array([0.1, -0.05, 0.08])
    R = np.linalg.qr(np.eye(3) + 0.05 * (R - R.T))[0]  # a small rotation, so the plane stays in view
    R = R * np.sign(np.diag(R))[None]
    n0, c0 = np.array([0.1, -0.2, 1.0]), 3.0          # the plane in view 0's frame
    n1, c1 = R @ n0, c0 + (R @ n0) @ t                # the same plane in view 1's frame: X1 = R X0 + t
    g = np.random.default_rng(6)
    k0 = np.stack([g.integers(20, w - 20, 1500), g.integers(20, h - 20, 1500)], -1).astype(np.float64)
    d0 = _plane_depth(K, n0, c0, h, w)
    X0 = np.stack([(k0[:, 0] - K[0, 2]) / K[0, 0], (k0[:, 1] - K[1, 2]) / K[1, 1], np.ones(len(k0))], -1)
    X0 = X0 * d0[k0[:, 1].astype(int), k0[:, 0].astype(int)][:, None]
    X1 = X0 @ R.T + t
    k1 = (X1 @ K.T)[:, :2] / X1[:, 2:]
    k1 = np.round(k1)  # view 1's keypoints on integer pixels too; lifting them gives nearby points of the plane
    inside = (k1[:, 0] >= 0) & (k1[:, 0] < w) & (k1[:, 1] >= 0) & (k1[:, 1] < h)
    m0 = np.where(inside, np.arange(len(k0)), -1)
    m0[::9] = g.permutation(len(k0))[: len(m0[::9])]  # wrong matches
    d1 = _plane_depth(K, n1, c1, h, w)
    d1[:40] = 0.0                                     # a band without depth: NaN points, invalid matches
    Kt = torch.from_numpy(K).cuda()
    p0 = _lift(_dev(k0[None]), _dev(d0[None]), Kt)
    p1 = _lift(_dev(np.clip(k1, 0, [w - 1, h - 1])[None]), _dev(d1[None]), Kt)
    r = estimate_rigid_3d(p0, p1, _dev(m0[None]), 0.02)
    assert bool(r["success"][0]) and int(r["num_inliers"][0]) > 1000
    Rg, tg = r["R"][0].cpu().numpy(), r["t"][0].cpu().numpy()
    assert np.abs(Rg - R).max() < 2e-3 and np.abs(tg - t).max() < 5e-3, (Rg, R, tg, t)
    got = {k: v.cpu().numpy() for k, v in r.items()}
    _assert_equal(ro.RIGID, got, _oracle(ro.RIGID, p0.cpu().numpy(), p1.cpu().numpy(), m0[None], 0.02))


@pytest.mark.parametrize("kind", KINDS)
def test_composes_with_the_matcher(kind):
    """LightGlue's matches0, with no read-back, on keypoints lifted to 3D by a known scene."""
    torch.manual_seed(0)
    data, perm = synth.make_pair(1024, seed=2024)
    matcher = LightGlue(features=None, depth_confidence=-1, width_confidence=-1, precision="bf16x3")
    matcher.load_state_dict(synth.make_state_dict(), strict=False)
    matcher = matcher.eval().cuda()
    cuda = {k: {kk: vv.cuda() for kk, vv in v.items()} for k, v in data.items()}
    k0 = data["image0"]["keypoints"][0].numpy().astype(np.float64)
    g = np.random.default_rng(77)
    X0 = np.concatenate([(k0 - 512.0) / 500.0 * 2.0, g.uniform(1.5, 4.0, (len(k0), 1))], 1)
    R, sc, t = ro.random_rotation(g), (1.7 if kind == ro.SIMILARITY else 1.0), g.uniform(-1, 1, 3)
    X1 = sc * X0[perm[0].numpy()] @ R.T + t + g.normal(0, 0.003, X0.shape)  # image 1's keypoints are image 0's permuted
    with torch.no_grad():
        pending = matcher.forward_async(cuda)
        m0 = pending.tensors["matches0"]
        r = FN[kind](_dev(X0[None].astype(np.float32)), _dev(X1[None].astype(np.float32)), m0, 0.02)
    got = {k: v.cpu().numpy() for k, v in r.items()}
    m0 = m0.cpu().numpy()
    assert (m0 >= 0).sum() >= 100 and got["success"][0]
    assert np.abs(got["R"][0] - R).max() < 0.01 and abs(got["scale"][0] / sc - 1) < 0.01
    _assert_equal(kind, got, _oracle(kind, X0[None], X1[None], m0, 0.02))


@pytest.mark.parametrize("kind", KINDS)
def test_nearest_neighbour_matches(kind):
    g = np.random.default_rng(40 + kind)
    b, m, n, d, count = 3, 700, 800, 128, 300
    d0, d1 = g.normal(size=(b, m, d)), g.normal(size=(b, n, d))
    d1[:, :count] = d0[:, :count] + 0.4 * g.normal(size=(b, count, d))
    d0 /= np.linalg.norm(d0, axis=-1, keepdims=True)
    d1 /= np.linalg.norm(d1, axis=-1, keepdims=True)
    p0 = np.stack([ro.depth_points(g, m) for _ in range(b)])
    p1 = np.stack([ro.depth_points(g, n) for _ in range(b)])
    for i in range(b):
        _, _, _, (R, t, sc), _ = ro.scene(kind, 8, 0.0, 300 + i)
        p1[i, :count] = sc * p0[i, :count] @ R.T + t + g.normal(0, 0.005, (count, 3))
    f = lambda x: torch.from_numpy(x.astype(np.float32)).cuda()  # noqa: E731
    kp = lambda x: f(x[..., :2] * 100.0)  # noqa: E731  the matcher reads descriptors only
    data = {"image0": {"descriptors": f(d0), "keypoints": kp(p0)}, "image1": {"descriptors": f(d1), "keypoints": kp(p1)}}
    out = NearestNeighborMatcher(ratio_thresh=0.9, mutual_check=True)(data)
    r = FN[kind](f(p0), f(p1), out["matches0"], THR)
    got = {k: v.cpu().numpy() for k, v in r.items()}
    assert got["success"].all() and (got["num_inliers"] > 200).all()
    _assert_equal(kind, got, _oracle(kind, p0, p1, out["matches0"].cpu().numpy()))
