"""GPU MAGSAC++ homography and fundamental matrix (lightglue_b200.geometry.find_homography_magsac and
find_fundamental_magsac over include/geometry_b200.h, steps MH1-MH8 and MF1-MF8) against the numpy oracle, pair by pair:
the same seeding hypothesis, samples drawn, local optimisations, cost, counts and inliers, and the model within 1e-8;
failures, the loss scale against the user's threshold, budgets at the chunk edges, batch shapes, CUDA graphs, and the
matchers' device output as input."""
import numpy as np
import pytest
import torch

from lightglue_b200 import LightGlue, NearestNeighborMatcher, synth
from lightglue_b200.geometry import (find_fundamental_lo, find_fundamental_magsac, find_homography_lo,
                                     find_homography_magsac)
from oracle import geometry_oracle as go
from oracle import geometry_synth as gs
from oracle import magsac_oracle as mo

pytestmark = pytest.mark.gpu

EXACT = ("best_hypothesis", "num_hypotheses", "num_local_optimizations", "cost", "num_inliers", "success")
KINDS = {"H": (find_homography_magsac, find_homography_lo, go.HOMOGRAPHY, 2000, 0.995),
         "F": (find_fundamental_magsac, find_fundamental_lo, go.FUNDAMENTAL, 1000, 0.99)}


def _scene(kind, m, outliers, seed, **kw):
    return (gs.planar if kind == "H" else gs.two_view)(m, outliers, seed, **kw)


def _run(kind, k0, k1, m0, lo=False, **kw):
    fn = KINDS[kind][1] if lo else KINDS[kind][0]
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()  # noqa: E731
    out = fn(t(k0), t(k1), t(m0), **kw)
    return {k: v.cpu().numpy() for k, v in out.items()}


def _oracle(kind, k0, k1, m0, ransac_reproj_threshold=3.0, max_threshold=7.5, max_iters=None, confidence=None,
            seed=0, pairs=None):
    _, _, k, mi, conf = KINDS[kind]
    mi = mi if max_iters is None else max_iters
    conf = conf if confidence is None else confidence
    pairs = range(len(m0)) if pairs is None else pairs
    return [mo.magsac_hf_pair(k, k0[b], k1[b], m0[b], ransac_reproj_threshold, max_threshold, mi, conf, seed)
            for b in pairs]


def _assert_equal(kind, got, refs, pairs=None):
    pairs = range(len(refs)) if pairs is None else pairs
    for r, b in zip(refs, pairs):
        for k in EXACT:
            assert got[k][b] == r[k], (kind, b, k, got[k][b], r[k])
        assert np.array_equal(got["inliers"][b], r["inliers"]), (b, int((got["inliers"][b] != r["inliers"]).sum()))
        assert np.isfinite(got[kind][b]).all(), b
        assert np.abs(got[kind][b] - r[kind]).max() <= 1e-8 * max(np.abs(r[kind]).max(), 1e-300), (b, got[kind][b],
                                                                                                     r[kind])


def _batch(kind, m, outliers, seeds, unmatched=0.1):
    return gs.batch(kind, m, outliers, seeds, unmatched=unmatched)[:3]


@pytest.mark.parametrize("kind", ["H", "F"])
@pytest.mark.parametrize("outliers", [0.2, 0.5, 0.7])
@pytest.mark.parametrize("confidence", [0.995, 1.0])
def test_matches_the_oracle(kind, outliers, confidence):
    pairs = [_scene(kind, 1024, outliers, 100 + b, noise=1.0, unmatched=u) for b, u in enumerate((0.05, 0.2, 0.35, 0.5))]
    k0, k1, m0 = (np.stack([p[i] for p in pairs]) for i in range(3))
    got = _run(kind, k0, k1, m0, confidence=confidence)
    _assert_equal(kind, got, _oracle(kind, k0, k1, m0, confidence=confidence))
    assert got["success"].all()
    if confidence == 1.0:
        assert (got["num_hypotheses"] == KINDS[kind][3]).all()


@pytest.mark.parametrize("kind", ["H", "F"])
@pytest.mark.parametrize("max_threshold", [1.5, 3.0, 12.0])
def test_loss_scale_below_at_and_above_the_threshold(kind, max_threshold):
    k0, k1, m0 = _batch(kind, 1024, [0.3, 0.6], [51, 52])
    got = _run(kind, k0, k1, m0, max_threshold=max_threshold)
    _assert_equal(kind, got, _oracle(kind, k0, k1, m0, max_threshold=max_threshold))
    # the inliers and their count are the user threshold's, whatever the loss scale
    for b in range(2):
        e = go.errors(KINDS[kind][2], got[kind][b].reshape(1, 9), go.compact(k0[b], k1[b], m0[b])[1])[0]
        assert got["num_inliers"][b] == int((e < np.float32(9.0)).sum())


@pytest.mark.parametrize("kind", ["H", "F"])
@pytest.mark.parametrize("max_iters", [1, 255, 257, 513])
def test_budgets_at_the_chunk_edges(kind, max_iters):
    k0, k1, m0 = _batch(kind, 700, [0.2, 0.5], [61, 62])
    got = _run(kind, k0, k1, m0, max_iters=max_iters, confidence=1.0)
    assert (got["num_hypotheses"] == max_iters).all()
    _assert_equal(kind, got, _oracle(kind, k0, k1, m0, max_iters=max_iters, confidence=1.0))


@pytest.mark.parametrize("kind", ["H", "F"])
def test_matches_the_oracle_at_scale(kind):
    k0, k1, m0 = _batch(kind, 4096, [0.2, 0.5, 0.7, 0.6] * 8, list(range(200, 232)))
    got = _run(kind, k0, k1, m0, max_iters=5000, confidence=1.0)
    assert (got["num_hypotheses"] == 5000).all() and got["success"].all()
    _assert_equal(kind, got, _oracle(kind, k0, k1, m0, max_iters=5000, confidence=1.0, pairs=[2, 29]), pairs=[2, 29])


@pytest.mark.parametrize("kind", ["H", "F"])
def test_more_pairs_than_two_waves(kind):
    B = 2 * torch.cuda.get_device_properties(0).multi_processor_count + 1
    k0, k1, m0 = _batch(kind, 300, [0.3] * B, list(range(300, 300 + B)))
    got = _run(kind, k0, k1, m0, max_iters=300)
    _assert_equal(kind, got, _oracle(kind, k0, k1, m0, max_iters=300, pairs=[0, B // 2, B - 1]),
                  pairs=[0, B // 2, B - 1])


@pytest.mark.parametrize("kind", ["H", "F"])
def test_empty_batch_and_empty_pairs(kind):
    got = _run(kind, np.zeros((0, 5, 2), np.float32), np.zeros((0, 5, 2), np.float32), np.zeros((0, 5), np.int64))
    assert all(v.shape[0] == 0 for v in got.values())
    got = _run(kind, np.zeros((2, 0, 2), np.float32), np.zeros((2, 7, 2), np.float32), np.zeros((2, 0), np.int64))
    assert not got["success"].any() and (got["best_hypothesis"] == -1).all() and (got["cost"] == 0).all()
    assert got["inliers"].shape == (2, 0) and not got[kind].any()


@pytest.mark.parametrize("kind", ["H", "F"])
@pytest.mark.parametrize("case", ["few", "collinear"])
def test_failures(kind, case):
    if case == "few":
        k0, k1, m0, _, _ = _scene(kind, 256, 0.0, 7, unmatched=0.0)
        m0 = m0.copy()
        m0[(4 if kind == "H" else 8) - 1:] = -1
    else:
        k0 = np.stack([np.linspace(0, 600, 300), np.linspace(10, 400, 300)], 1).astype(np.float32)
        k1 = k0.copy()
        m0 = np.arange(300, dtype=np.int64)
    got = _run(kind, k0[None], k1[None], m0[None], max_iters=512)
    assert not got["success"][0] and not got["inliers"].any() and got["num_inliers"][0] == 0
    assert got["cost"][0] == 0 and got["num_local_optimizations"][0] == 0 and not got[kind].any()
    _assert_equal(kind, got, _oracle(kind, k0[None], k1[None], m0[None], max_iters=512))


@pytest.mark.parametrize("kind", ["H", "F"])
def test_out_of_range_indices_and_nan_keypoints_are_unmatched(kind):
    k0, k1, m0, _, _ = _scene(kind, 512, 0.3, 8)
    bad = m0.copy()
    bad[::7] = 512 + np.arange(bad[::7].size)  # past N
    bad[3::11] = -5
    k0n = k0.copy()
    k0n[5::13, 1] = np.nan
    clean = np.where((bad >= 0) & (bad < 512), bad, -1)
    clean[5::13] = -1
    a = _run(kind, k0n[None], k1[None], bad[None])
    b = _run(kind, k0[None], k1[None], clean[None])
    for k in a:
        assert np.array_equal(a[k], b[k]), k
    _assert_equal(kind, a, _oracle(kind, k0[None], k1[None], clean[None]))


@pytest.mark.parametrize("kind", ["H", "F"])
def test_samples_are_those_of_lo(kind):
    # one sample: both estimators solve hypothesis 0 of the same hash; at the full budget the best hypothesis names a
    # sample whose minimal model is the one the LO estimator solves at that index
    k0, k1, m0 = _batch(kind, 1024, [0.0, 0.3], [105, 106], unmatched=0.0)
    a = _run(kind, k0, k1, m0, lo=True, max_iters=1)
    b = _run(kind, k0, k1, m0, max_iters=1)
    assert (a["best_hypothesis"] == 0).all() and (b["best_hypothesis"] == 0).all()
    assert np.array_equal(a["num_hypotheses"], b["num_hypotheses"])
    full = _run(kind, k0, k1, m0, max_iters=512, confidence=1.0)
    lo = _run(kind, k0, k1, m0, lo=True, max_iters=512, confidence=1.0)
    for i in range(2):  # go.hypotheses is the LO oracles' sampler and solver, which the LO estimator equals
        _, pts = go.compact(k0[i], k1[i], m0[i])
        h = np.array([full["best_hypothesis"][i], lo["best_hypothesis"][i]], dtype=np.int64)
        assert go.hypotheses(KINDS[kind][2], 0, h, pts, go.normalisation(pts))[1].all()
    _assert_equal(kind, full, _oracle(kind, k0, k1, m0, max_iters=512, confidence=1.0))


@pytest.mark.parametrize("kind", ["H", "F"])
def test_batch_equals_single_pairs_and_repeats(kind):
    k0, k1, m0 = _batch(kind, 777, [0.3, 0.6, 0.1], [31, 32, 33], unmatched=[0.1, 0.4, 0.0])
    full = _run(kind, k0, k1, m0)
    again = _run(kind, k0, k1, m0)
    for k in full:
        assert np.array_equal(full[k], again[k]), k
    for b in range(3):
        one = _run(kind, k0[b:b + 1], k1[b:b + 1], m0[b:b + 1])
        for k in full:
            assert np.array_equal(full[k][b], one[k][0]), (b, k)


@pytest.mark.parametrize("kind", ["H", "F"])
def test_cuda_graph_replay_equals_eager(kind):
    fn = KINDS[kind][0]
    k0, k1, m0 = (torch.from_numpy(x).cuda() for x in _batch(kind, 1024, [0.3, 0.5], [41, 42]))
    eager = fn(k0, k1, m0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn(k0, k1, m0)  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        captured = fn(k0, k1, m0)
    for v in captured.values():
        v.zero_()
    g.replay()
    torch.cuda.synchronize()
    for k in eager:
        assert torch.equal(eager[k], captured[k]), k


def test_composes_with_lightglue():
    torch.manual_seed(0)
    data, perm = synth.make_pair(1024, seed=2024)
    rng = np.random.default_rng(5)
    Hm = gs.true_homography(rng)
    k0 = data["image0"]["keypoints"][0].numpy().astype(np.float64)
    k1 = gs.apply_h(Hm, k0[perm[0].numpy()]) + rng.normal(0.0, 0.5, (1024, 2))
    data["image1"]["keypoints"] = torch.from_numpy(k1.astype(np.float32))[None]
    matcher = LightGlue(features=None, depth_confidence=-1, width_confidence=-1, precision="bf16x3")
    matcher.load_state_dict(synth.make_state_dict(), strict=False)
    matcher = matcher.eval().cuda()
    cuda = {k: {kk: vv.cuda() for kk, vv in v.items()} for k, v in data.items()}
    with torch.no_grad():
        m0 = matcher.forward_async(cuda).tensors["matches0"]
        r = find_homography_magsac(cuda["image0"]["keypoints"], cuda["image1"]["keypoints"], m0)
    got = {k: v.cpu().numpy() for k, v in r.items()}
    m0 = m0.cpu().numpy()
    assert (m0 >= 0).sum() >= 100 and got["success"][0]
    _assert_equal("H", got, _oracle("H", data["image0"]["keypoints"].numpy(), data["image1"]["keypoints"].numpy(), m0))


def test_composes_with_the_nearest_neighbour_matcher_and_guided_matching():
    # descriptors that match through a two-view geometry: image 1's are image 0's permuted, with noise
    k0, k1, m0, truth, Ft = gs.two_view(1024, 0.3, 17, noise=0.5, unmatched=0.0)
    rng = np.random.default_rng(17)
    d0 = rng.normal(size=(1024, 128))
    d0 /= np.linalg.norm(d0, axis=1, keepdims=True)
    d1 = np.zeros_like(d0)
    d1[m0] = d0 + rng.normal(0.0, 0.02, d0.shape)
    d1 /= np.linalg.norm(d1, axis=1, keepdims=True)
    dev = lambda x: torch.as_tensor(np.asarray(x)[None]).float().cuda()  # noqa: E731
    data = {"image0": {"descriptors": dev(d0), "keypoints": dev(k0)},
            "image1": {"descriptors": dev(d1), "keypoints": dev(k1)}}
    nn = NearestNeighborMatcher()
    mm = nn(data)["matches0"]
    r = find_fundamental_magsac(data["image0"]["keypoints"], data["image1"]["keypoints"], mm)
    guided = nn(data, F=r["F"], valid=r["success"])
    got = {k: v.cpu().numpy() for k, v in r.items()}
    mm = mm.cpu().numpy()
    assert (mm >= 0).sum() >= 500 and got["success"][0]
    _assert_equal("F", got, _oracle("F", k0[None], k1[None], mm))
    g = guided["matches0"].cpu().numpy()[0]
    assert (g >= 0).sum() >= 500
