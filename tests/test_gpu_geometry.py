"""GPU RANSAC (lightglue_b200.geometry over include/geometry_b200.h) against its numpy oracle, bit for bit: the same
hypotheses, counts, stops and inliers, and models within 1e-8; edge cases, batch composition, CUDA graphs and the
matcher's device output as input."""
import numpy as np
import pytest
import torch

from lightglue_b200 import LightGlue, synth
from lightglue_b200.geometry import find_fundamental, find_homography
from oracle import geometry_oracle as go
from oracle import geometry_synth as gs

pytestmark = pytest.mark.gpu

KINDS = {"H": (find_homography, go.HOMOGRAPHY, 3.0, 2000), "F": (find_fundamental, go.FUNDAMENTAL, 3.0, 1000)}


def _run(key, k0, k1, m0, **kw):
    fn = KINDS[key][0]
    out = fn(torch.from_numpy(k0).cuda(), torch.from_numpy(k1).cuda(), torch.from_numpy(m0).cuda(), **kw)
    return {k: v.cpu().numpy() for k, v in out.items()}


def _oracle(key, k0, k1, m0, ransac_reproj_threshold=3.0, max_iters=None, confidence=None, seed=0, pairs=None):
    _, kind, _, iters = KINDS[key]
    conf = confidence if confidence is not None else (0.995 if key == "H" else 0.99)
    pairs = range(len(m0)) if pairs is None else pairs
    return [go.estimate_pair(kind, k0[b], k1[b], m0[b], ransac_reproj_threshold, max_iters or iters, conf, seed)
            for b in pairs]


def _assert_equal(key, got, refs, pairs=None):
    pairs = range(len(refs)) if pairs is None else pairs
    for r, b in zip(refs, pairs):
        for k in ("best_hypothesis", "num_hypotheses", "num_inliers", "success"):
            assert got[k][b] == r[k], (b, k, got[k][b], r[k])
        assert np.array_equal(got["inliers"][b], r["inliers"]), (b, int((got["inliers"][b] != r["inliers"]).sum()))
        ref = r["model"]
        assert np.abs(got[key][b] - ref).max() <= 1e-8 * max(np.abs(ref).max(), 1e-300), (b, got[key][b], ref)


@pytest.mark.parametrize("key", ["H", "F"])
@pytest.mark.parametrize("outliers", [0.2, 0.5, 0.7])
@pytest.mark.parametrize("confidence", [0.995, 1.0])
def test_matches_the_oracle(key, outliers, confidence):
    # B = 4 pairs with 5 .. 50 % unmatched rows, so each pair has its own match count
    make = gs.planar if key == "H" else gs.two_view
    pairs = [make(1024, outliers, 100 + b, unmatched=u) for b, u in enumerate((0.05, 0.2, 0.35, 0.5))]
    k0, k1, m0 = (np.stack([p[i] for p in pairs]) for i in range(3))
    got = _run(key, k0, k1, m0, confidence=confidence)
    _assert_equal(key, got, _oracle(key, k0, k1, m0, confidence=confidence))
    assert got["success"].all()
    if confidence == 1.0:
        assert (got["num_hypotheses"] == KINDS[key][3]).all()


def test_matches_the_oracle_at_scale():
    k0, k1, m0, _, _ = gs.batch("H", 4096, [0.2, 0.5, 0.7, 0.6] * 8, list(range(200, 232)))
    got = _run("H", k0, k1, m0, max_iters=10000, confidence=1.0)
    assert (got["num_hypotheses"] == 10000).all() and got["success"].all()
    _assert_equal("H", got, _oracle("H", k0, k1, m0, max_iters=10000, confidence=1.0, pairs=[2, 29]), pairs=[2, 29])


@pytest.mark.parametrize("key,valid", [("H", 0), ("H", 3), ("F", 0), ("F", 7)])
def test_too_few_matches_fail(key, valid):
    make = gs.planar if key == "H" else gs.two_view
    k0, k1, m0, _, _ = make(256, 0.0, 7, unmatched=0.0)
    m0 = m0.copy()
    m0[valid:] = -1
    got = _run(key, k0[None], k1[None], m0[None])
    assert not got["success"][0] and got["num_inliers"][0] == 0 and not got["inliers"].any()
    assert not got[key].any() and got["best_hypothesis"][0] == -1 and got["num_hypotheses"][0] == 0


@pytest.mark.parametrize("key", ["H", "F"])
def test_collinear_points_fail(key):
    line = np.stack([np.linspace(0, 600, 300), np.linspace(10, 400, 300)], 1).astype(np.float32)
    m0 = np.arange(300, dtype=np.int64)
    got = _run(key, line[None], line[None].copy(), m0[None], max_iters=512)
    assert not got["success"][0] and not got["inliers"].any() and got["num_inliers"][0] == 0
    _assert_equal(key, got, _oracle(key, line[None], line[None], m0[None], max_iters=512))


def test_out_of_range_indices_are_unmatched():
    k0, k1, m0, _, _ = gs.planar(512, 0.3, 8)
    bad = m0.copy()
    bad[::7] = 512 + np.arange(bad[::7].size)  # past N
    bad[3::11] = -5
    clean = np.where((bad >= 0) & (bad < 512), bad, -1)
    a = _run("H", k0[None], k1[None], bad[None])
    b = _run("H", k0[None], k1[None], clean[None])
    for k in a:
        assert np.array_equal(a[k], b[k]), k
    _assert_equal("H", a, _oracle("H", k0[None], k1[None], clean[None]))


@pytest.mark.parametrize("key", ["H", "F"])
def test_batch_equals_single_pairs_and_repeats(key):
    k0, k1, m0, _, _ = gs.batch(key, 777, [0.3, 0.6, 0.1], [31, 32, 33], unmatched=[0.1, 0.4, 0.0])
    full = _run(key, k0, k1, m0)
    again = _run(key, k0, k1, m0)
    for k in full:
        assert np.array_equal(full[k], again[k]), k
    for b in range(3):
        one = _run(key, k0[b:b + 1], k1[b:b + 1], m0[b:b + 1])
        for k in full:
            assert np.array_equal(full[k][b], one[k][0]), (b, k)


def test_another_seed_recovers_the_truth():
    k0, k1, m0, truth, Hm = gs.planar(2048, 0.5, 9)
    a = _run("H", k0[None], k1[None], m0[None], seed=0)
    b = _run("H", k0[None], k1[None], m0[None], seed=987654321)
    assert a["best_hypothesis"][0] != b["best_hypothesis"][0]
    assert (b["inliers"][0] & truth).sum() / truth.sum() >= 0.98
    assert np.abs(gs.apply_h(b["H"][0], gs.CORNERS) - gs.apply_h(Hm, gs.CORNERS)).max() <= 1.0
    _assert_equal("H", b, _oracle("H", k0[None], k1[None], m0[None], seed=987654321))


def test_composes_with_the_matcher():
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
        pending = matcher.forward_async(cuda)
        m0 = pending.tensors["matches0"]
        r = find_homography(cuda["image0"]["keypoints"], cuda["image1"]["keypoints"], m0)
    got = {k: v.cpu().numpy() for k, v in r.items()}
    m0 = m0.cpu().numpy()
    assert (m0 >= 0).sum() >= 100
    corners = np.array([[0.0, 0.0], [1024.0, 0.0], [1024.0, 768.0], [0.0, 768.0]])
    assert got["success"][0]
    assert np.abs(gs.apply_h(got["H"][0], corners) - gs.apply_h(Hm, corners)).max() <= 1.0
    kk0 = data["image0"]["keypoints"].numpy()
    kk1 = data["image1"]["keypoints"].numpy()
    _assert_equal("H", got, _oracle("H", kk0, kk1, m0))


def test_cuda_graph_replay_equals_eager():
    k0, k1, m0, _, _ = gs.batch("F", 1024, [0.3, 0.5], [41, 42])
    k0, k1, m0 = (torch.from_numpy(x).cuda() for x in (k0, k1, m0))
    eager = find_fundamental(k0, k1, m0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        find_fundamental(k0, k1, m0)  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        captured = find_fundamental(k0, k1, m0)
    for v in captured.values():
        v.zero_()
    g.replay()
    torch.cuda.synchronize()
    for k in eager:
        assert torch.equal(eager[k], captured[k]), k
