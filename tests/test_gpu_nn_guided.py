"""Guided nearest-neighbour matching on the H100 against oracle/nn_guided_oracle.py: bit for bit where every product
and sum is exact, for H and F, at the gate's boundaries; monotonicity and the gate on any input; ungated pairs and an
all-passing gate against ``forward()`` without a model; synthetic scenes with repeated-structure decoys; ragged and
large batches, repeats and CUDA-graph replay; and SIFT -> NearestNeighborMatcher -> find_homography_lo -> guided
matching."""
import ctypes as C

import numpy as np
import pytest
import torch

from lightglue_b200 import SIFT, NearestNeighborMatcher, _cabi
from lightglue_b200.geometry import find_homography_lo
from oracle import geometry_oracle as geo
from oracle import geometry_synth as gs
from oracle import nn_guided_oracle as ngo
from oracle import sift_synth
from tests.test_nn_emulation import TOL_D, TOL_S  # the split-bf16 gates, calibrated by emulation

pytestmark = pytest.mark.gpu

KEYS = ("matches0", "matches1", "matching_scores0", "matching_scores1")
KIND = {"H": geo.HOMOGRAPHY, "F": geo.FUNDAMENTAL}
GATE_PX = {"H": 60.0, "F": 24.0}  # a disc of 60 px, a band of 2 x 24 px around the epipolar line


def _conf(ratio, dist, mutual):
    return {"ratio_thresh": ratio, "distance_thresh": dist, "mutual_check": mutual}


def _data(d0, d1, k0, k1, lens0=None, lens1=None):
    dev = lambda x: torch.as_tensor(x).float().cuda()  # noqa: E731
    data = {"image0": {"descriptors": dev(d0), "keypoints": dev(k0)},
            "image1": {"descriptors": dev(d1), "keypoints": dev(k1)}}
    if lens0 is not None:
        data["image0"]["num_keypoints"] = torch.tensor(lens0, dtype=torch.int32).cuda()
        data["image1"]["num_keypoints"] = torch.tensor(lens1, dtype=torch.int32).cuda()
    return data


def _guided(data, kind, model, valid=None, max_error=4.0, **conf):
    model = torch.as_tensor(np.array(model, dtype=np.float64)).cuda()
    v = None if valid is None else torch.as_tensor(np.asarray(valid)).cuda()
    return NearestNeighborMatcher(**conf)(data, max_error=max_error, valid=v, **{kind: model})


def _want(d0, d1, k0, k1, kind, model, valid=None, max_error=4.0, lens0=None, lens1=None, **conf):
    g = ngo.gate(KIND[kind], model, k0, k1, max_error, valid)
    return ngo.match(np.asarray(d0, np.float64), np.asarray(d1, np.float64), lens0, lens1, conf.get("ratio_thresh"),
                     conf.get("distance_thresh"), conf.get("mutual_check", True), gate=g), g


def _assert_equal(got, want, b_range=None):
    for k in KEYS:
        g, w = got[k].cpu().numpy(), want[k]
        if b_range is not None:
            g, w = g[b_range], w[b_range]
        np.testing.assert_array_equal(g, w, err_msg=k)
    for b in range(len(got["matches"])) if b_range is None else b_range:
        np.testing.assert_array_equal(got["matches"][b].cpu().numpy(), want["matches"][b])
        np.testing.assert_array_equal(got["scores"][b].cpu().numpy(), want["scores"][b])


def _grid_desc(g, b, m, n, d):
    """Entries k / 16, |k| <= 2: exact in bf16, every product and every sum of D <= 512 of them exact in fp32."""
    return tuple((g.integers(-2, 3, (b, rows, d)) / 16).astype(np.float32) for rows in (m, n))


def _scene(kind, g, b, m, n):
    """Keypoints in a 640 x 480 image and one model per pair: a near-identity H, or the F of a synthetic two-view
    scene.  GATE_PX[kind] lets a few per cent of the columns of a row through."""
    k0 = g.uniform([0, 0], [640, 480], (b, m, 2)).astype(np.float32)
    k1 = g.uniform([0, 0], [640, 480], (b, n, 2)).astype(np.float32)
    if kind == "H":
        model = np.stack([gs.true_homography(g) for _ in range(b)])
    else:
        model = np.stack([gs.two_view(8, 0.0, int(s))[4] for s in g.integers(0, 1000, b)])
    return k0, k1, model


@pytest.mark.parametrize("kind", ["H", "F"])
@pytest.mark.parametrize("ratio", [None, 0.8])
@pytest.mark.parametrize("dist", [None, 1.3])
@pytest.mark.parametrize("mutual", [True, False])
def test_exact_arithmetic_equals_the_oracle_bit_for_bit(kind, ratio, dist, mutual):
    g = np.random.default_rng(11)
    d0, d1 = _grid_desc(g, 3, 300, 260, 64)
    k0, k1, model = _scene(kind, g, 3, 300, 260)
    conf = _conf(ratio, dist, mutual)
    got = _guided(_data(d0, d1, k0, k1), kind, model, max_error=GATE_PX[kind], **conf)
    want, gate = _want(d0, d1, k0, k1, kind, model, max_error=GATE_PX[kind], **conf)
    assert 0.01 < gate.mean() < 0.5
    _assert_equal(got, want)


@pytest.mark.parametrize("d", [64, 128, 192, 256, 512])
@pytest.mark.parametrize("kind", ["H", "F"])
def test_exact_arithmetic_at_every_descriptor_size(d, kind):
    g = np.random.default_rng(d)
    d0, d1 = _grid_desc(g, 2, 200, 333, d)
    k0, k1, model = _scene(kind, g, 2, 200, 333)
    got = _guided(_data(d0, d1, k0, k1), kind, model, max_error=GATE_PX[kind], ratio_thresh=0.9)
    _assert_equal(got, _want(d0, d1, k0, k1, kind, model, max_error=GATE_PX[kind], ratio_thresh=0.9)[0])


@pytest.mark.parametrize("mutual", [True, False])
def test_planted_boundary_cases(mutual):
    """H = identity, max_error = 1: rows 0-5 of image 0 and their planted columns of image 1."""
    d = 128

    def e(i, x=1.0):
        v = np.zeros(d, np.float32)
        v[i] = x
        return v
    d0 = np.stack([e(0), e(1), e(2), e(3), e(4), e(5)])[None]
    d1 = np.stack([e(0), e(0, 0.875),           # row 0: the best column sits exactly at t2 and fails; 0.875 wins
                   e(1, 0.75), e(1, 0.75),      # row 1: a tie among gated columns (j1 = 2, s2 = s1): ratio fails
                   e(2, 0.5), e(2, 0.9375),     # row 2: one gated column (4): s2 = -inf, the ratio test passes
                   e(3),                        # row 3: its only candidate is gated out: nothing
                   e(4), e(5)])[None]           # row 4: a NaN keypoint; row 5: a gated twin of row 5
    k0 = np.array([[[10, 10], [100, 100], [200, 200], [300, 300], [np.nan, 5], [400, 400]]], np.float32)
    k1 = np.array([[[11, 10], [10, 10.5], [100, 100], [100.5, 100], [200, 200], [250, 200], [310, 300], [0, 5],
                    [400, 400.25]]], np.float32)
    model = np.eye(3)[None]
    conf = _conf(0.5, None, mutual)
    got = _guided(_data(d0, d1, k0, k1), "H", model, max_error=1.0, **conf)
    want, gate = _want(d0, d1, k0, k1, "H", model, max_error=1.0, **conf)
    assert not gate[0, 0, 0] and gate[0, 0, 1] and not gate[0, 4].any()
    _assert_equal(got, want)
    assert got["matches0"][0].tolist() == [1, -1, 4, -1, -1, 8]
    assert want["sides"][0][0]["j1"][1] == 2 and want["sides"][0][0]["s2"][1] == 0.75


def _unit_pair(g, b, m, n, d, dup=0.3):
    """Unit descriptors where a share `dup` of image 1 are noisy copies of image-0 rows (so many rows match)."""
    d0 = g.normal(size=(b, m, d))
    d1 = g.normal(size=(b, n, d))
    k = int(dup * min(m, n))
    d1[:, :k] = d0[:, :k] + 0.4 * g.normal(size=(b, k, d))
    d0 /= np.linalg.norm(d0, axis=-1, keepdims=True)
    d1 /= np.linalg.norm(d1, axis=-1, keepdims=True)
    return d0.astype(np.float32), d1.astype(np.float32)


def _place(kind, model, k0, k1, g, count):
    """Moves k1[:, :count] to where the model puts k0[:, :count], within about a pixel: H x0 plus noise, or the foot of
    a random point on the epipolar line F x0."""
    for b in range(k0.shape[0]):
        x0 = k0[b, :count].astype(np.float64)
        if kind == "H":
            k1[b, :count] = gs.apply_h(model[b], x0) + g.normal(0, 0.7, (count, 2))
        else:
            h0 = np.concatenate([x0, np.ones((count, 1))], 1)
            ln = h0 @ model[b].T
            x1 = k1[b, :count].astype(np.float64)
            r = (ln[:, :2] * x1).sum(1) + ln[:, 2]
            k1[b, :count] = x1 - (r / (ln[:, :2] ** 2).sum(1))[:, None] * ln[:, :2] + g.normal(0, 0.5, (count, 2))


def _pair_errors(kind, model, k0, k1, m0):
    """Gate of each matched (i, matches0[i]) row of every pair, by the oracle (False for unmatched rows)."""
    out = np.zeros(m0.shape, dtype=bool)
    for b in range(m0.shape[0]):
        i = np.flatnonzero(m0[b] >= 0)
        if i.size:
            pts = np.concatenate([k0[b, i], k1[b, m0[b, i]]], axis=1).astype(np.float32)
            err = geo.errors(KIND[kind], np.asarray(model[b], np.float64).reshape(1, 9), pts)[0]
            out[b, i] = err < np.float32(4.0 * 4.0)
    return out


def _monotone_and_gated(plain, got, kind, model, k0, k1):
    pm, ps = plain["matches0"].cpu().numpy(), plain["matching_scores0"].cpu().numpy()
    gm, gsc = got["matches0"].cpu().numpy(), got["matching_scores0"].cpu().numpy()
    assert _pair_errors(kind, model, k0, k1, gm)[gm >= 0].all()  # every guided match passes the gate
    keep = _pair_errors(kind, model, k0, k1, pm)  # unguided matches that pass the gate ...
    np.testing.assert_array_equal(gm[keep], pm[keep])  # ... are guided matches with the identical score
    np.testing.assert_array_equal(gsc[keep], ps[keep])
    return int(keep.sum()), int((gm >= 0).sum())


@pytest.mark.parametrize("kind", ["H", "F"])
@pytest.mark.parametrize("mutual", [True, False])
def test_monotone_in_the_gate_and_every_match_passes_it(kind, mutual):
    g = np.random.default_rng(3)
    d0, d1 = _unit_pair(g, 4, 700, 900, 256)
    k0, k1, model = _scene(kind, g, 4, 700, 900)
    _place(kind, model, k0, k1, g, 210)  # image 1's copies sit where the model puts their image-0 rows
    data = _data(d0, d1, k0, k1)
    conf = _conf(0.9, None, mutual)
    plain = NearestNeighborMatcher(**conf)(data)
    kept, total = _monotone_and_gated(plain, _guided(data, kind, model, **conf), kind, model, k0, k1)
    assert kept > 100 and total >= kept, (kept, total)


def test_ungated_pairs_and_an_all_passing_gate_equal_forward_without_a_model():
    g = np.random.default_rng(8)
    d0, d1 = _unit_pair(g, 4, 500, 450, 128)
    k0, k1, model = _scene("F", g, 4, 500, 450)
    data = _data(d0, d1, k0, k1)
    conf = _conf(0.8, None, True)
    plain = NearestNeighborMatcher(**conf)(data)
    for kind, valid in (("F", [1, 0, 1, 0]), ("H", [0, 0, 1, 1])):
        mdl = model if kind == "F" else np.stack([gs.true_homography(g) for _ in range(4)])
        got = _guided(data, kind, mdl, valid=np.array(valid, np.uint8), **conf)
        for b in range(4):
            if not valid[b]:
                for k in KEYS:
                    assert torch.equal(got[k][b], plain[k][b]), (kind, b, k)
                assert torch.equal(got["matches"][b], plain["matches"][b])
                assert torch.equal(got["scores"][b], plain["scores"][b])
        # the guided pairs of the mixed batch match as they do alone
        for b in np.flatnonzero(valid):
            one = _guided(_data(d0[b:b + 1], d1[b:b + 1], k0[b:b + 1], k1[b:b + 1]), kind, mdl[b:b + 1], **conf)
            for k in KEYS:
                assert torch.equal(got[k][b], one[k][0]), (kind, b, k)
    far = _guided(data, "H", np.broadcast_to(np.eye(3), (4, 3, 3)), max_error=1e6, **conf)
    bool_valid = _guided(data, "F", model, valid=torch.zeros(4, dtype=torch.bool), **conf)
    for out in (far, bool_valid):
        for k in KEYS:
            assert torch.equal(out[k], plain[k]), k
        for b in range(4):
            assert torch.equal(out["matches"][b], plain["matches"][b])


def _decoy_scene(kind, seed, m=500, n_decoy=150, d=128, max_error=4.0):
    """A scene of `geometry_synth` with descriptors, and repeated structure: for n_decoy inlier rows, image 1 also
    holds a look-alike of the row's descriptor at a place the model rules out.  Returns the arrays and the decoyed
    rows with their true partners."""
    make = gs.planar if kind == "H" else gs.two_view
    k0, k1, m0, inl, model = make(m, 0.2, seed, unmatched=0.0)
    g = np.random.default_rng(seed + 1)
    d0 = g.normal(size=(m, d))
    d0 /= np.linalg.norm(d0, axis=1, keepdims=True)
    d1 = np.empty((m, d))
    d1[m0] = d0 + 0.3 * g.normal(size=(m, d)) / np.sqrt(d) * 4
    d1[m0[~inl]] = g.normal(size=((~inl).sum(), d))
    rows = g.choice(np.flatnonzero(inl), n_decoy, replace=False)
    dk = np.empty((n_decoy, 2), np.float32)
    for t, i in enumerate(rows):
        while True:  # a look-alike at least 5 max_error from the model's prediction
            cand = g.uniform([0, 0], [640, 480], (1, 2)).astype(np.float32)
            pts = np.concatenate([k0[i:i + 1], cand], axis=1)
            if geo.errors(KIND[kind], model.reshape(1, 9), pts)[0, 0] > (5 * max_error) ** 2:
                dk[t] = cand[0]
                break
    dd = d0[rows] + 0.3 * g.normal(size=(n_decoy, d)) / np.sqrt(d) * 4
    d1 = np.concatenate([d1, dd])
    d1 /= np.linalg.norm(d1, axis=1, keepdims=True)
    k1 = np.concatenate([k1, dk])
    return (d0[None].astype(np.float32), d1[None].astype(np.float32), k0[None], k1[None], model[None], rows,
            m0[rows])


@pytest.mark.parametrize("kind", ["H", "F"])
def test_repeated_structure_scenes_against_the_oracle(kind):
    conf = _conf(0.9, None, True)
    report = []
    for seed in (1, 2, 3):
        d0, d1, k0, k1, model, rows, partner = _decoy_scene(kind, seed)
        data = _data(d0, d1, k0, k1)
        plain = NearestNeighborMatcher(**conf)(data)
        got = _guided(data, kind, model, **conf)
        want, _ = _want(d0, d1, k0, k1, kind, model, **conf)
        excluded = rows_total = 0
        for side, key, skey in ((0, "matches0", "matching_scores0"), (1, "matches1", "matching_scores1")):
            ok = ngo.decided(want, 0, side, TOL_S, TOL_D, True)
            gm, gsc = got[key][0].cpu().numpy(), got[skey][0].cpu().numpy()
            np.testing.assert_array_equal(gm[ok], want[key][0][ok])
            both = ok & (gm >= 0)
            np.testing.assert_allclose(gsc[both], want[skey][0][both], rtol=0, atol=TOL_S)
            excluded += int((~ok).sum())
            rows_total += ok.size
        assert excluded < 0.01 * rows_total, (excluded, rows_total)
        hit_plain = int((plain["matches0"][0].cpu().numpy()[rows] == partner).sum())
        hit_guided = int((got["matches0"][0].cpu().numpy()[rows] == partner).sum())
        assert hit_guided >= hit_plain
        report.append((seed, len(rows), hit_plain, hit_guided))
    print(f"\n{kind}: decoyed rows matched to their true partner (seed, decoyed, unguided, guided): {report}")
    assert sum(r[3] for r in report) > sum(r[2] for r in report)


def test_ragged_batch_equals_single_pairs():
    g = np.random.default_rng(21)
    b, M, N = 6, 400, 380
    d0, d1 = _unit_pair(g, b, M, N, 128)
    k0, k1, model = _scene("H", g, b, M, N)
    lens0, lens1 = [400, 0, 17, 1, 250, 399], [380, 33, 0, 1, 379, 12]
    conf = _conf(0.95, None, True)
    got = _guided(_data(d0, d1, k0, k1, lens0, lens1), "H", model, max_error=60.0, **conf)
    for i in range(b):
        m, n = lens0[i], lens1[i]
        one = _guided(_data(d0[i:i + 1, :m], d1[i:i + 1, :n], k0[i:i + 1, :m], k1[i:i + 1, :n]), "H", model[i:i + 1],
                      max_error=60.0, **conf)
        assert torch.equal(got["matches0"][i, :m], one["matches0"][0]) and (got["matches0"][i, m:] == -1).all()
        assert torch.equal(got["matches1"][i, :n], one["matches1"][0]) and (got["matches1"][i, n:] == -1).all()
        assert torch.equal(got["matching_scores0"][i, :m], one["matching_scores0"][0])
        assert torch.equal(got["matches"][i], one["matches"][0])


@pytest.mark.parametrize("b, n, kind", [(32, 2048, "F"), (8, 8192, "H")])
def test_large_batches_run(b, n, kind):
    g = np.random.default_rng(n)
    d0, d1 = _unit_pair(g, b, n, n, 128, dup=0.5)
    k0, k1, model = _scene(kind, g, b, n, n)
    _place(kind, model, k0, k1, g, n // 2)
    data = _data(d0, d1, k0, k1)
    plain = NearestNeighborMatcher(ratio_thresh=0.9)(data)
    got = _guided(data, kind, model, ratio_thresh=0.9)
    kept, total = _monotone_and_gated(plain, got, kind, model, k0, k1)
    assert kept > 0.1 * b * n and total >= kept, (kept, total)


def _abi_guided(d0, d1, k0, k1, model, valid, out, ws, handle):
    lib = _cabi.load()
    b, m, d = d0.shape
    n = d1.shape[1]
    cfg = _cabi.NnConfig(_cabi.NN_ABI_VERSION, d, 1, 0.8, 0.0)
    ins = _cabi.NnInputs(b, m, n, d0.data_ptr(), d1.data_ptr(), None, None)
    guide = _cabi.NnGuide(_cabi.NN_GUIDE_F, model.data_ptr(), valid.data_ptr(), k0.data_ptr(), k1.data_ptr(), 8.0)
    outs = _cabi.NnOutputs(*(t.data_ptr() for t in out))
    stream = torch.cuda.current_stream().cuda_stream
    _cabi.check(lib.nn_match_guided(handle, C.byref(cfg), C.byref(ins), C.byref(guide), C.byref(outs), ws.data_ptr(),
                                    ws.numel(), stream), "nn_match_guided")


def test_repeats_and_cuda_graph_replay_are_bit_identical():
    g = np.random.default_rng(4)
    b, m, n = 16, 2600, 3000  # two groups of pairs
    d0, d1 = _unit_pair(g, b, m, n, 256)
    k0, k1, model = _scene("F", g, b, m, n)
    valid = np.ones(b, np.uint8)
    valid[::5] = 0
    data = _data(d0, d1, k0, k1)
    first = _guided(data, "F", model, valid=valid, max_error=8.0, ratio_thresh=0.8)
    for _ in range(2):
        again = _guided(data, "F", model, valid=valid, max_error=8.0, ratio_thresh=0.8)
        for k in KEYS:
            assert torch.equal(first[k], again[k]), k
    x0, x1 = data["image0"]["descriptors"], data["image1"]["descriptors"]
    p0, p1 = data["image0"]["keypoints"], data["image1"]["keypoints"]
    mdl = torch.as_tensor(model).cuda().reshape(b, 9).contiguous()
    vd = torch.as_tensor(valid).cuda()
    out = [torch.empty(b, m, dtype=torch.int64, device="cuda"), torch.empty(b, n, dtype=torch.int64, device="cuda"),
           torch.empty(b, m, device="cuda"), torch.empty(b, n, device="cuda"),
           torch.empty(b, dtype=torch.int32, device="cuda"), torch.empty(b, m, 2, dtype=torch.int64, device="cuda"),
           torch.empty(b, m, device="cuda")]
    lib = _cabi.load()
    ws = torch.empty(lib.nn_guided_workspace_bytes(b, m, n, 256), dtype=torch.uint8, device="cuda")
    handle = NearestNeighborMatcher._handle(x0.device)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        _abi_guided(x0, x1, p0, p1, mdl, vd, out, ws, handle)
    torch.cuda.current_stream().wait_stream(side)
    eager = [t.clone() for t in out]
    for t in out:
        t.fill_(7)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _abi_guided(x0, x1, p0, p1, mdl, vd, out, ws, handle)
    graph.replay()
    torch.cuda.synchronize()
    for a, c in zip(eager[:5], out[:5]):
        assert torch.equal(a, c)
    cnt = eager[4].tolist()  # the lists: only the first n_matches[b] rows are defined
    for i in range(b):
        assert torch.equal(eager[5][i, : cnt[i]], out[5][i, : cnt[i]])
        assert torch.equal(eager[6][i, : cnt[i]], out[6][i, : cnt[i]])
        assert torch.equal(eager[5][i, : cnt[i]], first["matches"][i])
    assert torch.equal(eager[0], first["matches0"]) and torch.equal(eager[3], first["matching_scores1"])


def test_sift_homography_lo_then_guided_matching_with_no_checkpoint():
    """Two 240x320 crops of one canvas, 64 px apart: SIFT, unguided matching, LO-RANSAC H, then guided matching under
    that H with the estimator's success as `valid`; every stage's output stays on the device."""
    off = 64
    canvas = sift_synth.make_image(240 + off, 320 + off, 1, 21)
    a_img = canvas[:, :, off:, off:].contiguous().cuda()
    b_img = canvas[:, :, :240, :320].contiguous().cuda()
    sift = SIFT(max_num_keypoints=100000, nms_radius=None)
    fa, fb = sift({"image": a_img}), sift({"image": b_img})
    nnm = NearestNeighborMatcher(ratio_thresh=0.8)
    plain = nnm({"image0": fa, "image1": fb})
    h = find_homography_lo(fa["keypoints"], fb["keypoints"], plain["matches0"])
    got = nnm({"image0": fa, "image1": fb}, H=h["H"], valid=h["success"], max_error=3.0)
    assert bool(h["success"][0])
    ka, kb = fa["keypoints"][0].cpu().numpy(), fb["keypoints"][0].cpu().numpy()
    Hm = h["H"].cpu().numpy()
    pm, gm = plain["matches0"].cpu().numpy(), got["matches0"].cpu().numpy()
    pts = lambda m0: np.concatenate([ka[m0 >= 0], kb[m0[m0 >= 0]]], 1).astype(np.float32)  # noqa: E731
    gate_p = np.zeros(pm.shape[1], bool)
    gate_p[pm[0] >= 0] = geo.errors(geo.HOMOGRAPHY, Hm.reshape(1, 9), pts(pm[0]))[0] < np.float32(9.0)
    assert (gm[0][gate_p] == pm[0][gate_p]).all()  # the guided set contains the gated unguided set
    assert (geo.errors(geo.HOMOGRAPHY, Hm.reshape(1, 9), pts(gm[0]))[0] < np.float32(9.0)).all()

    def near_truth(m0):
        i = np.flatnonzero(m0 >= 0)
        return int((np.abs(kb[m0[i]] - (ka[i] + off)).max(1) <= 3.0).sum())
    n_plain, n_guided = near_truth(pm[0]), near_truth(gm[0])
    print(f"\nSIFT pair: matches within 3 px of the true shift, unguided {n_plain}, guided {n_guided} "
          f"(of {int((pm[0] >= 0).sum())} / {int((gm[0] >= 0).sum())} matches)")
    assert n_guided >= n_plain > 50
