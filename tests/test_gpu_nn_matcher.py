"""The nearest-neighbour matcher on the H100 against oracle/nn_oracle.py: bit for bit where every product and sum is
exact, within the split-bf16 bound on synthetic pairs, batch against single pairs, repeats and CUDA-graph replay, and
SIFT -> NearestNeighborMatcher -> find_homography on two crops of one image with no checkpoint."""
import ctypes as C

import numpy as np
import pytest
import torch

from lightglue_b200 import SIFT, NearestNeighborMatcher, _cabi, synth
from lightglue_b200.geometry import find_homography
from lightglue_b200.ragged import match_ragged
from oracle import nn_oracle as nno
from oracle import sift_synth
from tests.test_nn_emulation import TOL_D, TOL_S  # the split-bf16 gates, calibrated by emulation

pytestmark = pytest.mark.gpu

KEYS = ("matches0", "matches1", "matching_scores0", "matching_scores1")


def _run(d0, d1, lens0=None, lens1=None, **conf):
    data = {"image0": {"descriptors": d0.cuda()}, "image1": {"descriptors": d1.cuda()}}
    if lens0 is not None:
        data["image0"]["num_keypoints"] = torch.tensor(lens0, dtype=torch.int32).cuda()
        data["image1"]["num_keypoints"] = torch.tensor(lens1, dtype=torch.int32).cuda()
    return NearestNeighborMatcher(**conf)(data)


def _conf(ratio, dist, mutual):
    return {"ratio_thresh": ratio, "distance_thresh": dist, "mutual_check": mutual}


def _grid_pair(seed, b, m, n, d):
    """Entries k / 16 with |k| <= 2: bf16 holds them exactly (lo = 0), every product is a multiple of 2^-8 and every sum
    of D <= 512 of them is exact in fp32.  The coarse grid makes many exact ties."""
    g = np.random.default_rng(seed)
    return (torch.from_numpy(g.integers(-2, 3, (b, m, d)) / 16).float(),
            torch.from_numpy(g.integers(-2, 3, (b, n, d)) / 16).float())


def _planted(d=128):
    """Rows that sit on the boundaries with r = 0.5 and t = 0.5, and duplicated descriptors (the lowest j wins)."""
    def e(*iv):
        v = torch.zeros(d)
        for i, x in iv:
            v[i] = x
        return v
    d0 = torch.stack([e((0, 1.0)), e((1, 1.0)), e((2, 1.0)), e((3, 1.0)), e((4, 1.0)), e((5, -1.0))])
    d1 = torch.stack([
        e((0, 0.875)), e((0, 0.5)),      # row 0: D1 = 0.25 = 0.5^2 D2 (ratio boundary) and D1 = 0.5^2 (distance boundary)
        e((1, 0.875)), e((1, 0.5625)),   # row 1: D1 = 0.25 > 0.25 * 0.875
        e((2, 0.8125)),                  # row 2: D1 = 0.375 > 0.5^2
        e((3, 0.75)), e((3, 0.75)),      # row 3: an exact tie: j = 5 (s1 = s2)
        e((4, 1.0)), e((4, 1.0)), e((4, 1.0)),
    ])
    return d0[None], d1[None]


def _check_exact(d0, d1, lens0=None, lens1=None, **conf):
    got = _run(d0, d1, lens0, lens1, **conf)
    want = nno.match(d0.double().numpy(), d1.double().numpy(), lens0, lens1, conf.get("ratio_thresh"),
                     conf.get("distance_thresh"), conf.get("mutual_check", True))
    for k in KEYS:
        np.testing.assert_array_equal(got[k].cpu().numpy(), want[k], err_msg=k)
    for b in range(d0.shape[0]):
        np.testing.assert_array_equal(got["matches"][b].cpu().numpy(), want["matches"][b])
        np.testing.assert_array_equal(got["scores"][b].cpu().numpy(), want["scores"][b])
    return got


@pytest.mark.parametrize("ratio", [None, 0.5, 0.8])
@pytest.mark.parametrize("dist", [None, 0.5, 1.3])
@pytest.mark.parametrize("mutual", [True, False])
def test_exact_arithmetic_equals_the_oracle_bit_for_bit(ratio, dist, mutual):
    d0, d1 = _grid_pair(3, 3, 300, 260, 64)
    _check_exact(d0, d1, **_conf(ratio, dist, mutual))


@pytest.mark.parametrize("d", [64, 128, 256, 512])
def test_exact_arithmetic_at_every_descriptor_size(d):
    d0, d1 = _grid_pair(d, 2, 130, 400, d)
    _check_exact(d0, d1, **_conf(0.9, None, True))


@pytest.mark.parametrize("mutual", [True, False])
def test_exact_boundaries_and_duplicates(mutual):
    d0, d1 = _planted()
    for ratio, dist in ((0.5, None), (None, 0.5), (0.5, 0.5), (None, None)):
        got = _check_exact(d0, d1, **_conf(ratio, dist, mutual))
        m0 = got["matches0"][0].tolist()
        assert m0[3] == (5 if ratio is None and dist is None else -1)  # a tie: the lower j, and s1 = s2 fails r < 1
        assert m0[4] == 7  # three equal descriptors: the lowest index (D1 = D2 = 0 passes both tests)
    got = _check_exact(d0, d1, **_conf(0.5, None, False))
    assert got["matches0"][0].tolist()[:3] == [0, -1, 4]  # the ratio boundary is kept, 0.5625 fails
    got = _check_exact(d0, d1, **_conf(None, 0.5, False))
    assert got["matches0"][0].tolist()[:3] == [0, 2, -1]  # the distance boundary is kept, D1 = 0.375 fails


@pytest.mark.parametrize("d", [256, 128])
@pytest.mark.parametrize("ratio", [None, 0.8])
@pytest.mark.parametrize("dist", [None, 0.7])
@pytest.mark.parametrize("mutual", [True, False])
def test_synthetic_pairs_within_the_split_bf16_bound(d, ratio, dist, mutual):
    data, _ = synth.make_pair(700, d=d, b=4, m=900, seed=40 + d)
    d0, d1 = data["image0"]["descriptors"], data["image1"]["descriptors"]
    got = _run(d0, d1, **_conf(ratio, dist, mutual))
    want = nno.match(d0.double().numpy(), d1.double().numpy(), None, None, ratio, dist, mutual)
    rows = excluded = 0
    for side, key, skey in ((0, "matches0", "matching_scores0"), (1, "matches1", "matching_scores1")):
        g_m, g_s = got[key].cpu().numpy(), got[skey].cpu().numpy()
        for b in range(4):
            ok = nno.decided(want, b, side, TOL_S, TOL_D, mutual)
            rows += ok.size
            excluded += int((~ok).sum())
            np.testing.assert_array_equal(g_m[b][ok], want[key][b][ok])
            both = ok & (g_m[b] >= 0)
            np.testing.assert_allclose(g_s[b][both], want[skey][b][both], rtol=0, atol=1e-4)
    assert excluded < 0.01 * rows, (excluded, rows)
    assert (got["matches0"] >= 0).sum() > 1000


def test_ragged_batch_equals_single_pairs():
    g = torch.Generator().manual_seed(5)
    sizes = [(0, 5), (5, 0), (1, 1), (1, 40), (40, 1), (0, 0)] + [(int(a), int(b)) for a, b in
                                                                  torch.randint(2, 700, (26, 2), generator=g)]
    pairs = []
    for i, (m, n) in enumerate(sizes):
        data, _ = synth.make_pair(max(n, 1), d=128, m=max(m, 1), seed=100 + i)
        f0 = {k: data["image0"][k][:, :m].cuda() for k in ("keypoints", "descriptors")}
        f1 = {k: data["image1"][k][:, :n].cuda() for k in ("keypoints", "descriptors")}
        pairs.append({"image0": f0, "image1": f1})
    assert len(pairs) == 32
    nnm = NearestNeighborMatcher(ratio_thresh=0.9)
    batch = match_ragged(nnm, pairs)
    for p, r in zip(pairs, batch):
        one = nnm(p)
        for k in KEYS + ("matches", "scores"):
            a, b = r[k], one[k]
            if isinstance(a, list):
                a, b = a[0], b[0]
            assert torch.equal(a, b), k


def _abi_call(d0, d1, conf, out, ws, handle):
    lib = _cabi.load()
    b, m, d = d0.shape
    n = d1.shape[1]
    cfg = _cabi.NnConfig(_cabi.NN_ABI_VERSION, d, int(conf["mutual_check"]), conf["ratio_thresh"] or 0.0,
                         conf["distance_thresh"] or 0.0)
    ins = _cabi.NnInputs(b, m, n, d0.data_ptr(), d1.data_ptr(), None, None)
    outs = _cabi.NnOutputs(*(t.data_ptr() for t in out))
    stream = torch.cuda.current_stream().cuda_stream
    _cabi.check(lib.nn_match(handle, C.byref(cfg), C.byref(ins), C.byref(outs), ws.data_ptr(), ws.numel(), stream),
                "nn_match")


def test_repeats_and_cuda_graph_replay_are_bit_identical():
    data, _ = synth.make_pair(3000, d=256, b=16, m=2600, seed=7)  # two groups of pairs
    d0, d1 = data["image0"]["descriptors"].cuda(), data["image1"]["descriptors"].cuda()
    conf = _conf(0.8, None, True)
    nnm = NearestNeighborMatcher(**conf)
    first = nnm({"image0": {"descriptors": d0}, "image1": {"descriptors": d1}})
    for _ in range(3):
        again = nnm({"image0": {"descriptors": d0}, "image1": {"descriptors": d1}})
        for k in KEYS:
            assert torch.equal(first[k], again[k]), k
    b, m, n = 16, 2600, 3000
    out = [torch.empty(b, m, dtype=torch.int64, device="cuda"), torch.empty(b, n, dtype=torch.int64, device="cuda"),
           torch.empty(b, m, device="cuda"), torch.empty(b, n, device="cuda"),
           torch.empty(b, dtype=torch.int32, device="cuda"), torch.empty(b, m, 2, dtype=torch.int64, device="cuda"),
           torch.empty(b, m, device="cuda")]
    lib = _cabi.load()
    ws = torch.empty(lib.nn_workspace_bytes(b, m, n, 256), dtype=torch.uint8, device="cuda")
    handle = NearestNeighborMatcher._handle(d0.device)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        _abi_call(d0, d1, conf, out, ws, handle)
    torch.cuda.current_stream().wait_stream(side)
    eager = [t.clone() for t in out]
    for t in out:
        t.fill_(7)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _abi_call(d0, d1, conf, out, ws, handle)
    graph.replay()
    torch.cuda.synchronize()
    for a, c in zip(eager, out):
        assert torch.equal(a, c)
    assert torch.equal(eager[0], first["matches0"]) and torch.equal(eager[2], first["matching_scores0"])
    cnt = eager[4].tolist()
    for i in range(b):
        assert torch.equal(eager[5][i, : cnt[i]], first["matches"][i])


def test_sift_to_homography_with_no_checkpoint():
    """Two 240x320 crops of one canvas, 64 px apart on each axis: a whole number of pixels at every octave of SIFT's
    pyramid (8 octaves at 240x320, the deepest with a 64 px step), so interior keypoints shift exactly."""
    off = 64
    canvas = sift_synth.make_image(240 + off, 320 + off, 1, 21)
    a_img = canvas[:, :, off:, off:].contiguous().cuda()  # a's pixel p is b's pixel p + off
    b_img = canvas[:, :, :240, :320].contiguous().cuda()
    sift = SIFT(max_num_keypoints=100000, nms_radius=None)
    fa, fb = sift({"image": a_img}), sift({"image": b_img})
    out = NearestNeighborMatcher(ratio_thresh=0.8)({"image0": fa, "image1": fb})
    h = find_homography(fa["keypoints"], fb["keypoints"], out["matches0"])  # matches0 stays on the device
    ka, kb = fa["keypoints"][0].cpu(), fb["keypoints"][0].cpu()
    da, db = fa["descriptors"][0].cpu(), fb["descriptors"][0].cpu()
    m0 = out["matches0"][0].cpu()
    shared = hit = 0
    for i in range(ka.shape[0]):
        near = torch.nonzero((kb - (ka[i] + off)).abs().max(dim=1).values <= 1e-3).flatten()
        twins = [int(k) for k in near if (db[k] - da[i]).abs().max() <= 1e-6]
        if not twins:
            continue
        shared += 1
        hit += int(m0[i]) in twins
    assert shared >= 50, shared
    assert hit >= 0.95 * shared, (hit, shared)
    assert bool(h["success"][0])
    H = h["H"][0].cpu()
    corners = torch.tensor([[0.0, 0.0, 1.0], [320.0, 0.0, 1.0], [0.0, 240.0, 1.0], [320.0, 240.0, 1.0]], dtype=torch.float64)
    proj = corners @ H.T
    proj = proj[:, :2] / proj[:, 2:]
    inl = h["inliers"][0].cpu()
    err = (kb[m0[inl].clamp(min=0)] - ka[inl] - off).abs().max(dim=1).values
    stats = (int(inl.sum()), int((err <= 1e-3).sum()), float(err.max()))  # inliers, exactly shifted ones, worst error
    assert (proj - (corners[:, :2] + off)).abs().max() <= 0.05, (proj, stats)
