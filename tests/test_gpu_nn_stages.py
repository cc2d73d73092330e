"""The nearest-neighbour matcher stage by stage on the H100, at every slot, tile, chunk and group edge.

``nn_match`` / ``nn_match_guided`` are called through the C ABI on a workspace the test owns (filled with 0xff
first); ``nn_workspace_layout`` says where the last group of pairs left each stage's output.  Each stage is checked
from the captured output of the stage before it:

* pack: hi / lo bit for bit, zero padding rows, the length and stop words;
* sweep: every live row's (s1, s2, j1) of every slot with live columns, bit for bit on split-grid data
  (oracle/nn_cases.py), from float64 split products; a guided slot with no gated live column holds s1 = -inf;
* tail: jbest / sbest from the captured partials (oracle/nn_cases.tail);
* outputs: from the captured jbest / sbest, and every pair against the split oracle (nn_oracle.match_chunked, float64
  on the GPU) bit for bit, ``matches``, ``scores`` and ``n_matches`` included.

Every shape asserts the regime it exists for from the plan.  Unit descriptors at 8192 keypoints are compared with the
float64 dot product on the rows no perturbation below the calibrated gates of tests/test_nn_emulation.py can flip.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from lightglue_b200 import NearestNeighborMatcher, _cabi
from oracle import geometry_oracle as geo
from oracle import geometry_synth as gs
from oracle import nn_cases as nc
from oracle import nn_guided_oracle as ngo
from oracle import nn_oracle as nno
from tests.test_nn_emulation import TOL_D, TOL_S

pytestmark = pytest.mark.gpu

DEV = "cuda"
KEYS = ("matches0", "matches1", "matching_scores0", "matching_scores1")
NAMES = ("hi", "lo", "part", "parg", "jbest", "sbest", "len", "stop", "rec", "gate_on")
CONFS = ((None, None, True), (0.8, None, False), (0.95, 1.3, True), (0.7, None, True), (0.5, 0.9, False))
EDGES = (1, 127, 128, 129, 255, 256, 257, 1023, 1024, 1025, 2049, 4097)
INT_MAX = 2**31 - 1


def _layout(B, M, N, D, guided):
    off = (C.c_int64 * _cabi.NN_LAYOUT_BUFFERS)()
    size = (C.c_int64 * _cabi.NN_LAYOUT_BUFFERS)()
    plan = (C.c_int32 * 4)()
    total = _cabi.load().nn_workspace_layout(B, M, N, D, int(guided), off, size, plan)
    assert total > 0
    return dict(zip(NAMES, zip(off, size))), tuple(plan), total


def _call(d0, d1, lens0, lens1, ratio, dist, mutual, guide=None):
    """One nn_match / nn_match_guided call; returns the outputs (numpy), the workspace and its layout."""
    lib = _cabi.load()
    B, M, D = d0.shape
    N = d1.shape[1]
    bufs, plan, total = _layout(B, M, N, D, guide is not None)
    x0, x1 = torch.as_tensor(d0).to(DEV).contiguous(), torch.as_tensor(d1).to(DEV).contiguous()
    l0 = None if lens0 is None else torch.tensor(lens0, dtype=torch.int32, device=DEV)
    l1 = None if lens1 is None else torch.tensor(lens1, dtype=torch.int32, device=DEV)
    out = [torch.full((B, M), 7, dtype=torch.int64, device=DEV), torch.full((B, N), 7, dtype=torch.int64, device=DEV),
           torch.full((B, M), 7.0, device=DEV), torch.full((B, N), 7.0, device=DEV),
           torch.full((B,), 7, dtype=torch.int32, device=DEV), torch.full((B, M, 2), 7, dtype=torch.int64, device=DEV),
           torch.full((B, M), 7.0, device=DEV)]
    ws = torch.full((total,), 0xFF, dtype=torch.uint8, device=DEV)
    cfg = _cabi.NnConfig(_cabi.NN_ABI_VERSION, D, int(mutual), ratio or 0.0, dist or 0.0)
    ins = _cabi.NnInputs(B, M, N, x0.data_ptr(), x1.data_ptr(), None if l0 is None else l0.data_ptr(),
                         None if l1 is None else l1.data_ptr())
    outs = _cabi.NnOutputs(*(t.data_ptr() for t in out))
    handle = NearestNeighborMatcher._handle(torch.device(DEV, torch.cuda.current_device()))
    stream = torch.cuda.current_stream().cuda_stream
    if guide is None:
        rc = lib.nn_match(handle, C.byref(cfg), C.byref(ins), C.byref(outs), ws.data_ptr(), total, stream)
    else:
        kind, model, valid, k0, k1, px = guide
        mdl = torch.as_tensor(np.asarray(model, np.float64)).reshape(B, 9).to(DEV).contiguous()
        vd = None if valid is None else torch.as_tensor(np.asarray(valid, np.uint8)).to(DEV)
        p0, p1 = torch.as_tensor(k0).to(DEV).contiguous(), torch.as_tensor(k1).to(DEV).contiguous()
        g = _cabi.NnGuide(kind, mdl.data_ptr(), None if vd is None else vd.data_ptr(), p0.data_ptr(), p1.data_ptr(), px)
        rc = lib.nn_match_guided(handle, C.byref(cfg), C.byref(ins), C.byref(g), C.byref(outs), ws.data_ptr(), total,
                                 stream)
    _cabi.check(rc, "nn_match")
    torch.cuda.synchronize()
    o = [t.cpu().numpy() for t in out]
    got = dict(zip(KEYS, o[:4]))
    got["n_matches"], got["matches"], got["scores"] = o[4], o[5], o[6]
    return got, ws, bufs, plan


def _view(ws, bufs, name, dtype, shape):
    o, s = bufs[name]
    n = int(np.prod(shape))
    return ws[o:o + s].view(dtype)[:n].view(shape)


def _lens(lens, B, cap):
    return [cap] * B if lens is None else [min(max(int(v), 0), cap) for v in lens]


def _check(d0, d1, lens0=None, lens1=None, conf=(None, None, True), guide=None):
    """One call, every stage of its last group and every pair's outputs; returns (got, want, plan)."""
    ratio, dist, mutual = conf
    B, M, D = d0.shape
    N = d1.shape[1]
    got, ws, bufs, plan = _call(d0, d1, lens0, lens1, ratio, dist, mutual, guide)
    G, Lp, pstride, groups = plan
    gate = None
    if guide is not None:
        kind, model, valid, k0, k1, px = guide
        gate = ngo.chunk_gate(kind, model, k0, k1, px, valid, lens0, lens1, device=DEV)
    want = nno.match_chunked(d0, d1, lens0, lens1, ratio, dist, mutual, split=True, gate=gate, device=DEV)
    # every pair's outputs against the oracle
    for k in KEYS:
        np.testing.assert_array_equal(got[k], want[k], err_msg=k)
    for b in range(B):
        c = len(want["matches"][b])
        assert got["n_matches"][b] == c, b
        np.testing.assert_array_equal(got["matches"][b, :c], want["matches"][b])
        np.testing.assert_array_equal(got["scores"][b, :c], want["scores"][b])

    # the last group's stages
    b0 = (groups - 1) * G
    g = B - b0
    m_all, n_all = _lens(lens0, B, M), _lens(lens1, B, N)
    ln = _view(ws, bufs, "len", torch.int32, (2 * g,)).cpu().numpy()
    np.testing.assert_array_equal(ln, m_all[b0:] + n_all[b0:])
    assert (_view(ws, bufs, "stop", torch.int32, (g,)) == 0).all()
    # pack: the device's split of each live row, zero rows past the lengths
    X = torch.zeros(2 * g, Lp, D, device=DEV)
    for s in range(g):
        X[s, :m_all[b0 + s]] = torch.as_tensor(d0[b0 + s, :m_all[b0 + s]], device=DEV)
        X[g + s, :n_all[b0 + s]] = torch.as_tensor(d1[b0 + s, :n_all[b0 + s]], device=DEV)
    hi = X.bfloat16()
    lo = (X - hi.float()).bfloat16()
    for name, ref in (("hi", hi), ("lo", lo)):
        cap = _view(ws, bufs, name, torch.int16, (2 * g, Lp, D))
        assert torch.equal(cap, ref.view(torch.int16)), name
    del X, hi, lo
    # sweep, tail and outputs per pair of the group, from the stage before
    part = _view(ws, bufs, "part", torch.float32, (2 * g * Lp, pstride, 2))
    parg = _view(ws, bufs, "parg", torch.int32, (2 * g * Lp, pstride))
    jbest = _view(ws, bufs, "jbest", torch.int32, (2 * g * Lp,)).cpu().numpy()
    sbest = _view(ws, bufs, "sbest", torch.float32, (2 * g * Lp,)).cpu().numpy()
    r2, t2 = nno.thresholds(ratio, dist)
    for s in range(g):
        b = b0 + s
        m, n = m_all[b], n_all[b]
        x0 = torch.as_tensor(d0[b, :m], device=DEV)
        x1 = torch.as_tensor(d1[b, :n], device=DEV)
        tails = []
        for side, (rows, cols, seq) in enumerate(((m, n, s), (n, m, g + s))):
            r0 = seq * Lp
            nt = (cols + 127) // 128
            if rows and nt:
                A, Bm = (x0, x1) if side == 0 else (x1, x0)
                (ah, al), (bh, bl) = nno._split_t(A.float()), nno._split_t(Bm.float())
                for ra in range(0, rows, 4096):
                    rb = min(ra + 4096, rows)
                    Gm = gate(b, side, ra, rb) if gate is not None else None
                    S = ah[ra:rb] @ bh.T + ah[ra:rb] @ bl.T + al[ra:rb] @ bh.T
                    e1, e2, ej = nc.slot_partials(S, cols, Gm)
                    c1, c2 = part[r0 + ra:r0 + rb, :nt, 0], part[r0 + ra:r0 + rb, :nt, 1]
                    cj = parg[r0 + ra:r0 + rb, :nt]
                    assert torch.equal(c1, e1), (b, side, ra, "s1")
                    assert torch.equal(c2, e2), (b, side, ra, "s2")
                    assert torch.equal(cj, ej), (b, side, ra, "j1")
                    if Gm is not None:
                        assert torch.equal(c1 == -np.inf, cj == INT_MAX)  # a slot with no gated live column
                    del S, e1, e2, ej
                p = part[r0:r0 + rows, :nt].cpu().numpy()
                pa = parg[r0:r0 + rows, :nt].cpu().numpy()
            else:
                p, pa = np.zeros((rows, nt, 2), np.float32), np.zeros((rows, nt), np.int32)  # no rows or columns
            jb, sb = nc.tail(p, pa, cols, r2, t2)
            np.testing.assert_array_equal(jbest[r0:r0 + rows], jb, err_msg=f"jbest {b} {side}")
            np.testing.assert_array_equal(sbest[r0:r0 + rows], sb, err_msg=f"sbest {b} {side}")
            tails.append((jbest[r0:r0 + rows], sbest[r0:r0 + rows]))
        out = nc.outputs(*tails[0], *tails[1], M, N, mutual)
        for k in KEYS:
            np.testing.assert_array_equal(got[k][b], out[k], err_msg=f"{k} from the tail, pair {b}")
        assert got["n_matches"][b] == out["n_matches"]
        np.testing.assert_array_equal(got["matches"][b, :out["n_matches"]], out["matches"])
        np.testing.assert_array_equal(got["scores"][b, :out["n_matches"]], out["scores"])
    return got, want, plan


def _planted_ties_hold(want, planted, b):
    """Each planted tie is its row's maximum: j1 the lowest tied column and s2 = s1."""
    a = want["sides"][b][0]
    for row, cols in planted[b][0]:
        assert a["j1"][row] == cols[0] and a["s1"][row] == a["s2"][row], (row, cols)
    return len(planted[b][0])


# ------------------------------------------------------------------------------------------------------------ shapes
SHAPES = sorted({(m, m) for m in EDGES} | {(m, n) for m, n in zip(EDGES, reversed(EDGES))} |
                {(EDGES[i], EDGES[(i + 5) % 12]) for i in range(12)})


@pytest.mark.parametrize("m, n", SHAPES)
def test_every_stage_at_the_edges(m, n):
    i = SHAPES.index((m, n))
    D = (64, 128, 192, 256, 512)[i % 5]
    conf = CONFS[i % len(CONFS)]
    d0, d1, planted = nc.make_pair(100 + i, 1, m, n, D)
    got, want, (G, Lp, pstride, groups) = _check(d0, d1, conf=conf)
    assert (G, groups, Lp) == (1, 1, (max(m, n) + 127) // 128 * 128)
    _planted_ties_hold(want, planted, 0)
    if m > 1024 and conf[2]:  # matched rows on both sides of the tail's 1024-row scan chunks
        m0 = got["matches0"][0]
        assert (m0[:1024] >= 0).any() and (m0[1024:] >= 0).any()


@pytest.mark.parametrize("m, n", [(1, 40000), (40000, 1)])
def test_one_row_against_40000(m, n):
    d0, d1, _ = nc.make_pair(7, 1, m, n, 64)
    got, want, (G, Lp, _, groups) = _check(d0, d1, conf=(0.8, None, True))
    assert G == 1 and groups == 1 and Lp > _cabi.NN_GROUP_ROWS
    a, c = want["sides"][0]
    assert (c["s2"] == -np.inf).all() if m == 1 else (a["s2"] == -np.inf).all()  # one column: s2 = -inf
    assert (got["matches0"] >= 0).sum() <= 1


def test_more_row_tiles_than_sms_and_a_pair_wider_than_a_group():
    d0, d1, planted = nc.make_pair(8, 2, 33000, 20000, 64)
    got, want, (G, Lp, _, groups) = _check(d0, d1, conf=(None, None, True))
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert G == 1 and groups == 2 and Lp > _cabi.NN_GROUP_ROWS and 2 * G * Lp // 128 > sms
    assert _planted_ties_hold(want, planted, 1) == len(nc.TIES)
    assert (got["matches0"][1, 30000:] >= 0).any()


def _ragged17():
    lens0 = [3000] * 9 + [3000, 0, 2999, 1, 1500, 2049, 1025, 3000]
    lens1 = [3000] * 9 + [2500, 3000, 0, 1, 3000, 1024, 2049, 129]
    return lens0, lens1


@pytest.mark.parametrize("conf", [(None, None, True), (0.8, 1.3, False)])
def test_two_groups_of_a_ragged_batch(conf):
    lens0, lens1 = _ragged17()
    d0, d1, _ = nc.make_pair(17, 17, 3000, 3000, 128, lens0, lens1)
    got, _, (G, Lp, _, groups) = _check(d0, d1, lens0, lens1, conf=conf)
    assert (G, groups, Lp) == (9, 2, 3072)  # groups of 9 and 8
    assert (got["matches0"][10] == -1).all() and (got["matches1"][11] == -1).all()


@pytest.mark.parametrize("D", [64, 192, 512])
def test_descriptor_sizes_in_a_batch(D):
    """D = 64 is one K block, fewer than the sweep's ring stages."""
    d0, d1, _ = nc.make_pair(D, 3, 1100, 700, D, [1100, 129, 0], [700, 700, 5])
    _check(d0, d1, [1100, 129, 0], [700, 700, 5], conf=(0.9, None, True))


def test_without_the_mutual_check_several_rows_name_one_j():
    d0, d1, planted = nc.make_pair(12, 1, 1100, 600, 128)
    got, _, _ = _check(d0, d1, conf=(None, None, False))
    m0 = got["matches0"][0]
    for rows in planted[0][1]:
        assert len({int(m0[r]) for r in rows}) == 1 and m0[rows[0]] >= 0, rows
    assert len(np.unique(m0[m0 >= 0])) < (m0 >= 0).sum()


@pytest.mark.parametrize("ratio", [0.5, 0.7, 0.95])
def test_ratio_boundaries(ratio):
    """The fp32 product keeps the row at the boundary (a float64 product would not at 0.7 and 0.95)."""
    e0, e1, _ = nc.ratio_pair(ratio)
    d0 = np.concatenate([e0, e0]).astype(np.float32)
    d1 = np.concatenate([e1, e1[:, ::-1]]).astype(np.float32)
    got, _, _ = _check(d0, d1, conf=(ratio, None, False))
    assert got["matches0"][:, 0].tolist() == [0, 1]
    got, _, _ = _check(d0, d1, conf=(ratio * 0.999, None, False))
    assert got["matches0"][:, 0].tolist() == [-1, -1]


def test_distance_boundary():
    e0, e1, _ = nc.ratio_pair(0.5)  # s1 = 0.875: D1 = 0.25 = 0.5^2
    got, _, _ = _check(e0, e1, conf=(None, 0.5, True))
    assert got["matches0"][0].tolist() == [0]
    got, _, _ = _check(e0, e1, conf=(None, 0.4999, True))
    assert got["matches0"][0].tolist() == [-1]


# ----------------------------------------------------------------------------------------------------------- guided
def _scene(kind, g, B, M, N, hit=0.5):
    k0 = g.uniform([0, 0], [640, 480], (B, M, 2)).astype(np.float32)
    k1 = g.uniform([0, 0], [640, 480], (B, N, 2)).astype(np.float32)
    if kind == geo.HOMOGRAPHY:
        model = np.stack([gs.true_homography(g) for _ in range(B)])
    else:
        model = np.stack([gs.two_view(8, 0.0, int(s))[4] for s in g.integers(0, 1000, B)])
    if M > 7:
        k0[:, 7] = np.nan  # a non-finite keypoint fails every gate
    return k0, k1, model


@pytest.mark.parametrize("kind", [geo.HOMOGRAPHY, geo.FUNDAMENTAL])
@pytest.mark.parametrize("m, n", [(129, 1025), (2049, 257), (1, 4097)])
def test_guided_stages(kind, m, n):
    g = np.random.default_rng(m + n + kind)
    d0, d1, _ = nc.make_pair(m + kind, 1, m, n, 128)
    k0, k1, model = _scene(kind, g, 1, m, n)
    px = 60.0 if kind == geo.HOMOGRAPHY else 24.0
    got, want, _ = _check(d0, d1, conf=(0.9, None, True), guide=(kind, model, None, k0, k1, px))
    if m > 7:
        assert got["matches0"][0, 7] == -1


@pytest.mark.parametrize("kind", [geo.HOMOGRAPHY, geo.FUNDAMENTAL])
def test_guided_two_groups_with_ungated_pairs(kind):
    lens0, lens1 = _ragged17()
    g = np.random.default_rng(5 + kind)
    d0, d1, _ = nc.make_pair(40 + kind, 17, 3000, 3000, 128, lens0, lens1)
    k0, k1, model = _scene(kind, g, 17, 3000, 3000)
    valid = np.ones(17, np.uint8)
    valid[[9, 12, 16]] = 0
    px = 60.0 if kind == geo.HOMOGRAPHY else 24.0
    _, _, (G, _, _, groups) = _check(d0, d1, lens0, lens1, conf=(0.8, None, True),
                                     guide=(kind, model, valid, k0, k1, px))
    assert (G, groups) == (9, 2)


def test_guided_pair_wider_than_a_group():
    g = np.random.default_rng(3)
    d0, d1, _ = nc.make_pair(33, 1, 33000, 2000, 64)
    k0, k1, model = _scene(geo.FUNDAMENTAL, g, 1, 33000, 2000)
    _, _, (G, Lp, _, _) = _check(d0, d1, conf=(None, None, True), guide=(geo.FUNDAMENTAL, model, None, k0, k1, 24.0))
    assert G == 1 and Lp > _cabi.NN_GROUP_ROWS


@pytest.mark.parametrize("mutual", [True, False])
def test_guided_gate_boundary_and_nan(mutual):
    """Identity H, max_error = 1: a column exactly at t2 fails, a NaN keypoint gates out every column, a row with one
    gated column has s2 = -inf."""
    d = 64

    def e(i, x=1.0):
        v = np.zeros(d, np.float32)
        v[i] = x
        return v
    d0 = np.stack([e(0), e(1), e(2), e(3), e(4)])[None]
    d1 = np.stack([e(0), e(0, 0.875), e(1, 0.75), e(1, 0.75), e(2, 0.5), e(2, 0.9375), e(3), e(4)])[None]
    k0 = np.array([[[10, 10], [100, 100], [200, 200], [300, 300], [np.nan, 5]]], np.float32)
    k1 = np.array([[[11, 10], [10, 10.5], [100, 100], [100.5, 100], [200, 200], [250, 200], [310, 300], [0, 5]]],
                  np.float32)
    got, want, _ = _check(d0, d1, conf=(0.5, None, mutual), guide=(geo.HOMOGRAPHY, np.eye(3)[None], None, k0, k1, 1.0))
    assert got["matches0"][0].tolist() == [1, -1, 4, -1, -1]
    assert want["sides"][0][0]["s2"][2] == -np.inf and want["sides"][0][0]["j1"][4] == -1


# ------------------------------------------------------------------------------------------------- real descriptors
def _unit_pair(g, B, m, n, d):
    x0 = g.normal(size=(B, m, d))
    x1 = g.normal(size=(B, n, d))
    k = min(m, n) // 2
    x1[:, :k] = x0[:, :k] + 0.4 * g.normal(size=(B, k, d))
    x0 /= np.linalg.norm(x0, axis=-1, keepdims=True)
    x1 /= np.linalg.norm(x1, axis=-1, keepdims=True)
    return x0.astype(np.float32), x1.astype(np.float32)


@pytest.mark.parametrize("B, D", [(4, 128), (4, 256), (9, 128)])
def test_unit_descriptors_within_the_calibrated_gates(B, D):
    g = np.random.default_rng(B * D)
    d0, d1 = _unit_pair(g, B, 8192, 8192, D)
    conf = (0.8, None, True)
    got, ws, bufs, (G, Lp, _, groups) = _call(d0, d1, None, None, *conf)
    assert groups == (1 if B == 4 else 3)
    want = nno.match_chunked(d0, d1, None, None, *conf, device=DEV)
    excluded = rows = 0
    for side, key, skey in ((0, "matches0", "matching_scores0"), (1, "matches1", "matching_scores1")):
        for b in range(B):
            ok = nno.decided(want, b, side, TOL_S, TOL_D, True)
            rows += ok.size
            excluded += int((~ok).sum())
            np.testing.assert_array_equal(got[key][b][ok], want[key][b][ok])
            both = ok & (got[key][b] >= 0)
            np.testing.assert_allclose(got[skey][b][both], want[skey][b][both], rtol=0, atol=TOL_S)
    assert excluded < 0.01 * rows and (got["matches0"] >= 0).sum() > 0.3 * B * 8192, (excluded, rows)
    # the worst deviation of the device's s1 from float64 on the last group's decided rows
    b0 = (groups - 1) * G
    sb = _view(ws, bufs, "sbest", torch.float32, (2 * (B - b0) * Lp,)).cpu().numpy()
    worst = 0.0
    for s in range(B - b0):
        for side, seq in ((0, s), (1, B - b0 + s)):
            o = want["sides"][b0 + s][side]
            ok = nno.decided(want, b0 + s, side, TOL_S, TOL_D, True)
            dev = np.abs(sb[seq * Lp:seq * Lp + 8192].astype(np.float64) - o["s1"])[ok]
            worst = max(worst, float(dev.max()))
    print(f"\nB = {B}, D = {D}: worst |s1 - float64| on decided rows {worst:.2e} (gate {TOL_S:g})")
    assert worst <= TOL_S


def test_pack_of_arbitrary_values():
    """hi / lo of unit rows, +-0, bf16 rounding ties, large and tiny values; zero rows past the lengths; the length
    words clamped.  Only the pack is checked: such rows overflow the similarities."""
    g = np.random.default_rng(1)
    B, M, N, D = 2, 300, 130, 128
    d0 = g.normal(size=(B, M, D))
    d0 /= np.linalg.norm(d0, axis=-1, keepdims=True)
    d1 = g.normal(size=(B, N, D)) * 10.0 ** g.integers(-35, 35, (B, N, D))
    d0[:, 0] = 0.0
    d0[:, 1] = -0.0
    d0[:, 2, :4] = (1 + 2.0 ** -8, 1 + 3 * 2.0 ** -8, -(1 + 2.0 ** -8), 2.0 ** -8 + 2.0 ** -17)  # ties, and just above
    d1[:, 3, :3] = (3e38, -1e-38 * 3, 1e30)
    d0, d1 = d0.astype(np.float32), d1.astype(np.float32)
    lens0, lens1 = [300, 5], [131, -2]
    got, ws, bufs, (G, Lp, _, groups) = _call(d0, d1, lens0, lens1, None, None, True)
    assert (G, groups) == (2, 1)
    m, n = [300, 5], [130, 0]
    np.testing.assert_array_equal(_view(ws, bufs, "len", torch.int32, (4,)).cpu().numpy(), m + n)
    assert (_view(ws, bufs, "stop", torch.int32, (2,)) == 0).all()
    X = torch.zeros(4, Lp, D, device=DEV)
    for s in range(2):
        X[s, :m[s]] = torch.as_tensor(d0[s, :m[s]], device=DEV)
        X[2 + s, :n[s]] = torch.as_tensor(d1[s, :n[s]], device=DEV)
    hi = X.bfloat16()
    lo = (X - hi.float()).bfloat16()
    assert hi[0, 2, :4].tolist() == [1.0, 1 + 4 * 2.0 ** -8, -1.0, 2.0 ** -8]  # ties to even
    assert torch.signbit(hi[0, 1]).all() and not torch.signbit(lo[0, 1]).any()
    for name, ref in (("hi", hi), ("lo", lo)):
        assert torch.equal(_view(ws, bufs, name, torch.int16, (4, Lp, D)), ref.view(torch.int16)), name
