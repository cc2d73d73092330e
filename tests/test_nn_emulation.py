"""The nearest-neighbour matcher's gates and oracles without a GPU.

* The split-bf16 tolerance: the sweep's arithmetic emulated on the synthetic pairs of the tolerance tests (exact split
  products, fp32 accumulation in oracle/nn_cases.emulate's order) sets ``TOL_S`` / ``TOL_D`` at >= 3x its error and
  <= 1/3 of each lost pass's deviation.  tests/test_gpu_nn_matcher.py, test_gpu_nn_guided.py and test_gpu_nn_stages.py
  import them.
* The split grid (oracle/nn_cases.py) is exact in every pass, and the oracle's outputs on it move under each defect the
  bit-exact GPU tests exist to catch.
* The oracle follows the header's fp32 ratio product; the chunked torch oracle and gate equal the readable ones.
* ``nn_workspace_layout`` and the stage restatements of oracle/nn_cases.py against the oracle.
"""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from lightglue_b200 import _cabi, synth
from oracle import geometry_oracle as geo
from oracle import geometry_synth as gs
from oracle import nn_cases as nc
from oracle import nn_guided_oracle as ngo
from oracle import nn_oracle as nno

# Gates of the split-bf16 path against the float64 dot product on unit descriptors: s within TOL_S, D = 2 (1 - s)
# within TOL_D.  Emulated error <= 2.3e-6 (D = 128, 256); a lost hi lo or lo hi pass moves s by >= 4.9e-4.
TOL_S, TOL_D = 1e-4, 2e-4
LOST_PASSES = {"lost hi.lo": ("hh", "lh"), "lost lo.hi": ("hh", "hl")}


def _synthetic(d):
    """The pairs of test_gpu_nn_matcher.py::test_synthetic_pairs_within_the_split_bf16_bound."""
    data, _ = synth.make_pair(700, d=d, b=4, m=900, seed=40 + d)
    return data["image0"]["descriptors"].numpy(), data["image1"]["descriptors"].numpy()


@pytest.mark.parametrize("d", [128, 256])
def test_tolerance_is_three_times_the_emulated_error_and_a_third_of_each_lost_pass(d):
    d0, d1 = _synthetic(d)
    err, lost = 0.0, {k: np.inf for k in LOST_PASSES}
    for b in range(d0.shape[0]):
        exact = torch.as_tensor(d0[b].astype(np.float64) @ d1[b].astype(np.float64).T)
        err = max(err, float((nc.emulate(d0[b], d1[b]) - exact).abs().max()))
        for name, passes in LOST_PASSES.items():
            lost[name] = min(lost[name], float((nc.emulate(d0[b], d1[b], passes) - exact).abs().max()))
    print(f"\nD = {d}: emulated error {err:.2e}, lost passes {lost}")
    assert 3 * err <= TOL_S and 3 * 2 * err <= TOL_D, err
    for name, dev in lost.items():
        assert dev >= 3 * TOL_S and 2 * dev >= 3 * TOL_D, (name, dev)


# ------------------------------------------------------------------------------------------------------- split grid
def test_split_grid_splits_exactly_into_a_grid_hi_and_a_one_bit_lo():
    g = np.random.default_rng(0)
    x = nc.split_grid(g, (64, 512))
    hi, lo = nno.split(x)
    np.testing.assert_array_equal(hi * 16, np.round(hi * 16))  # hi on the k / 16 grid, |k| <= 2
    assert np.abs(hi).max() == 2 / 16
    np.testing.assert_array_equal(x.astype(np.float64) - hi, lo)  # d - hi = lo exactly
    nz = hi != 0
    assert (lo[~nz] == 0).all() and (lo[nz] != 0).all()
    np.testing.assert_array_equal(np.abs(lo[nz]), np.abs(hi[nz]) * 2.0 ** -10)  # one bit, below half an ulp
    assert (lo[nz] > 0).any() and (lo[nz] < 0).any()


@pytest.mark.parametrize("d", [64, 512])
def test_split_grid_products_and_partial_sums_fit_22_bits(d):
    """Every product of the three passes is a multiple of 2^-18, and the sum of their magnitudes along a row is below
    2^4: every partial sum in any order holds in 22 significant bits, so fp32 sums them exactly."""
    g = np.random.default_rng(d)
    a, b = nc.split_grid(g, (40, d)), nc.split_grid(g, (50, d))
    (ah, al), (bh, bl) = nno.split(a), nno.split(b)
    terms = [ah[:, None] * bh[None], ah[:, None] * bl[None], al[:, None] * bh[None]]
    for t in terms:
        q = t * 2.0 ** 18
        np.testing.assert_array_equal(q, np.round(q))
    total = sum(np.abs(t).sum(-1) for t in terms)
    assert total.max() < 16.0
    # the worst case over the whole grid: D (2^-6 + 2 2^-3 2^-13) < 16
    assert d * (2.0 ** -6 + 2 * 2.0 ** -16) < 16.0
    # and the sum is what fp32 makes of it: a sequential fp32 sum equals the float64 one
    s64 = nno.similarity(a.astype(np.float64), b.astype(np.float64), True)
    acc = np.zeros((40, 50), np.float32)
    for t in terms:
        for k in range(d):
            acc = (acc + t[..., k].astype(np.float32)).astype(np.float32)
    np.testing.assert_array_equal(acc.astype(np.float64), s64)


def _defect_match(d0, d1, ratio=None, dist=None, mutual=True, passes=nc.PASSES, f64_product=False, last_tie=False):
    """nno.match(split=True) with one defect: other products in s, the ratio product in float64, or the last index
    among the maxima."""
    hi0, lo0 = nno.split(d0)
    hi1, lo1 = nno.split(d1)
    P = {"hh": (hi0, hi1), "hl": (hi0, lo1), "lh": (lo0, hi1), "ll": (lo0, lo1)}
    S = sum(np.einsum("bmd,bnd->bmn", *P[p]) for p in passes)
    r2, t2 = nno.thresholds(ratio, dist)
    out = []
    for b in range(S.shape[0]):
        res = []
        for M in (S[b], S[b].T):
            j1 = M.shape[1] - 1 - np.argmax(M[:, ::-1], 1) if last_tie else np.argmax(M, 1)
            s1 = M[np.arange(len(M)), j1]
            s2 = np.where(np.eye(M.shape[1], dtype=bool)[j1], -np.inf, M).max(1)
            d1_, d2_ = 2 * (1 - s1), 2 * (1 - s2)
            keep = np.ones(len(M), bool)
            if r2 is not None:
                keep &= (d1_ <= r2 * d2_) if f64_product else (d1_.astype(np.float32) <= np.float32(r2) * d2_.astype(np.float32))
            if t2 is not None:
                keep &= d1_.astype(np.float32) <= np.float32(t2)
            res.append((np.where(keep, j1, -1), s1))
        (a, sa), (c, sc) = res
        if mutual:
            a, c = (np.where((a >= 0) & (c[np.clip(a, 0, None)] == np.arange(len(a))), a, -1),
                    np.where((c >= 0) & (a[np.clip(c, 0, None)] == np.arange(len(c))), c, -1))
        out.append((a, c, sa, sc))
    return out


def test_oracle_outputs_move_under_every_defect():
    """On split-grid pairs with planted ties, the split oracle's (matches, s1) differ from each defect's."""
    d0, d1, planted = nc.make_pair(3, 2, 300, 400, 128)
    assert all(len(p[0]) >= 6 for p in planted)
    base = _defect_match(d0, d1)
    want = nno.match(d0, d1, split=True)
    for b, (a, c, sa, _) in enumerate(base):  # the restatement is the oracle
        np.testing.assert_array_equal(a, want["matches0"][b])
        np.testing.assert_array_equal(sa, want["sides"][b][0]["s1"])

    def moved(other):
        return any(not np.array_equal(x, y) for o, t in zip(other, base) for x, y in zip(o, t))
    for name, passes in (("lost hi.lo", ("hh", "lh")), ("lost lo.hi", ("hh", "hl")),
                         ("lo.lo added", ("hh", "hl", "lh", "ll")), ("hi only", ("hh",))):
        assert moved(_defect_match(d0, d1, passes=passes)), name
    tie = _defect_match(d0, d1, mutual=False, last_tie=True)
    ok = _defect_match(d0, d1, mutual=False)
    for row, cols in planted[0][0]:
        assert ok[0][0][row] == cols[0] and tie[0][0][row] == cols[-1], (row, cols)
    for ratio in (0.7, 0.95):
        e0, e1, _ = nc.ratio_pair(ratio)
        assert _defect_match(e0, e1, ratio=ratio, mutual=False)[0][0].tolist() == [0]
        assert _defect_match(e0, e1, ratio=ratio, mutual=False, f64_product=True)[0][0].tolist() == [-1]


@pytest.mark.parametrize("ratio", [0.5, 0.7, 0.95])
def test_the_ratio_boundary_is_kept_with_the_fp32_product(ratio):
    d0, d1, (k1, k2) = nc.ratio_pair(ratio)
    res = nno.match(d0, d1, ratio_thresh=ratio, mutual_check=False)
    assert res["matches0"][0].tolist() == [0]
    a = res["sides"][0][0]
    assert a["s1"][0] == k1 / 256 and a["s2"][0] == k2 / 256
    r2, _ = nno.thresholds(ratio, None)
    d1_, d2_ = np.float32(a["d1"][0]), np.float32(a["d2"][0])
    assert d1_ == np.float32(np.float32(r2) * d2_)  # on the fp32 boundary
    if ratio != 0.5:
        assert float(d1_) > r2 * float(d2_)  # and past it in float64
    assert nno.match(d0, d1, ratio_thresh=ratio * 0.999, mutual_check=False)["matches0"][0].tolist() == [-1]
    fast = nno.match_chunked(d0, d1, ratio_thresh=ratio, mutual_check=False)
    assert fast["matches0"][0].tolist() == [0]


# ----------------------------------------------------------------------------------------------- the chunked oracle
def _assert_same(fast, slow):
    for k in ("matches0", "matches1", "matching_scores0", "matching_scores1"):
        np.testing.assert_array_equal(fast[k], slow[k], err_msg=k)
    for b in range(len(slow["matches"])):
        np.testing.assert_array_equal(fast["matches"][b], slow["matches"][b])
        np.testing.assert_array_equal(fast["scores"][b], slow["scores"][b])
        for fs, ss in zip(fast["sides"][b], slow["sides"][b]):
            for k in ss:
                np.testing.assert_array_equal(fs[k], ss[k], err_msg=k)


def _existing_cases():
    """The inputs of tests/test_nn_oracle.py and the grid pairs of the GPU tests."""
    def e(*iv, d=8):
        v = np.zeros(d)
        for i, x in iv:
            v[i] = x
        return v
    g = np.random.default_rng(1)
    cases = [
        (np.array([[e((0, 1.0)), e((1, 1.0))]]), np.array([[e((2, 1.0)), e((0, .5)), e((0, .5)), e((1, 1.0)),
                                                             e((1, 1.0))]]), {"mutual_check": False}),
        (np.array([[e((0, 1.0))]]), np.array([[e((0, .5)), e((0, .5)), e((1, 1.0))]]), {"ratio_thresh": 0.99}),
        (np.array([[e((0, 1.0)), e((1, 1.0))]]), np.array([[e((0, .875)), e((0, .5)), e((1, .875)), e((1, .5625))]]),
         {"ratio_thresh": 0.5, "mutual_check": False}),
        (np.array([[e((0, 1.0)), e((1, -1.0))]]), np.array([[e((0, 1.0))]]), {"ratio_thresh": 0.1}),
        (np.array([[e((0, 1.0)), e((1, 1.0))]]), np.array([[e((0, .875)), e((1, .8125))]]), {"distance_thresh": 0.5}),
        (np.array([[e((0, 1.0)), e((0, .9))]]), np.array([[e((0, 1.0)), e((1, 1.0))]]), {}),
        (np.ones((2, 0, 8)), np.ones((2, 3, 8)), {"ratio_thresh": 0.8}),
        (np.ones((2, 3, 8)), np.ones((2, 0, 8)), {"ratio_thresh": 0.8}),
    ]
    for kw in ({}, {"ratio_thresh": 0.5}, {"distance_thresh": 0.9},
               {"ratio_thresh": 0.8, "distance_thresh": 1.2, "mutual_check": False}):
        cases.append((g.integers(-2, 3, (3, 40, 64)) / 16, g.integers(-2, 3, (3, 33, 64)) / 16, kw))
    for ratio, dist, mutual in ((None, None, True), (0.8, 0.5, False), (0.9, 1.3, True)):
        cases.append((g.integers(-2, 3, (3, 300, 64)) / 16, g.integers(-2, 3, (3, 260, 64)) / 16,
                      {"ratio_thresh": ratio, "distance_thresh": dist, "mutual_check": mutual}))
    return cases


def test_chunked_oracle_equals_the_row_loop_on_every_existing_case():
    for d0, d1, kw in _existing_cases():
        for chunk in (7, 4096):
            _assert_same(nno.match_chunked(d0, d1, chunk=chunk, **kw), nno.match(d0, d1, **kw))
    g = np.random.default_rng(0)
    d0, d1 = g.integers(-2, 3, (3, 9, 64)) / 16, g.integers(-2, 3, (3, 7, 64)) / 16
    lens0, lens1 = [9, 4, 0], [7, 1, 5]
    _assert_same(nno.match_chunked(d0, d1, lens0, lens1, ratio_thresh=0.9, chunk=3),
                 nno.match(d0, d1, lens0, lens1, ratio_thresh=0.9))


@pytest.mark.parametrize("ratio, dist, mutual", [(None, None, True), (0.8, None, False), (0.95, 1.3, True)])
def test_chunked_split_oracle_equals_the_row_loop_on_split_grid_pairs(ratio, dist, mutual):
    lens0, lens1 = [300, 0, 123], [260, 77, 260]
    d0, d1, _ = nc.make_pair(5, 3, 300, 260, 128, lens0, lens1)
    kw = dict(ratio_thresh=ratio, distance_thresh=dist, mutual_check=mutual, split=True)
    _assert_same(nno.match_chunked(d0, d1, lens0, lens1, chunk=100, **kw), nno.match(d0, d1, lens0, lens1, **kw))


def _guided_cases():
    out = []
    for kind in (geo.HOMOGRAPHY, geo.FUNDAMENTAL):
        g = np.random.default_rng(11 + kind)
        b, m, n = 3, 120, 90
        d0, d1 = nc.split_grid(g, (b, m, 64)), nc.split_grid(g, (b, n, 64))
        k0 = g.uniform([0, 0], [640, 480], (b, m, 2)).astype(np.float32)
        k1 = g.uniform([0, 0], [640, 480], (b, n, 2)).astype(np.float32)
        k0[0, 5] = np.nan
        if kind == geo.HOMOGRAPHY:
            model = np.stack([gs.true_homography(g) for _ in range(b)])
        else:
            model = np.stack([gs.two_view(8, 0.0, int(s))[4] for s in g.integers(0, 1000, b)])
        out.append((kind, d0, d1, k0, k1, model, 60.0 if kind == geo.HOMOGRAPHY else 24.0))
    return out


def test_chunked_gate_is_the_gate_bit_for_bit():
    for kind, _, _, k0, k1, model, px in _guided_cases():
        want = ngo.gate(kind, model, k0, k1, px)
        fn = ngo.chunk_gate(kind, model, k0, k1, px)
        for b in range(len(model)):
            np.testing.assert_array_equal(torch.cat([fn(b, 0, r, min(r + 50, 120)) for r in range(0, 120, 50)]).numpy(),
                                          want[b])
            np.testing.assert_array_equal(torch.cat([fn(b, 1, r, min(r + 40, 90)) for r in range(0, 90, 40)]).numpy(),
                                          want[b].T)
        assert 0.01 < want.mean() < 0.6 and not want[0, 5].any()
    # an error exactly at t2 fails (identity H, max_error 1: x1 = x0 + (1, 0)); half of it passes
    k0 = np.array([[[10, 10]]], np.float32)
    k1 = np.array([[[11, 10], [10.5, 10]]], np.float32)
    fn = ngo.chunk_gate(geo.HOMOGRAPHY, np.eye(3)[None], k0, k1, 1.0)
    assert fn(0, 0, 0, 1).tolist() == [[False, True]] == ngo.gate(geo.HOMOGRAPHY, np.eye(3)[None], k0, k1, 1.0)[0].tolist()


@pytest.mark.parametrize("mutual", [True, False])
def test_chunked_guided_oracle_equals_the_row_loop(mutual):
    for kind, d0, d1, k0, k1, model, px in _guided_cases():
        valid = [1, 0, 1]
        lens0, lens1 = [120, 50, 0], [90, 90, 33]
        kw = dict(ratio_thresh=0.9, mutual_check=mutual, split=True)
        slow = ngo.match(d0, d1, lens0, lens1, gate=ngo.gate(kind, model, k0, k1, px, valid), **kw)
        fast = nno.match_chunked(d0, d1, lens0, lens1, chunk=32, **kw,
                                 gate=ngo.chunk_gate(kind, model, k0, k1, px, valid, lens0, lens1))
        _assert_same(fast, slow)


# ----------------------------------------------------------------------------------------------- stage restatements
@pytest.mark.parametrize("ratio, dist, mutual", [(None, None, True), (0.8, 1.3, False), (0.95, None, True)])
def test_stage_restatements_compose_to_the_oracle(ratio, dist, mutual):
    d0, d1, _ = nc.make_pair(9, 1, 300, 270, 64)
    want = nno.match(d0, d1, ratio_thresh=ratio, distance_thresh=dist, mutual_check=mutual, split=True)
    r2, t2 = nno.thresholds(ratio, dist)
    S = torch.as_tensor(nno.similarity(d0[0].astype(np.float64), d1[0].astype(np.float64), True))
    sides = []
    for X, n in ((S, 270), (S.T, 300)):
        s1, s2, j1 = nc.slot_partials(X, n)
        part = torch.stack([s1, s2], -1).numpy()
        sides.append(nc.tail(part, j1.numpy(), n, r2, t2))
    out = nc.outputs(*sides[0], *sides[1], 300, 270, mutual)
    for k in ("matches0", "matches1", "matching_scores0", "matching_scores1"):
        np.testing.assert_array_equal(out[k], want[k][0], err_msg=k)
    np.testing.assert_array_equal(out["matches"], want["matches"][0])


# --------------------------------------------------------------------------------------------- nn_workspace_layout
NAMES = ("hi", "lo", "part", "parg", "jbest", "sbest", "len", "stop", "rec", "gate_on")


def _layout(b, m, n, d, guided):
    off = (C.c_int64 * _cabi.NN_LAYOUT_BUFFERS)()
    size = (C.c_int64 * _cabi.NN_LAYOUT_BUFFERS)()
    plan = (C.c_int32 * 4)()
    total = _cabi.load().nn_workspace_layout(b, m, n, d, int(guided), off, size, plan)
    return dict(zip(NAMES, zip(off, size))), tuple(plan), total


@pytest.mark.parametrize("b, m, n, d", [(1, 1, 1, 64), (17, 3000, 3000, 128), (1, 40000, 1, 64), (2, 33000, 20000, 64),
                                        (32, 2048, 2048, 256), (3, 300, 5000, 512)])
@pytest.mark.parametrize("guided", [False, True])
def test_workspace_layout(b, m, n, d, guided):
    lib = _cabi.load()
    bufs, (G, Lp, pstride, groups), total = _layout(b, m, n, d, guided)
    assert total == (lib.nn_guided_workspace_bytes if guided else lib.nn_workspace_bytes)(b, m, n, d)
    assert Lp == (max(m, n) + 127) // 128 * 128 and pstride == 2 * ((Lp + 255) // 256)
    assert G * Lp <= _cabi.NN_GROUP_ROWS or G == 1
    assert groups == -(-b // G) and (groups - 1) * G < b
    R = 2 * G * Lp
    sizes = {"hi": R * d * 2, "lo": R * d * 2, "part": R * pstride * 8, "parg": R * pstride * 4, "jbest": R * 4,
             "sbest": R * 4, "len": 2 * G * 4, "stop": G * 4, "rec": R * 24 if guided else 0,
             "gate_on": G * 4 if guided else 0}
    spans = []
    for k in NAMES:
        o, s = bufs[k]
        assert s == sizes[k], k
        if not guided and k in ("rec", "gate_on"):
            assert o == -1
            continue
        assert o % 256 == 0 and o + s <= total, k
        spans.append((o, o + s))
    spans.sort()
    assert all(a[1] <= b_[0] for a, b_ in zip(spans, spans[1:]))  # disjoint


def test_workspace_layout_regimes():
    with open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "nn_b200.h")) as f:
        assert re.search(r"#define NN_LAYOUT_BUFFERS (\d+)", f.read()).group(1) == str(_cabi.NN_LAYOUT_BUFFERS)
    assert _layout(17, 3000, 3000, 128, False)[1][::3] == (9, 2)  # groups of 9 and 8
    assert _layout(2, 33000, 20000, 64, False)[1][:2] == (1, 33024)  # one pair wider than NN_GROUP_ROWS
    assert _layout(1, 1, 1, 64, False)[1] == (1, 128, 2, 1)


def test_workspace_layout_rejects_bad_arguments():
    lib = _cabi.load()
    for args in ((0, 10, 10, 64), (-1, 10, 10, 64), (1, -1, 10, 64), (1, 10, -1, 64), (1, 10, 10, 96), (1, 10, 10, 576)):
        assert lib.nn_workspace_layout(*args, 0, None, None, None) == 0, args
    assert lib.nn_workspace_layout(1, 10, 10, 64, 0, None, None, None) == lib.nn_workspace_bytes(1, 10, 10, 64)
