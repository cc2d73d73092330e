"""The guided matcher's oracle (oracle/nn_guided_oracle.py): its gate is the estimators' inlier test, its ``match``
follows include/nn_b200.h's rules over the gated columns, and without a gate it is oracle/nn_oracle.py's."""
import numpy as np
import pytest

from oracle import geometry_oracle as geo
from oracle import geometry_synth as gs
from oracle import nn_guided_oracle as ngo
from oracle import nn_oracle as nno


def _unit(g, *shape):
    x = g.normal(size=shape)
    return x / np.linalg.norm(x, axis=-1, keepdims=True)


@pytest.mark.parametrize("kind", [geo.HOMOGRAPHY, geo.FUNDAMENTAL])
@pytest.mark.parametrize("thr", [1.0, 3.0])
def test_gate_is_the_estimators_inlier_mask_at_the_same_threshold(kind, thr):
    k0, k1, m0, _, _ = gs.batch("H" if kind == geo.HOMOGRAPHY else "F", 120, 0.3, [11, 12])
    est = geo.estimate(kind, k0, k1, m0, thr, 200, 0.999, 7)
    g = ngo.gate(kind, est["model"], k0, k1, thr)
    for b in range(2):
        assert est["success"][b]
        i = np.flatnonzero(m0[b] >= 0)
        np.testing.assert_array_equal(g[b, i, m0[b, i]], est["inliers"][b, i])
        assert g[b, i, m0[b, i]].sum() == est["num_inliers"][b]


@pytest.mark.parametrize("kind", [geo.HOMOGRAPHY, geo.FUNDAMENTAL])
def test_gate_is_errors_below_the_float_threshold(kind):
    k0, k1, _, _, model = gs.batch("H" if kind == geo.HOMOGRAPHY else "F", 40, 0.5, [3])
    k1 = k1[:, :33]
    g = ngo.gate(kind, model, k0, k1, 2.5)
    pts = np.array([[*k0[0, i], *k1[0, j]] for i in range(40) for j in range(33)], dtype=np.float32)
    err = geo.errors(kind, model.reshape(1, 9), pts)[0].reshape(40, 33)
    np.testing.assert_array_equal(g[0], err < np.float32(2.5 * 2.5))
    assert 0 < g.sum() < g.size


def test_gate_fails_nan_errors_and_passes_invalid_pairs():
    k0 = np.array([[[10.0, 20.0], [np.nan, 1.0], [5.0, 5.0]]] * 2, dtype=np.float32)
    k1 = np.array([[[10.0, 20.0], [11.0, 20.0], [np.inf, 0.0]]] * 2, dtype=np.float32)
    Hm = np.broadcast_to(np.eye(3), (2, 3, 3))
    g = ngo.gate(geo.HOMOGRAPHY, Hm, k0, k1, 1.0, valid=np.array([1, 0], dtype=np.uint8))
    assert g[0].tolist() == [[True, False, False], [False, False, False], [False, False, False]]
    assert g[1].all()
    # an error of exactly t2 fails: (11 - 10)^2 = 1 = 1.0^2
    assert not ngo.gate(geo.HOMOGRAPHY, Hm[:1], k0[:1], k1[:1], 1.0)[0, 0, 1]
    assert ngo.gate(geo.HOMOGRAPHY, Hm[:1], k0[:1], k1[:1], 1.0 + 1e-6)[0, 0, 1]
    # a zero F gives 0 * inf = NaN on both sides
    assert not ngo.gate(geo.FUNDAMENTAL, np.zeros((1, 3, 3)), k0[:1], k1[:1], 100.0).any()


@pytest.mark.parametrize("ratio, dist, mutual", [(None, None, True), (0.8, None, True), (0.9, 1.2, False),
                                                 (None, 0.9, False)])
def test_an_all_true_gate_is_the_ungated_match(ratio, dist, mutual):
    g = np.random.default_rng(5)
    d0, d1 = _unit(g, 3, 50, 64), _unit(g, 3, 40, 64)
    lens0, lens1 = [50, 17, 0], [40, 40, 9]
    a = nno.match(d0, d1, lens0, lens1, ratio, dist, mutual)
    assert ngo.match(d0, d1, lens0, lens1, ratio, dist, mutual)["matches0"].tolist() == a["matches0"].tolist()
    b = ngo.match(d0, d1, lens0, lens1, ratio, dist, mutual, gate=np.ones((3, 50, 40), dtype=bool))
    for k in ("matches0", "matches1", "matching_scores0", "matching_scores1"):
        np.testing.assert_array_equal(a[k], b[k])
    for x, y in zip(a["sides"], b["sides"]):
        for sa, sb in zip(x, y):
            for k in sa:
                np.testing.assert_array_equal(sa[k], sb[k], err_msg=k)


def test_gated_rows_follow_the_rules_over_gated_columns_only():
    s = np.array([[0.9, 0.8, 0.7, 0.1],    # row 0: the best column is gated out; 0.7 wins over 0.1
                  [0.5, 0.5, 0.2, 0.5],    # row 1: a tie among gated columns: the lowest gated j (1)
                  [0.9, 0.3, 0.2, 0.1],    # row 2: one gated column: s2 = -inf, the ratio test passes
                  [0.9, 0.8, 0.7, 0.6]])   # row 3: no gated column: nothing
    gate = np.array([[0, 0, 1, 1], [0, 1, 0, 1], [0, 1, 0, 0], [0, 0, 0, 0]], dtype=bool)
    r2, _ = nno.thresholds(0.5, None)
    o = ngo.one_way(s, r2, None, gate)
    assert o["j1"].tolist() == [2, 1, 1, -1]
    assert o["s2"][0] == 0.1 and o["s2"][1] == 0.5 and o["s2"][2] == -np.inf and o["s1"][3] == -np.inf
    assert o["keep"].tolist() == [False, False, True, False]
    assert o["gap"][1] == 0.0 and o["gap"][2] == np.inf and o["gap"][3] == np.inf
    assert o["ratio_margin"][2] == np.inf and o["ratio_margin"][3] == np.inf
    # without the gate row 0 names column 0, with s2 = 0.8 over every other column
    o = nno.one_way(s, r2, None)
    assert o["j1"][0] == 0 and o["s2"][0] == 0.8


def test_guided_match_uses_the_gate_from_both_sides_and_decided_still_works():
    g = np.random.default_rng(9)
    d0, d1 = _unit(g, 2, 60, 64), _unit(g, 2, 70, 64)
    gate = g.random((2, 60, 70)) < 0.2
    gate[0, 5] = False  # a row of image 0 with no gated column
    res = ngo.match(d0, d1, ratio_thresh=0.95, gate=gate)
    for b in range(2):
        i = np.flatnonzero(res["matches0"][b] >= 0)
        assert gate[b, i, res["matches0"][b, i]].all()
        j = np.flatnonzero(res["matches1"][b] >= 0)
        assert gate[b, res["matches1"][b, j], j].all()
        for side in (0, 1):
            ok = ngo.decided(res, b, side, 2e-4, 4e-4, True)
            assert ok.shape == (60 if side == 0 else 70,) and ok.any()
    assert res["matches0"][0, 5] == -1 and ngo.decided(res, 0, 0, 2e-4, 4e-4, False)[5]
    # monotonicity: an unguided match that passes the gate is a guided match with the same score
    plain = nno.match(d0, d1, ratio_thresh=0.95)
    for b in range(2):
        i = np.flatnonzero(plain["matches0"][b] >= 0)
        kept = i[gate[b, i, plain["matches0"][b, i]]]
        np.testing.assert_array_equal(res["matches0"][b, kept], plain["matches0"][b, kept])
        np.testing.assert_array_equal(res["matching_scores0"][b, kept], plain["matching_scores0"][b, kept])
