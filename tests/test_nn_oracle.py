"""The nearest-neighbour oracle (oracle/nn_oracle.py) against a brute-force torch float64 restatement of
include/nn_b200.h, on hand-made cases for every rule: ties, the ratio and distance boundaries, a single neighbour,
empty images and the mutual check."""
import numpy as np
import pytest
import torch

from oracle import nn_oracle as nno


def brute(d0, d1, ratio=None, dist=None, mutual=True):
    """The same rules in torch: einsum, argmax (first maximum), the second best by masking, the mutual check by a
    gather.  Returns matches0, matches1, scores0, scores1."""
    d0 = torch.as_tensor(d0, dtype=torch.float64)
    d1 = torch.as_tensor(d1, dtype=torch.float64)
    r2, t2 = nno.thresholds(ratio, dist)

    def side(S):
        rows, cols = S.shape
        if cols == 0:
            return torch.full((rows,), -1, dtype=torch.int64), torch.zeros(rows, dtype=torch.float64)
        j1 = S.argmax(-1)  # documented: the first maximal value
        s1 = S.gather(-1, j1[:, None])[:, 0]
        masked = S.clone()
        masked[torch.arange(rows), j1] = -torch.inf
        s2 = masked.max(-1).values if cols > 1 else torch.full((rows,), -torch.inf, dtype=torch.float64)
        d1_, d2_ = 2 * (1 - s1), 2 * (1 - s2)
        keep = torch.ones(rows, dtype=torch.bool)
        if r2 is not None:
            keep &= d1_ <= r2 * d2_
        if t2 is not None:
            keep &= d1_ <= t2
        return torch.where(keep, j1, torch.full_like(j1, -1)), s1

    out = []
    for b in range(d0.shape[0]):
        S = d0[b] @ d1[b].T
        a, s_a = side(S)
        c, s_c = side(S.T)
        if mutual and len(a) and len(c):  # an empty side has matched nothing already
            a, c = (torch.where((a >= 0) & (c.gather(0, a.clamp(min=0)) == torch.arange(len(a))), a, -1),
                    torch.where((c >= 0) & (a.gather(0, c.clamp(min=0)) == torch.arange(len(c))), c, -1))
        out.append((a, c, torch.where(a >= 0, (s_a + 1) / 2, 0.0).float(), torch.where(c >= 0, (s_c + 1) / 2, 0.0).float()))
    return [torch.stack([o[k] for o in out]) for k in range(4)]


def check(d0, d1, **kw):
    res = nno.match(d0, d1, ratio_thresh=kw.get("ratio"), distance_thresh=kw.get("dist"),
                    mutual_check=kw.get("mutual", True))
    m0, m1, s0, s1 = brute(d0, d1, **kw)
    np.testing.assert_array_equal(res["matches0"], m0.numpy())
    np.testing.assert_array_equal(res["matches1"], m1.numpy())
    np.testing.assert_array_equal(res["matching_scores0"], s0.numpy())
    np.testing.assert_array_equal(res["matching_scores1"], s1.numpy())
    for b in range(len(res["matches"])):
        rows = np.flatnonzero(res["matches0"][b] >= 0)
        np.testing.assert_array_equal(res["matches"][b], np.stack([rows, res["matches0"][b, rows]], 1).reshape(-1, 2))
    return res


def e(*idx_val, d=8):
    v = np.zeros(d)
    for i, x in idx_val:
        v[i] = x
    return v


def test_exact_tie_goes_to_the_lowest_index():
    d0 = np.array([[e((0, 1.0)), e((1, 1.0))]])
    d1 = np.array([[e((2, 1.0)), e((0, 0.5)), e((0, 0.5)), e((1, 1.0)), e((1, 1.0))]])
    res = check(d0, d1, mutual=False)
    assert res["matches0"][0].tolist() == [1, 3]
    a, _ = res["sides"][0]
    assert a["s1"][1] == a["s2"][1] == 1.0  # s1 == s2 on a tie


def test_equal_best_and_second_fails_any_ratio_below_one():
    d0 = np.array([[e((0, 1.0))]])
    d1 = np.array([[e((0, 0.5)), e((0, 0.5)), e((1, 1.0))]])
    assert check(d0, d1, ratio=0.99, mutual=False)["matches0"][0].tolist() == [-1]
    assert check(d0, d1, ratio=1.0, mutual=False)["matches0"][0].tolist() == [0]


def test_ratio_boundary_is_kept():
    # s1 = 0.875, s2 = 0.5: D1 = 0.25 = 0.5^2 * D2 exactly; 0.5625 as second best fails it
    d0 = np.array([[e((0, 1.0)), e((1, 1.0))]])
    d1 = np.array([[e((0, 0.875)), e((0, 0.5)), e((1, 0.875)), e((1, 0.5625))]])
    res = check(d0, d1, ratio=0.5, mutual=False)
    assert res["matches0"][0].tolist() == [0, -1]
    a, _ = res["sides"][0]
    assert a["d1"][0] == 0.25 and a["d2"][0] == 1.0


def test_single_neighbour_passes_the_ratio_test():
    d0 = np.array([[e((0, 1.0)), e((1, -1.0))]])
    d1 = np.array([[e((0, 1.0))]])
    res = check(d0, d1, ratio=0.1, mutual=False)
    assert res["matches0"][0].tolist() == [0, 0]
    assert res["sides"][0][0]["s2"][0] == -np.inf


def test_distance_test_alone():
    # s = 0.875: D1 = 0.25 = 0.5^2 is kept; s = 0.8125 (D1 = 0.375) is not
    d0 = np.array([[e((0, 1.0)), e((1, 1.0))]])
    d1 = np.array([[e((0, 0.875)), e((1, 0.8125))]])
    assert check(d0, d1, dist=0.5)["matches0"][0].tolist() == [0, -1]
    assert check(d0, d1, dist=0.5, mutual=False)["matches0"][0].tolist() == [0, -1]
    assert check(d0, d1)["matches0"][0].tolist() == [0, 1]


def test_mutual_versus_one_way():
    d0 = np.array([[e((0, 1.0)), e((0, 0.9))]])
    d1 = np.array([[e((0, 1.0)), e((1, 1.0))]])
    one = check(d0, d1, mutual=False)
    assert one["matches0"][0].tolist() == [0, 0] and one["matches1"][0].tolist() == [0, 0]
    mut = check(d0, d1, mutual=True)
    assert mut["matches0"][0].tolist() == [0, -1] and mut["matches1"][0].tolist() == [0, -1]
    assert [m.tolist() for m in mut["matches"]] == [[[0, 0]]]
    assert mut["matching_scores0"][0].tolist() == [1.0, 0.0]


@pytest.mark.parametrize("m,n", [(0, 3), (3, 0), (0, 0)])
def test_empty_images_match_nothing(m, n):
    res = check(np.ones((2, m, 8)), np.ones((2, n, 8)), ratio=0.8)
    assert (res["matches0"] == -1).all() and (res["matches1"] == -1).all()
    assert all(len(x) == 0 for x in res["matches"])


def test_ragged_lengths_cut_each_pair():
    g = np.random.default_rng(0)
    d0 = g.integers(-2, 3, (3, 9, 64)) / 16
    d1 = g.integers(-2, 3, (3, 7, 64)) / 16
    lens0, lens1 = [9, 4, 0], [7, 1, 5]
    res = nno.match(d0, d1, lens0, lens1, ratio_thresh=0.9)
    for b in range(3):
        one = nno.match(d0[b : b + 1, : lens0[b]], d1[b : b + 1, : lens1[b]], ratio_thresh=0.9)
        assert res["matches0"][b, : lens0[b]].tolist() == one["matches0"][0].tolist()
        assert (res["matches0"][b, lens0[b] :] == -1).all() and (res["matches1"][b, lens1[b] :] == -1).all()


@pytest.mark.parametrize("kw", [{}, {"ratio": 0.5}, {"dist": 0.9}, {"ratio": 0.8, "dist": 1.2, "mutual": False}])
def test_coarse_grid_descriptors_with_many_ties(kw):
    g = np.random.default_rng(1)
    check(g.integers(-2, 3, (3, 40, 64)) / 16, g.integers(-2, 3, (3, 33, 64)) / 16, **kw)


def test_decided_rows_leave_out_near_ties():
    d0 = np.array([[e((0, 1.0)), e((1, 1.0))]])
    d1 = np.array([[e((0, 1.0)), e((0, 0.99995)), e((1, 1.0)), e((2, 1.0))]])
    res = nno.match(d0, d1, mutual_check=True)
    assert nno.decided(res, 0, 0, 2e-4, 4e-4, True).tolist() == [False, True]
