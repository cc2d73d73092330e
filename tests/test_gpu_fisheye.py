"""Batched fisheye undistortion and distortion on the GPU (lightglue_b200.camera.fisheye_undistort_points and
fisheye_distort_points, header steps FE1-FE4) bit for bit against oracle/fisheye_oracle.py: float32 and float64
inputs, per-pair K and D, every criterion variant; clamped, flipped and centre points, NaN rows, invalid K and D;
B = 32 x 8192; batches against single pairs; repeats and CUDA-graph replay."""
import numpy as np
import pytest
import torch

from lightglue_b200.camera import fisheye_distort_points, fisheye_undistort_points
from oracle import fisheye_oracle as fo

pytestmark = pytest.mark.gpu

D0 = np.array([0.03, -0.012, 0.004, -0.0006])
D_FAIL = np.array([-0.3, 0.1, -0.05, 0.01])   # FE3 fails on a large share of the image
CRITERIA = {"default": (10, 1e-8), "count_only": (10, 0.0), "count_eps_3": (3, 1e-3), "count_eps_30": (30, 1e-12),
            "zero_iters": (0, 1e-8)}


def _batch(B, N, dtype, seed=0, D=D0):
    """Pixels over a 1024 x 1024 fisheye image and beyond its 180 degree circle (the clamp), with the principal point
    and points a hair off it in every pair; per-pair K (with skew) and D."""
    rng = np.random.default_rng(seed)
    px = rng.uniform(-300, 1324, (B, N, 2))
    K = np.tile(np.array([[280.0, 0.0, 512.0], [0.0, 284.0, 505.0], [0.0, 0.0, 1.0]]), (B, 1, 1))
    K[:, 0, 0] += rng.uniform(-20, 20, B)
    K[:, 0, 1] = rng.uniform(-0.5, 0.5, B)
    K[:, :2, 2] += rng.uniform(-10, 10, (B, 2))
    px[:, 0] = K[:, :2, 2]
    px[:, 1] = K[:, :2, 2] + np.array([1e-7, 0.0])
    px[:, 2] = K[:, :2, 2] + np.array([0.0, 3e-6])
    d = D[None] * rng.uniform(0.5, 1.2, (B, 1))
    return px.astype(dtype), K, d


def _cuda(*xs):
    return [torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in xs]


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("crit", list(CRITERIA))
@pytest.mark.parametrize("lens", ["mild", "failing"])
def test_undistort_bit_for_bit(dtype, crit, lens):
    it, eps = CRITERIA[crit]
    px, K, d = _batch(4, 2000, dtype, seed=len(crit), D=D0 if lens == "mild" else D_FAIL)
    got = fisheye_undistort_points(*_cuda(px, K, d), max_iters=it, eps=eps).cpu().numpy()
    ref = fo.undistort_points(px, K, d, max_iters=it, eps=eps)
    assert got.dtype == dtype and np.array_equal(got, ref, equal_nan=True)
    if lens == "failing" and it > 0:
        assert np.isnan(got).any() and np.isfinite(got).any()


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_distort_bit_for_bit(dtype):
    px, K, d = _batch(4, 2000, dtype, seed=9)
    got = fisheye_distort_points(*_cuda(px, K, d)).cpu().numpy()
    assert got.dtype == dtype and np.array_equal(got, fo.distort_points(px, K, d), equal_nan=True)


def test_large_batch_and_single_pairs():
    px, K, d = _batch(32, 8192, np.float32, seed=3)
    tp, tK, td = _cuda(px, K, d)
    got = fisheye_undistort_points(tp, tK, td)
    for p in (0, 17, 31):
        one = fisheye_undistort_points(tp[p:p + 1], tK[p], td[p])  # [3, 3] and [4] broadcast over a batch of one
        assert torch.equal(got[p:p + 1].isnan(), one.isnan())
        assert torch.equal(got[p:p + 1].nan_to_num(), one.nan_to_num())
        assert np.array_equal(got[p].cpu().numpy(), fo.undistort_points(px[p:p + 1], K[p], d[p])[0], equal_nan=True)
    dist = fisheye_distort_points(tp, tK, td)
    assert torch.equal(dist[5], fisheye_distort_points(tp[5:6], tK[5:6], td[5:6])[0])
    assert np.array_equal(dist[31].cpu().numpy(), fo.distort_points(px[31:], K[31], d[31])[0])


def test_nan_rows_and_invalid_cameras():
    px, K, d = _batch(4, 64, np.float64, seed=4)
    px[0, 3, 0] = np.nan
    px[0, 4, 1] = np.inf
    K[1, 2, 2] = 0.5          # invalid K
    d[2, 1] = np.nan          # invalid coefficients
    for f, g in ((fisheye_undistort_points, fo.undistort_points), (fisheye_distort_points, fo.distort_points)):
        got = f(*_cuda(px, K, d)).cpu().numpy()
        assert np.array_equal(got, g(px, K, d), equal_nan=True)
        assert np.isnan(got[0, [3, 4]]).all()
        assert np.isnan(got[1]).all() and np.isnan(got[2]).all() and not np.isnan(got[3]).all()


def test_repeats_and_graph_replay():
    px, K, d = _batch(8, 4096, np.float32, seed=5)
    tp, tK, td = _cuda(px, K, d)
    first = fisheye_undistort_points(tp, tK, td, max_iters=20, eps=1e-10)
    assert torch.equal(first.nan_to_num(), fisheye_undistort_points(tp, tK, td, max_iters=20, eps=1e-10).nan_to_num())
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):  # warm up (and load the library) outside the capture
        fisheye_undistort_points(tp, tK, td, max_iters=20, eps=1e-10)
        fisheye_distort_points(tp, tK, td)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        u = fisheye_undistort_points(tp, tK, td, max_iters=20, eps=1e-10)
        v = fisheye_distort_points(u, tK, td)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(u.nan_to_num(), first.nan_to_num())
    assert torch.equal(v.nan_to_num(), fisheye_distort_points(first, tK, td).nan_to_num())
    tp.copy_(torch.flip(tp, [0]))
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(u.nan_to_num(), fisheye_undistort_points(tp, tK, td, max_iters=20, eps=1e-10).nan_to_num())
