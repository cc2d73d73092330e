"""Batched undistortion and distortion on the GPU (lightglue_b200.camera, header steps D1-D3) bit for bit against
oracle/camera_oracle.py: float32 and float64 inputs, per-pair K and coefficients, with and without the EPS stop, at
B = 32 x 8192; NaN rows and invalid K or coefficients; batches against single pairs; repeats and CUDA-graph replay."""
import numpy as np
import pytest
import torch

from lightglue_b200.camera import distort_points, undistort_points
from oracle import camera_oracle as co

pytestmark = pytest.mark.gpu

DIST = {4: [-0.3, 0.09, 1e-3, -5e-4], 5: [-0.28, 0.07, 8e-4, -6e-4, -0.01],
        8: [-0.25, 0.05, 5e-4, -3e-4, 0.002, 0.02, 0.004, 0.001],
        12: [-0.25, 0.06, 6e-4, -4e-4, 0.003, 0.01, 0.002, 0.0005, 1e-3, -2e-4, -8e-4, 3e-4]}


def _batch(B, N, nd, dtype, seed=0):
    rng = np.random.default_rng(seed)
    px = np.stack([rng.uniform(0, 640, (B, N)), rng.uniform(0, 480, (B, N))], -1).astype(dtype)
    K = np.tile(np.array([[500.0, 0.3, 320.0], [0.0, 480.0, 240.0], [0.0, 0.0, 1.0]]), (B, 1, 1))
    K[:, 0, 0] += rng.uniform(-50, 50, B)
    K[:, 1, 2] += rng.uniform(-10, 10, B)
    d = np.array(DIST[nd])[None] * rng.uniform(0.5, 1.2, (B, 1))
    return px, K, d


def _cuda(*xs):
    return [torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in xs]


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("nd", [4, 5, 8, 12])
@pytest.mark.parametrize("eps", [0.0, 1e-4])
def test_undistort_bit_for_bit(dtype, nd, eps):
    px, K, d = _batch(4, 1000, nd, dtype, seed=nd)
    it = 5 if eps == 0.0 else 30
    got = undistort_points(*_cuda(px, K, d), max_iters=it, eps=eps).cpu().numpy()
    ref = co.undistort_points(px, K, d, max_iters=it, eps=eps)
    assert got.dtype == dtype and np.array_equal(got, ref)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("nd", [4, 5, 8, 12])
def test_distort_bit_for_bit(dtype, nd):
    px, K, d = _batch(4, 1000, nd, dtype, seed=10 + nd)
    got = distort_points(*_cuda(px, K, d)).cpu().numpy()
    assert got.dtype == dtype and np.array_equal(got, co.distort_points(px, K, d))


def test_large_batch_and_single_pairs():
    px, K, d = _batch(32, 8192, 8, np.float32, seed=3)
    tp, tK, td = _cuda(px, K, d)
    got = undistort_points(tp, tK, td)
    for p in (0, 17, 31):
        one = undistort_points(tp[p:p + 1], tK[p], td[p])  # [3, 3] and [k] broadcast over a batch of one
        assert torch.equal(got[p:p + 1], one)
        assert np.array_equal(got[p].cpu().numpy(), co.undistort_points(px[p:p + 1], K[p], d[p])[0])
    assert torch.equal(distort_points(tp, tK, td)[5], distort_points(tp[5:6], tK[5:6], td[5:6])[0])


def test_nan_rows_and_invalid_cameras():
    px, K, d = _batch(4, 64, 5, np.float64, seed=4)
    px[0, 3, 0] = np.nan
    px[0, 4, 1] = np.inf
    K[1, 2, 2] = 0.5          # invalid K
    d[2, 1] = np.nan          # invalid coefficients
    for f, g in ((undistort_points, co.undistort_points), (distort_points, co.distort_points)):
        got = f(*_cuda(px, K, d)).cpu().numpy()
        ref = g(px, K, d)
        assert np.array_equal(got, ref, equal_nan=True)
        assert np.isnan(got[0, [3, 4]]).all() and np.isfinite(np.delete(got[0], [3, 4], 0)).all()
        assert np.isnan(got[1]).all() and np.isnan(got[2]).all() and np.isfinite(got[3]).all()


def test_repeats_and_graph_replay():
    px, K, d = _batch(8, 4096, 12, np.float32, seed=5)
    tp, tK, td = _cuda(px, K, d)
    first = undistort_points(tp, tK, td, max_iters=20, eps=1e-3)
    assert torch.equal(first, undistort_points(tp, tK, td, max_iters=20, eps=1e-3))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):  # warm up (and load the library) outside the capture
        undistort_points(tp, tK, td, max_iters=20, eps=1e-3)
        distort_points(tp, tK, td)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        u = undistort_points(tp, tK, td, max_iters=20, eps=1e-3)
        v = distort_points(u, tK, td)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(u, first)
    assert torch.equal(v, distort_points(first, tK, td))
    tp.copy_(torch.flip(tp, [0]))
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(u, undistort_points(tp, tK, td, max_iters=20, eps=1e-3))
