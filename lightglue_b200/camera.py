"""Lens distortion on the GPU: batched undistortion and distortion of keypoints under OpenCV's camera model and its
fisheye model (C ABI ``include/geometry_b200.h``, steps D1-D3 and FE1-FE4, CUDA ``csrc/camera_api.cu``).

The model is OpenCV's rational model with thin prism terms, coefficients (k1, k2, p1, p2[, k3[, k4, k5, k6[, s1, s2,
s3, s4]]]): 4, 5, 8 or 12 of them, missing trailing ones zero.  COLMAP's ``SIMPLE_RADIAL`` (f, cx, cy, k) is
``[k, 0, 0, 0]``, ``RADIAL`` (f, cx, cy, k1, k2) ``[k1, k2, 0, 0]``, ``OPENCV`` (fx, fy, cx, cy, k1, k2, p1, p2)
``[k1, k2, p1, p2]`` and ``FULL_OPENCV`` its eight coefficients in their order, which is OpenCV's.  The 14-coefficient
tilted model is refused.

The fisheye model (``cv2.fisheye``, equidistant or Kannala-Brandt) has exactly 4 coefficients (k1, k2, k3, k4) and its
own functions, ``fisheye_undistort_points`` and ``fisheye_distort_points``.  COLMAP's ``OPENCV_FISHEYE`` is K and its
four coefficients, ``RADIAL_FISHEYE`` (f, cx, cy, k1, k2) ``[k1, k2, 0, 0]`` and ``SIMPLE_RADIAL_FISHEYE`` (f, cx, cy,
k) ``[k, 0, 0, 0]``; ``FOV`` and ``THIN_PRISM_FISHEYE`` are other models and are not supported.

All four functions run on the current stream, return device tensors of fixed shapes without synchronising with the host
and launch one kernel, so they can be captured in a CUDA graph and chained into any estimator of
``lightglue_b200.geometry`` or into ``NearestNeighborMatcher``.  An invalid K (a non-finite entry, fx or fy <= 0, or a
bottom row other than [0, 0, 1]), a non-finite coefficient or a non-finite input pixel gives a NaN row, which every
estimator treats as an invalid match.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _cabi

DIST_LENGTHS = (4, 5, 8, 12)


def _check_pixels(name: str, pts) -> None:
    if not isinstance(pts, torch.Tensor):
        raise ValueError(f"{name} must be a torch.Tensor")
    if pts.device.type != "cuda":
        raise RuntimeError("lightglue_b200.camera runs on CUDA (sm_90a) tensors only; there is no CPU path")
    if pts.dim() != 3 or pts.shape[-1] != 2:
        raise ValueError(f"{name} {tuple(pts.shape)}: expected [B, N, 2]")
    if pts.dtype not in (torch.float32, torch.float64):
        raise ValueError(f"{name} must be float32 or float64, not {pts.dtype}")


def check_fisheye_count(name: str, d) -> None:
    """Refuses fisheye coefficients that are missing or not 4 per pair ([4] or [B, 4]); the rest of the checks are
    dist_coeffs'."""
    if d is None:
        raise ValueError(f"{name}: the fisheye model needs its 4 coefficients (k1, k2, k3, k4), not None")
    if isinstance(d, torch.Tensor) and d.dim() in (1, 2) and d.shape[-1] != 4:
        raise ValueError(f"{name}: {d.shape[-1]} coefficients; the fisheye model takes exactly 4 (k1, k2, k3, k4)")


def dist_coeffs(name: str, d, b: int, device, fisheye: bool = False) -> torch.Tensor:
    """Checks distortion coefficients [k] or [B, k] (k = 4 for the fisheye model) and returns them as a contiguous
    [B, k] float64 tensor."""
    if not isinstance(d, torch.Tensor):
        raise ValueError(f"{name} must be a torch.Tensor")
    if not d.is_floating_point():
        raise ValueError(f"{name} must be floating point")
    if d.dim() == 1:
        d = d.expand(b, d.shape[0])
    elif d.dim() != 2 or d.shape[0] != b:
        raise ValueError(f"{name} {tuple(d.shape)}: expected [k] or [B, k] with B = {b}")
    k = d.shape[1]
    if fisheye:
        check_fisheye_count(name, d)
    if k == 14:
        raise ValueError(f"{name}: the 14-coefficient tilted model (tauX, tauY) is not supported")
    if k not in DIST_LENGTHS:
        raise ValueError(f"{name}: {k} coefficients; expected 4, 5, 8 or 12 (k1, k2, p1, p2[, k3[, k4, k5, k6[, s1, "
                         f"s2, s3, s4]]])")
    if d.device.type != "cuda":
        raise RuntimeError("lightglue_b200 runs on CUDA (sm_90a) tensors only; there is no CPU path")
    if d.device != device:
        raise ValueError(f"{name} must be on the device of the keypoints")
    return d.detach().to(torch.float64).contiguous()


def _camera(entry: str, pts, K, dist, max_iters: int, eps: float, fisheye: bool = False) -> torch.Tensor:
    from .geometry import _intrinsics

    _check_pixels("kpts", pts)
    b, n = pts.shape[0], pts.shape[1]
    k = _intrinsics("K", K, b, pts.device)
    d = dist_coeffs("D" if fisheye else "dist_coeffs", dist, b, pts.device, fisheye)
    p = pts.detach().contiguous()
    out = torch.empty_like(p)
    if b == 0 or n == 0:
        return out
    dtype = _cabi.GEO_CAMERA_FLOAT64 if p.dtype == torch.float64 else _cabi.GEO_CAMERA_FLOAT32
    with torch.cuda.device(p.device):
        lib = _cabi.load()
        cfg = _cabi.GeoCameraConfig(_cabi.GEO_ABI_VERSION, d.shape[1], max_iters, dtype, float(eps))
        ins = _cabi.GeoCameraInputs(b, n, p.data_ptr(), k.data_ptr(), d.data_ptr())
        outs = _cabi.GeoCameraOutputs(out.data_ptr())
        _cabi.check(getattr(lib, entry)(C.byref(cfg), C.byref(ins), C.byref(outs),
                                        torch.cuda.current_stream(p.device).cuda_stream), entry)
    return out


def undistort_points(kpts: torch.Tensor, K: torch.Tensor, dist_coeffs: torch.Tensor, max_iters: int = 5,
                     eps: float = 0.0) -> torch.Tensor:
    """Undistorted pixels of ``kpts`` [B, N, 2] (float32 or float64) through ``K`` ([3, 3] or [B, 3, 3]) and
    ``dist_coeffs`` ([k] or [B, k], k = 4, 5, 8 or 12), as [B, N, 2] in the input's dtype, computed in double.

    OpenCV's fixed-point iteration (header step D2): at most ``max_iters`` iterations (in [0, 1000]), stopping early
    once the previous iterate reprojects within ``eps`` pixels (0: never).  The defaults give
    ``cv2.undistortPoints(kpts, K, d, P=K)``; ``cv2.undistortPointsIter`` with a COUNT + EPS criterion is
    ``max_iters`` and ``eps``.  The trade-off: at strong distortion OpenCV's 5 iterations are measurably
    unconverged (at f = 500, 640x480 and k1 = -0.3, the image corners round-trip with errors up to 0.14 px), and
    every further iteration costs one more pass of the iteration per point; raise ``max_iters`` (or set a small
    ``eps``, which stops each point once it has converged) where sub-pixel accuracy matters more than matching
    ``cv2.undistortPoints``."""
    _check_criteria(max_iters, eps, "pixels")
    return _camera("geo_undistort_points", kpts, K, dist_coeffs, max_iters, eps)


def _check_criteria(max_iters, eps, unit: str) -> None:
    bound = _cabi.GEO_UNDISTORT_MAX_ITERS
    if not isinstance(max_iters, int) or isinstance(max_iters, bool) or not 0 <= max_iters <= bound:
        raise ValueError(f"max_iters={max_iters!r}: an int in [0, {_cabi.GEO_UNDISTORT_MAX_ITERS}]")
    if not 0.0 <= float(eps) < float("inf"):
        raise ValueError(f"eps={eps!r}: a finite number of {unit} >= 0")


def distort_points(kpts: torch.Tensor, K: torch.Tensor, dist_coeffs: torch.Tensor) -> torch.Tensor:
    """Distorted pixels of the undistorted pixels ``kpts`` [B, N, 2]: ``cv2.projectPoints`` of K^-1 [u, v, 1]
    through (K, dist_coeffs) (header step D1).  Arguments as ``undistort_points``."""
    return _camera("geo_distort_points", kpts, K, dist_coeffs, 0, 0.0)


def fisheye_undistort_points(kpts: torch.Tensor, K: torch.Tensor, D: torch.Tensor, max_iters: int = 10,
                             eps: float = 1e-8) -> torch.Tensor:
    """Undistorted pixels of the fisheye pixels ``kpts`` [B, N, 2] (float32 or float64) through ``K`` ([3, 3] or
    [B, 3, 3]) and ``D`` ([4] or [B, 4]: k1, k2, k3, k4), as [B, N, 2] in the input's dtype, computed in double:
    ``cv2.fisheye.undistortPoints(kpts, K, D, P=K, criteria)`` (header step FE3).

    Newton on the field angle theta, at most ``max_iters`` steps (in [0, 1000]).  ``eps`` > 0 is OpenCV's EPS
    criterion in radians of theta (not pixels): a point converges once a step is below it, and one that does not
    converge gives a NaN row; ``eps`` = 0 is the COUNT-only criterion.  The defaults are OpenCV's (10, 1e-8).  A
    point whose theta changes sign gives a NaN row too, and so does the principal point with ``eps`` = 0 (OpenCV's
    0 / 0); where OpenCV writes (-1e6, -1e6) for a failed point, this writes NaN, which every estimator treats as an
    invalid match.  As in OpenCV, the distorted angle is clamped to pi/2: a pixel beyond the model's 180 degree field
    comes back at a plausible but wrong angle."""
    _check_criteria(max_iters, eps, "radians")
    return _camera("geo_fisheye_undistort_points", kpts, K, D, max_iters, eps, fisheye=True)


def fisheye_distort_points(kpts: torch.Tensor, K: torch.Tensor, D: torch.Tensor) -> torch.Tensor:
    """Fisheye pixels of the undistorted pixels ``kpts`` [B, N, 2]: ``cv2.fisheye.distortPoints`` of K^-1 [u, v, 1]
    through (K, D) with ``alpha = K[0, 1] / K[0, 0]`` (header step FE2).  Arguments as ``fisheye_undistort_points``."""
    return _camera("geo_fisheye_distort_points", kpts, K, D, 0, 0.0, fisheye=True)
