"""Geometric verification on the GPU: batched RANSAC homography and fundamental-matrix, relative-pose,
absolute-pose, affine and 3D rigid and similarity estimation on the matcher's output, each of the first four plain and
LO-RANSAC, and the first two MAGSAC++ as well (C ABI ``include/geometry_b200.h``, CUDA ``csrc/geo_api.cu``, ``csrc/lo_hf_api.cu``, ``csrc/pose_api.cu``,
``csrc/lo_pose_api.cu``, ``csrc/pnp_api.cu``, ``csrc/lo_pnp_api.cu``, ``csrc/affine_api.cu`` and
``csrc/rigid_api.cu``).

All fourteen functions take ``matches0`` [B, M] int64 exactly as ``LightGlue.forward``, ``PendingMatch.tensors`` and
``match_ragged`` give it (-1 or any index outside [0, N) is unmatched), run every pair of the batch in one call on the
current stream, and return device tensors of fixed shapes without synchronising with the host, so a call can follow a
matcher forward with no read-back in between, or be captured in a CUDA graph.  A match whose keypoint in either image,
or whose 3D point, has a NaN or infinite coordinate is invalid like an unmatched row: it is never an inlier and does
not count towards the pair's matches.  Parameter names and defaults are those of
``cv2.findHomography(RANSAC)``, ``cv2.findFundamentalMat(FM_RANSAC)``, ``cv2.findEssentialMat(RANSAC)`` with
``cv2.recoverPose``, ``cv2.solvePnPRansac``, and ``cv2.estimateAffine2D`` and ``cv2.estimateAffinePartial2D`` with
``method=cv2.RANSAC``.

``find_homography`` and ``find_fundamental`` return a dict: ``H`` or ``F`` [B, 3, 3] float64 (H scaled to H[2, 2] = 1; F to unit Frobenius norm with its largest
entry positive), ``inliers`` [B, M] bool, ``num_inliers`` [B] int32, ``success`` [B] bool, and the diagnostics
``best_hypothesis`` [B] int32 (-1 without one) and ``num_hypotheses`` [B] int32.  A failed pair (fewer valid matches than
the sample size, 4 or 8, or no non-degenerate hypothesis) has ``success`` False, a zero model and no inliers.
``find_homography_lo`` and ``find_fundamental_lo`` return the keys of ``find_homography`` and ``find_fundamental`` plus
``num_local_optimizations`` and ``cost``; so do ``find_homography_magsac`` and ``find_fundamental_magsac`` (MAGSAC++,
``cv2.USAC_MAGSAC``), and ``estimate_relative_pose_lo`` and ``estimate_absolute_pose_lo`` with
those of ``estimate_relative_pose`` and ``estimate_absolute_pose``.  ``estimate_affine_2d`` and
``estimate_affine_partial_2d`` return those of ``find_homography`` with ``A`` [B, 2, 3] in place of ``H``.
``estimate_rigid_3d`` and ``estimate_similarity_3d`` register matched 3D points (``cv2.estimateAffine3D`` with
``force_rotation=True`` fits the same model without RANSAC) and return ``R``, ``t`` and ``scale`` in place of ``H``.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _cabi
from .camera import check_fisheye_count, dist_coeffs


def _check_params(threshold, max_iters, confidence, seed, name="ransac_reproj_threshold",
                  what="a positive number of pixels") -> None:
    if not isinstance(max_iters, int) or isinstance(max_iters, bool) or not 1 <= max_iters <= 1 << 24:
        raise ValueError(f"max_iters={max_iters!r}: an int in [1, 2**24]")
    if not float(threshold) > 0.0 or float(threshold) == float("inf"):
        raise ValueError(f"{name}={threshold!r}: {what}")
    if not 0.0 <= float(confidence) <= 1.0:
        raise ValueError(f"confidence={confidence!r}: in [0, 1]")
    if not isinstance(seed, int) or isinstance(seed, bool) or not 0 <= seed < 1 << 32:
        raise ValueError(f"seed={seed!r}: an int in [0, 2**32)")


def _check_inputs(kpts0, kpts1, matches0, name1="kpts1", dim1=2, name0="kpts0", dim0=2) -> None:
    for name, t in ((name0, kpts0), (name1, kpts1), ("matches0", matches0)):
        if not isinstance(t, torch.Tensor):
            raise ValueError(f"{name} must be a torch.Tensor")
        if t.device.type != "cuda":
            raise RuntimeError("lightglue_b200.geometry runs on CUDA (sm_90a) tensors only; there is no CPU path")
    if kpts0.dim() != 3 or kpts0.shape[-1] != dim0 or kpts1.dim() != 3 or kpts1.shape[-1] != dim1:
        raise ValueError(f"{name0} {tuple(kpts0.shape)} and {name1} {tuple(kpts1.shape)}: expected [B, M, {dim0}] and "
                         f"[B, N, {dim1}]")
    if matches0.dim() != 2 or matches0.shape != kpts0.shape[:2] or kpts1.shape[0] != kpts0.shape[0]:
        raise ValueError(f"matches0 {tuple(matches0.shape)}: expected [B, M] of {name0} {tuple(kpts0.shape)} with the "
                         f"batch of {name1} {tuple(kpts1.shape)}")
    if not kpts0.is_floating_point() or not kpts1.is_floating_point():
        raise ValueError(f"{name0} and {name1} must be floating point" + (" pixels" if dim1 == 2 else ""))
    if matches0.dtype != torch.int64:
        raise ValueError(f"matches0 must be int64, not {matches0.dtype}")
    if kpts1.device != kpts0.device or matches0.device != kpts0.device:
        raise ValueError(f"{name0}, {name1} and matches0 must be on one device")


def _run(entry: str, ws_entry: str, shapes: dict, device, b: int, m: int, max_iters: int, make_args) -> dict:
    """Allocates the outputs of ``shapes`` (key -> (shape, dtype)) and, unless the batch is empty, a workspace of
    ``ws_entry``'s size, then calls ``entry`` on the ctypes structs ``make_args(out)`` returns."""
    out = {k: torch.empty(*shape, dtype=dtype, device=device) for k, (shape, dtype) in shapes.items()}
    if b == 0:
        return out
    with torch.cuda.device(device):
        lib = _cabi.load()
        ws = torch.empty(getattr(lib, ws_entry)(b, m, max_iters), dtype=torch.uint8, device=device)
        cfg, ins, outs = make_args(out)
        _cabi.check(getattr(lib, entry)(C.byref(cfg), C.byref(ins), C.byref(outs), ws.data_ptr(), ws.numel(),
                                        torch.cuda.current_stream(device).cuda_stream), entry)
    return out


def _estimate(kind: int, key: str, kpts0, kpts1, matches0, threshold, max_iters, confidence, seed,
              lo: bool = False, max_threshold=None) -> dict:
    """Plain RANSAC, LO-RANSAC (lo) or MAGSAC++ (lo and a max_threshold)."""
    _check_inputs(kpts0, kpts1, matches0)
    _check_params(threshold, max_iters, confidence, seed)
    if max_threshold is not None:
        _check_params(max_threshold, max_iters, confidence, seed, "max_threshold", "a positive finite number of pixels")
    if lo and kpts0.shape[1] > _cabi.GEO_LO_MAX_MATCHES:
        raise ValueError(f"kpts0 {tuple(kpts0.shape)}: at most {_cabi.GEO_LO_MAX_MATCHES} rows per pair")
    device = kpts0.device
    b, m, n = kpts0.shape[0], kpts0.shape[1], kpts1.shape[1]
    k0 = kpts0.detach().to(torch.float32).contiguous()
    k1 = kpts1.detach().to(torch.float32).contiguous()
    m0 = matches0.detach().contiguous()
    f64, i32, bl = torch.float64, torch.int32, torch.bool
    shapes = {key: ((b, 3, 3), f64), "inliers": ((b, m), bl), "num_inliers": ((b,), i32), "success": ((b,), bl),
              "best_hypothesis": ((b,), i32), "num_hypotheses": ((b,), i32)}
    if lo:
        shapes.update(num_local_optimizations=((b,), i32), cost=((b,), torch.int64))

    def make_args(out):
        cfg = _cabi.GeoConfig(_cabi.GEO_ABI_VERSION, kind, max_iters, seed, float(threshold), float(confidence))
        if max_threshold is not None:
            cfg = _cabi.GeoMagsacConfig(cfg, float(max_threshold))
        ins = _cabi.GeoInputs(b, m, n, k0.data_ptr(), k1.data_ptr(), m0.data_ptr())
        outs = _cabi.GeoOutputs(*(out[k].data_ptr() for k in list(shapes)[:6]))
        if lo:
            outs = _cabi.GeoLoOutputs(outs, out["num_local_optimizations"].data_ptr(), out["cost"].data_ptr())
        return cfg, ins, outs

    if not lo:
        return _run("geo_estimate", "geo_workspace_bytes", shapes, device, b, m, max_iters, make_args)
    name = "homography" if kind == _cabi.GEO_HOMOGRAPHY else "fundamental"
    entry = f"geo_{name}_lo" if max_threshold is None else f"geo_{name}_magsac"
    return _run(entry, f"geo_lo_{name}_workspace_bytes", shapes, device, b, m, max_iters, make_args)


def find_homography(kpts0: torch.Tensor, kpts1: torch.Tensor, matches0: torch.Tensor, ransac_reproj_threshold: float = 3.0,
                    max_iters: int = 2000, confidence: float = 0.995, seed: int = 0) -> dict:
    """RANSAC homography per pair, mapping kpts0 to kpts1: an inlier has a squared forward transfer error below
    ``ransac_reproj_threshold ** 2``.  Defaults of ``cv2.findHomography(method=cv2.RANSAC)``."""
    return _estimate(_cabi.GEO_HOMOGRAPHY, "H", kpts0, kpts1, matches0, ransac_reproj_threshold, max_iters, confidence,
                     seed)


def find_homography_lo(kpts0: torch.Tensor, kpts1: torch.Tensor, matches0: torch.Tensor,
                       ransac_reproj_threshold: float = 3.0, max_iters: int = 2000, confidence: float = 0.995,
                       seed: int = 0) -> dict:
    """LO-RANSAC homography per pair: the samples and four-point hypotheses of ``find_homography``, scored by a
    truncated (MSAC) transfer cost, with Levenberg-Marquardt local optimisation of H after each chunk of 256 samples
    that improves the best model, and a final Levenberg-Marquardt refinement.  The accuracy of PoseLib's and OpenCV's
    USAC LO-RANSAC, on the GPU; ``find_homography`` stays the one that follows ``cv2.RANSAC``.  Arguments and defaults
    are ``find_homography``'s, so the two compare like for like; at most 2**20 - 1 rows of ``matches0`` per pair.

    Returns the keys of ``find_homography`` (``H`` the final model with H[2, 2] = 1; ``inliers`` the points within the
    threshold of that H; ``best_hypothesis`` the sample the final model grew from) plus ``num_local_optimizations``
    [B] int32, the local optimisations whose model was adopted, and ``cost`` [B] int64, the final model's integer MSAC
    score.  Failures are those of ``find_homography``, with ``num_local_optimizations`` and ``cost`` 0."""
    return _estimate(_cabi.GEO_HOMOGRAPHY, "H", kpts0, kpts1, matches0, ransac_reproj_threshold, max_iters, confidence,
                     seed, lo=True)


def find_fundamental(kpts0: torch.Tensor, kpts1: torch.Tensor, matches0: torch.Tensor, ransac_reproj_threshold: float = 3.0,
                     max_iters: int = 1000, confidence: float = 0.99, seed: int = 0) -> dict:
    """RANSAC fundamental matrix per pair (x1^T F x0 = 0) by the normalised 8-point method: an inlier's larger distance
    to its two epipolar lines is below ``ransac_reproj_threshold``.  Defaults of
    ``cv2.findFundamentalMat(method=cv2.FM_RANSAC)``."""
    return _estimate(_cabi.GEO_FUNDAMENTAL, "F", kpts0, kpts1, matches0, ransac_reproj_threshold, max_iters, confidence,
                     seed)


def find_fundamental_lo(kpts0: torch.Tensor, kpts1: torch.Tensor, matches0: torch.Tensor,
                        ransac_reproj_threshold: float = 3.0, max_iters: int = 1000, confidence: float = 0.99,
                        seed: int = 0) -> dict:
    """LO-RANSAC fundamental matrix per pair: the samples and eight-point hypotheses of ``find_fundamental``, scored by
    a truncated (MSAC) epipolar-distance cost, with Levenberg-Marquardt local optimisation of a rank-2 F on the Sampson
    error after each chunk of 256 samples that improves the best model, and a final Levenberg-Marquardt refinement.
    The accuracy of PoseLib's and OpenCV's USAC LO-RANSAC, on the GPU; ``find_fundamental`` stays the one that follows
    ``cv2.FM_RANSAC``.  Arguments and defaults are ``find_fundamental``'s, so the two compare like for like; at most
    2**20 - 1 rows of ``matches0`` per pair.

    Returns the keys of ``find_fundamental`` (``F`` the final model: rank 2, unit Frobenius norm, largest entry
    positive; ``inliers`` the points whose larger distance to their two epipolar lines under that F is below the
    threshold; ``best_hypothesis`` the sample the final model grew from) plus ``num_local_optimizations`` [B] int32, the
    local optimisations whose model was adopted, and ``cost`` [B] int64, the final model's integer MSAC score.
    Failures are those of ``find_fundamental``, with ``num_local_optimizations`` and ``cost`` 0."""
    return _estimate(_cabi.GEO_FUNDAMENTAL, "F", kpts0, kpts1, matches0, ransac_reproj_threshold, max_iters, confidence,
                     seed, lo=True)


def find_homography_magsac(kpts0: torch.Tensor, kpts1: torch.Tensor, matches0: torch.Tensor,
                           ransac_reproj_threshold: float = 3.0, max_threshold: float = 7.5, max_iters: int = 2000,
                           confidence: float = 0.995, seed: int = 0) -> dict:
    """MAGSAC++ homography per pair (Barath et al., CVPR 2020; ``cv2.USAC_MAGSAC``): the samples and four-point
    hypotheses of ``find_homography_lo``, scored by the MAGSAC++ loss marginalised over the noise scale, with local
    optimisation by Levenberg-Marquardt reweighted by the same marginalisation, on the schedule of
    ``find_homography_lo``.  Returns the keys of ``find_homography_lo``, ``cost`` being the final model's integer
    MAGSAC++ score; failures are those of ``find_homography_lo``.

    ``ransac_reproj_threshold`` keeps its meaning from every other estimator here: it sets ``inliers``,
    ``num_inliers`` and the inlier count that drives the adaptive stop.  ``max_threshold`` is new: T = k * sigma_max
    (k = 3.64, the square root of the 0.99 quantile of chi-square with 4 degrees of freedom) is the scale of the loss
    and the weights, so a point whose error is T or more costs as an outlier and has weight 0.  The default of 7.5 px
    follows OpenCV's USAC_MAGSAC, whose accuracy does not move with the user's threshold.  Neither does this one's: on
    the synthetic scenes of tests/test_magsac_oracle.py the model is the same at every user threshold from 1 to 6 px,
    and the median homography error moves by 1.5x over T from 5 to 15 px (lower at larger T under 1.5 px of noise).
    At most 2**20 - 1 rows of ``matches0`` per pair."""
    return _estimate(_cabi.GEO_HOMOGRAPHY, "H", kpts0, kpts1, matches0, ransac_reproj_threshold, max_iters, confidence,
                     seed, lo=True, max_threshold=max_threshold)


def find_fundamental_magsac(kpts0: torch.Tensor, kpts1: torch.Tensor, matches0: torch.Tensor,
                            ransac_reproj_threshold: float = 3.0, max_threshold: float = 7.5, max_iters: int = 1000,
                            confidence: float = 0.99, seed: int = 0) -> dict:
    """MAGSAC++ fundamental matrix per pair (``cv2.USAC_MAGSAC``): the samples and eight-point hypotheses of
    ``find_fundamental_lo``, scored by the MAGSAC++ loss of the epipolar distance, with local optimisation of a rank-2
    F by Levenberg-Marquardt on the Sampson error reweighted by the same marginalisation, on the schedule of
    ``find_fundamental_lo``.  Returns the keys of ``find_fundamental_lo``, ``cost`` being the final model's integer
    MAGSAC++ score; failures are those of ``find_fundamental_lo``.

    ``ransac_reproj_threshold`` keeps its meaning from every other estimator here: it sets ``inliers``,
    ``num_inliers`` and the inlier count that drives the adaptive stop.  ``max_threshold`` is new: T = k * sigma_max
    (k = 3.64, the square root of the 0.99 quantile of chi-square with 4 degrees of freedom) is the scale of the loss
    and the weights, so a point whose error is T or more costs as an outlier and has weight 0.  The default of 7.5 px
    follows OpenCV's USAC_MAGSAC, whose accuracy does not move with the user's threshold.  Neither does this one's: on
    the synthetic scenes of tests/test_magsac_oracle.py the model is the same at every user threshold from 1 to 6 px,
    and the median homography error moves by 1.5x over T from 5 to 15 px (lower at larger T under 1.5 px of noise).
    At most 2**20 - 1 rows of ``matches0`` per pair."""
    return _estimate(_cabi.GEO_FUNDAMENTAL, "F", kpts0, kpts1, matches0, ransac_reproj_threshold, max_iters, confidence,
                     seed, lo=True, max_threshold=max_threshold)


def _intrinsics(name: str, K, b: int, device) -> torch.Tensor:
    if not isinstance(K, torch.Tensor):
        raise ValueError(f"{name} must be a torch.Tensor")
    if K.device.type != "cuda":
        raise RuntimeError("lightglue_b200.geometry runs on CUDA (sm_90a) tensors only; there is no CPU path")
    if not K.is_floating_point():
        raise ValueError(f"{name} must be floating point")
    if K.shape == (3, 3):
        K = K.expand(b, 3, 3)
    elif K.dim() != 3 or K.shape != (b, 3, 3):
        raise ValueError(f"{name} {tuple(K.shape)}: expected [3, 3] or [B, 3, 3] with B = {b}")
    if K.device != device:
        raise ValueError(f"{name} must be on the device of kpts0")
    return K.detach().to(torch.float64).contiguous()


def estimate_relative_pose(kpts0: torch.Tensor, kpts1: torch.Tensor, matches0: torch.Tensor, K0: torch.Tensor,
                           K1: torch.Tensor | None = None, ransac_reproj_threshold: float = 1.0, max_iters: int = 1000,
                           confidence: float = 0.999, distance_threshold: float = 50.0, seed: int = 0) -> dict:
    """Relative pose per pair: a five-point RANSAC essential matrix on calibrated coordinates, then the (R, t) of
    ``cv2.recoverPose`` by its cheirality test.  ``K0`` and ``K1`` are [3, 3] or [B, 3, 3] (``K1=None``: K0); the pixel
    threshold is divided by the pair's mean focal length (fx0 + fy0 + fx1 + fy1) / 4.  Defaults of
    ``cv2.findEssentialMat(method=cv2.RANSAC)`` and ``cv2.recoverPose``.

    Returns ``E``, ``R`` [B, 3, 3] and ``t`` [B, 3] float64 with x1 = R x0 + t, |t| = 1 and E of unit Frobenius norm
    with its largest entry positive; ``inliers`` [B, M] bool and ``num_inliers`` [B] int32 of the RANSAC;
    ``pose_inliers`` and ``num_pose_inliers``, the inliers that pass the chosen pose's cheirality test; ``success``
    [B] bool; and the diagnostics ``best_hypothesis``, ``best_solution`` and ``num_hypotheses`` [B] int32.  A pair
    with fewer than 5 valid matches, an invalid K (a non-finite entry, fx or fy <= 0, or a bottom row other than
    [0, 0, 1]) or no non-degenerate sample has ``success`` False, zero E, R and t, and no inliers."""
    return _relative_pose(False, kpts0, kpts1, matches0, K0, K1, ransac_reproj_threshold, max_iters, confidence,
                          distance_threshold, seed)


def estimate_relative_pose_lo(kpts0: torch.Tensor, kpts1: torch.Tensor, matches0: torch.Tensor, K0: torch.Tensor,
                              K1: torch.Tensor | None = None, ransac_reproj_threshold: float = 1.0, max_iters: int = 1000,
                              confidence: float = 0.999, distance_threshold: float = 50.0, seed: int = 0) -> dict:
    """LO-RANSAC relative pose per pair: the samples and five-point solutions of ``estimate_relative_pose``, scored by
    a truncated (MSAC) Sampson cost, with Levenberg-Marquardt local optimisation of (R, t) after each chunk of 256
    samples that improves the best model, and a final Levenberg-Marquardt refinement.  The accuracy of PoseLib's and
    OpenCV's USAC LO-RANSAC, on the GPU; ``estimate_relative_pose`` stays the one that follows ``cv2.RANSAC``.
    Arguments and defaults are ``estimate_relative_pose``'s, so the two compare like for like; at most 2**20 - 1 rows of
    ``matches0`` per pair.

    Returns the keys of ``estimate_relative_pose`` (E = [t]x R of the final pose, unit Frobenius norm with its largest
    entry positive; ``inliers`` the points within the threshold of that E; ``best_hypothesis`` and ``best_solution``
    the five-point solution the final model grew from) plus ``num_local_optimizations`` [B] int32, the local
    optimisations whose model was adopted, and ``cost`` [B] int64, the final model's integer MSAC score.  Failures are
    those of ``estimate_relative_pose``, with ``num_local_optimizations`` and ``cost`` 0."""
    return _relative_pose(True, kpts0, kpts1, matches0, K0, K1, ransac_reproj_threshold, max_iters, confidence,
                          distance_threshold, seed)


def _relative_pose(lo: bool, kpts0, kpts1, matches0, K0, K1, ransac_reproj_threshold, max_iters, confidence,
                   distance_threshold, seed) -> dict:
    _check_inputs(kpts0, kpts1, matches0)
    _check_params(ransac_reproj_threshold, max_iters, confidence, seed)
    if not float(distance_threshold) > 0.0 or float(distance_threshold) == float("inf"):
        raise ValueError(f"distance_threshold={distance_threshold!r}: a positive number")
    if lo and kpts0.shape[1] > _cabi.GEO_LO_MAX_MATCHES:
        raise ValueError(f"kpts0 {tuple(kpts0.shape)}: at most {_cabi.GEO_LO_MAX_MATCHES} rows per pair")
    device = kpts0.device
    b, m, n = kpts0.shape[0], kpts0.shape[1], kpts1.shape[1]
    k0 = _intrinsics("K0", K0, b, device)
    k1 = k0 if K1 is None else _intrinsics("K1", K1, b, device)
    p0 = kpts0.detach().to(torch.float32).contiguous()
    p1 = kpts1.detach().to(torch.float32).contiguous()
    m0 = matches0.detach().contiguous()
    f64, i32, bl = torch.float64, torch.int32, torch.bool
    shapes = {"E": ((b, 3, 3), f64), "R": ((b, 3, 3), f64), "t": ((b, 3), f64), "inliers": ((b, m), bl),
              "num_inliers": ((b,), i32), "pose_inliers": ((b, m), bl), "num_pose_inliers": ((b,), i32),
              "success": ((b,), bl), "best_hypothesis": ((b,), i32), "best_solution": ((b,), i32),
              "num_hypotheses": ((b,), i32)}
    if lo:
        shapes.update(num_local_optimizations=((b,), i32), cost=((b,), torch.int64))

    def make_args(out):
        args = (max_iters, seed, 0, float(ransac_reproj_threshold), float(confidence), float(distance_threshold))
        ins = _cabi.GeoPoseInputs(b, m, n, p0.data_ptr(), p1.data_ptr(), m0.data_ptr(), k0.data_ptr(), k1.data_ptr())
        outs = _cabi.GeoPoseOutputs(*(out[k].data_ptr() for k in list(shapes)[:11]))
        if not lo:
            return _cabi.GeoPoseConfig(_cabi.GEO_ABI_VERSION, *args), ins, outs
        louts = _cabi.GeoLoPoseOutputs(outs, out["num_local_optimizations"].data_ptr(), out["cost"].data_ptr())
        return _cabi.GeoLoPoseConfig(_cabi.GEO_ABI_VERSION, *args), ins, louts

    if lo:
        return _run("geo_relative_pose_lo", "geo_lo_pose_workspace_bytes", shapes, device, b, m, max_iters, make_args)
    return _run("geo_relative_pose", "geo_pose_workspace_bytes", shapes, device, b, m, max_iters, make_args)


def estimate_absolute_pose(kpts0: torch.Tensor, points3d1: torch.Tensor, matches0: torch.Tensor, K0: torch.Tensor,
                           ransac_reproj_threshold: float = 8.0, max_iters: int = 100, confidence: float = 0.99,
                           seed: int = 0, dist_coeffs0: torch.Tensor | None = None) -> dict:
    """Absolute pose per pair from 2D-3D matches: Lambda Twist P3P RANSAC on the query pixels ``kpts0`` [B, M, 2] and
    the world points ``points3d1`` [B, N, 3] of image 1's keypoints (a row with a non-finite coordinate has no 3D point,
    so its matches are invalid), then Levenberg-Marquardt on the inliers.  An inlier lies in front of the camera with a
    squared reprojection error through ``K0`` ([3, 3] or [B, 3, 3]; lens distortion: ``dist_coeffs0`` below) below
    ``ransac_reproj_threshold ** 2``.  Defaults of ``cv2.solvePnPRansac``.

    Returns ``R`` [B, 3, 3] and ``t`` [B, 3] float64 with x_cam = R X + t (OpenCV's rvec/tvec convention);
    ``inliers`` [B, M] bool and ``num_inliers`` [B] int32 of the final pose; ``success`` [B] bool; and the
    diagnostics ``best_hypothesis``, ``best_solution`` and ``num_hypotheses`` [B] int32.  A pair with fewer than 3
    valid matches, an invalid K0 (a non-finite entry, fx or fy <= 0, or a bottom row other than [0, 0, 1]) or no
    non-degenerate sample has ``success`` False, zero R and t, no inliers and -1 for ``best_hypothesis`` and
    ``best_solution``.

    ``dist_coeffs0`` ([k] or [B, k], k = 4, 5, 8 or 12; see ``lightglue_b200.camera``) gives the query camera's lens
    distortion, as ``cv2.solvePnPRansac(..., distCoeffs)`` takes it: the P3P samples see the pixels undistorted by
    OpenCV's 5 fixed-point iterations, and the inlier test and the refit measure the reprojection error in distorted
    pixels (header steps AD1-AD4).  A pair with a non-finite coefficient fails as one with an invalid K0.  A fisheye
    lens is ``estimate_absolute_pose_fisheye``'s."""
    return _absolute_pose(False, kpts0, points3d1, matches0, K0, ransac_reproj_threshold, max_iters, confidence, seed,
                          dist_coeffs0)


def estimate_absolute_pose_lo(kpts0: torch.Tensor, points3d1: torch.Tensor, matches0: torch.Tensor, K0: torch.Tensor,
                              ransac_reproj_threshold: float = 8.0, max_iters: int = 100, confidence: float = 0.99,
                              seed: int = 0, dist_coeffs0: torch.Tensor | None = None) -> dict:
    """LO-RANSAC absolute pose per pair: the samples and P3P solutions of ``estimate_absolute_pose``, scored by a
    truncated (MSAC) squared reprojection error, with Levenberg-Marquardt local optimisation of (R, t) after each chunk
    of 256 samples that improves the best model, and a final Levenberg-Marquardt refinement.  The accuracy of PoseLib's
    and OpenCV's USAC LO-RANSAC, on the GPU: a rotation-error tail close to USAC's where ``estimate_absolute_pose``'s
    one refit from one sample leaves outliers in the tail; ``estimate_absolute_pose`` stays the one that follows
    ``cv2.solvePnPRansac``.  Arguments and defaults are ``estimate_absolute_pose``'s, so the two compare like for like;
    at most 2**20 - 1 rows of ``matches0`` per pair.

    Returns the keys of ``estimate_absolute_pose`` (R and t the final pose; ``inliers`` the rows in front of the camera
    within the threshold of it; ``best_hypothesis`` and ``best_solution`` the P3P solution the final model grew from)
    plus ``num_local_optimizations`` [B] int32, the local optimisations whose model was adopted, and ``cost`` [B]
    int64, the final model's integer MSAC score.  Failures are those of ``estimate_absolute_pose``, with
    ``num_local_optimizations`` and ``cost`` 0.  ``dist_coeffs0`` is ``estimate_absolute_pose``'s: the MSAC score
    and the Levenberg-Marquardt steps then read the reprojection error in distorted pixels."""
    return _absolute_pose(True, kpts0, points3d1, matches0, K0, ransac_reproj_threshold, max_iters, confidence, seed,
                          dist_coeffs0)


def estimate_absolute_pose_fisheye(kpts0: torch.Tensor, points3d1: torch.Tensor, matches0: torch.Tensor,
                                   K0: torch.Tensor, D0: torch.Tensor, ransac_reproj_threshold: float = 8.0,
                                   max_iters: int = 100, confidence: float = 0.99, seed: int = 0) -> dict:
    """``estimate_absolute_pose`` for a query camera with a fisheye lens: ``K0`` and ``D0`` ([4] or [B, 4]: k1, k2,
    k3, k4, see ``lightglue_b200.camera``) as ``cv2.fisheye`` takes them (header steps AE1-AE4).  The P3P samples see
    the pixels undistorted as ``cv2.fisheye.undistortPoints`` does with its default criteria, and a match whose pixel
    does not undistort is invalid; the inlier test and the refit measure the reprojection error in fisheye pixels.
    ``cv2.fisheye.solvePnPRansac`` instead tests undistorted pinhole pixels, where a fixed threshold grows as
    1 / cos^2 of the field angle and drops true inliers toward the edge of a wide lens;
    ``camera.fisheye_undistort_points`` followed by ``estimate_absolute_pose`` reproduces that.  Arguments, outputs and
    failures are ``estimate_absolute_pose``'s; non-finite coefficients fail the pair as an invalid K0 does, and a
    ``D0`` that is None or does not hold exactly 4 coefficients per pair is a ``ValueError``.

    This is a function of its own, not a keyword of ``estimate_absolute_pose``, so that the signatures of
    ``estimate_absolute_pose`` and ``estimate_absolute_pose_lo`` stay as they were, ending at ``dist_coeffs0``."""
    return _absolute_pose(False, kpts0, points3d1, matches0, K0, ransac_reproj_threshold, max_iters, confidence, seed,
                          D0, fisheye=True)


def estimate_absolute_pose_lo_fisheye(kpts0: torch.Tensor, points3d1: torch.Tensor, matches0: torch.Tensor,
                                      K0: torch.Tensor, D0: torch.Tensor, ransac_reproj_threshold: float = 8.0,
                                      max_iters: int = 100, confidence: float = 0.99, seed: int = 0) -> dict:
    """``estimate_absolute_pose_lo`` for a query camera with a fisheye lens, as ``estimate_absolute_pose_fisheye``:
    the MSAC score and the Levenberg-Marquardt steps read the reprojection error in fisheye pixels."""
    return _absolute_pose(True, kpts0, points3d1, matches0, K0, ransac_reproj_threshold, max_iters, confidence, seed,
                          D0, fisheye=True)


def _absolute_pose(lo: bool, kpts0, points3d1, matches0, K0, ransac_reproj_threshold, max_iters, confidence,
                   seed, dist_coeffs0=None, fisheye: bool = False) -> dict:
    if fisheye:  # a fisheye pose never falls back to the pinhole or the rational lens
        check_fisheye_count("D0", dist_coeffs0)
    _check_inputs(kpts0, points3d1, matches0, "points3d1", 3)
    _check_params(ransac_reproj_threshold, max_iters, confidence, seed)
    if lo and kpts0.shape[1] > _cabi.GEO_LO_MAX_MATCHES:
        raise ValueError(f"kpts0 {tuple(kpts0.shape)}: at most {_cabi.GEO_LO_MAX_MATCHES} rows per pair")
    device = kpts0.device
    b, m, n = kpts0.shape[0], kpts0.shape[1], points3d1.shape[1]
    k0 = _intrinsics("K0", K0, b, device)
    d0 = None if dist_coeffs0 is None else dist_coeffs("D0" if fisheye else "dist_coeffs0", dist_coeffs0, b, device,
                                                       fisheye)
    p0 = kpts0.detach().to(torch.float32).contiguous()
    x1 = points3d1.detach().to(torch.float32).contiguous()
    m0 = matches0.detach().contiguous()
    f64, i32, bl = torch.float64, torch.int32, torch.bool
    shapes = {"R": ((b, 3, 3), f64), "t": ((b, 3), f64), "inliers": ((b, m), bl), "num_inliers": ((b,), i32),
              "success": ((b,), bl), "best_hypothesis": ((b,), i32), "best_solution": ((b,), i32),
              "num_hypotheses": ((b,), i32)}
    if lo:
        shapes.update(num_local_optimizations=((b,), i32), cost=((b,), torch.int64))

    def make_args(out):
        cfg = _cabi.GeoPnpConfig(_cabi.GEO_ABI_VERSION, max_iters, seed, 0, float(ransac_reproj_threshold),
                                 float(confidence))
        ins = _cabi.GeoPnpInputs(b, m, n, p0.data_ptr(), x1.data_ptr(), m0.data_ptr(), k0.data_ptr())
        if d0 is not None:
            ins = _cabi.GeoPnpDistInputs(ins, d0.shape[1], d0.data_ptr())
        outs = _cabi.GeoPnpOutputs(*(out[k].data_ptr() for k in list(shapes)[:8]))
        if lo:
            outs = _cabi.GeoLoPnpOutputs(outs, out["num_local_optimizations"].data_ptr(), out["cost"].data_ptr())
        return cfg, ins, outs

    entry = "geo_absolute_pose_lo" if lo else "geo_absolute_pose"
    ws = "geo_lo_pnp_workspace_bytes" if lo else "geo_pnp_workspace_bytes"
    suffix = "" if d0 is None else "_fisheye" if fisheye else "_dist"
    return _run(entry + suffix, ws, shapes, device, b, m, max_iters, make_args)


def _affine(kind: int, kpts0, kpts1, matches0, threshold, max_iters, confidence, refine_iters, seed) -> dict:
    _check_inputs(kpts0, kpts1, matches0)
    _check_params(threshold, max_iters, confidence, seed)
    if (not isinstance(refine_iters, int) or isinstance(refine_iters, bool)
            or not 0 <= refine_iters <= _cabi.GEO_AFFINE_MAX_REFINE):
        raise ValueError(f"refine_iters={refine_iters!r}: an int in [0, {_cabi.GEO_AFFINE_MAX_REFINE}]")
    device = kpts0.device
    b, m, n = kpts0.shape[0], kpts0.shape[1], kpts1.shape[1]
    k0 = kpts0.detach().to(torch.float32).contiguous()
    k1 = kpts1.detach().to(torch.float32).contiguous()
    m0 = matches0.detach().contiguous()
    i32, bl = torch.int32, torch.bool
    shapes = {"model": ((b, 3, 3), torch.float64), "inliers": ((b, m), bl), "num_inliers": ((b,), i32),
              "success": ((b,), bl), "best_hypothesis": ((b,), i32), "num_hypotheses": ((b,), i32)}

    def make_args(out):
        cfg = _cabi.GeoAffineConfig(_cabi.GEO_ABI_VERSION, kind, max_iters, seed, refine_iters, 0, float(threshold),
                                    float(confidence))
        ins = _cabi.GeoInputs(b, m, n, k0.data_ptr(), k1.data_ptr(), m0.data_ptr())
        return cfg, ins, _cabi.GeoOutputs(*(out[k].data_ptr() for k in shapes))

    out = _run("geo_estimate_affine", "geo_affine_workspace_bytes", shapes, device, b, m, max_iters, make_args)
    return {"A": out.pop("model")[:, :2].contiguous(), **out}


def estimate_affine_2d(kpts0: torch.Tensor, kpts1: torch.Tensor, matches0: torch.Tensor,
                       ransac_reproj_threshold: float = 3.0, max_iters: int = 2000, confidence: float = 0.99,
                       refine_iters: int = 10, seed: int = 0) -> dict:
    """RANSAC affine transform per pair (6 degrees of freedom) from 3-point samples, mapping kpts0 to kpts1, then
    ``refine_iters`` Levenberg-Marquardt steps on the best sample's inliers (0: none): an inlier has a squared transfer
    error below ``ransac_reproj_threshold ** 2``.  Defaults of ``cv2.estimateAffine2D(method=cv2.RANSAC)``.

    Returns ``A`` [B, 2, 3] float64 (OpenCV's layout: x1 = A [x0, y0, 1]^T); ``inliers`` [B, M] bool and
    ``num_inliers`` [B] int32 of the final A (OpenCV returns the minimal sample's mask); ``success`` [B] bool; and the
    diagnostics ``best_hypothesis`` [B] int32 (-1 without one) and ``num_hypotheses`` [B] int32.  A pair with fewer
    than 3 valid matches, a failed normalisation or only degenerate (collinear) samples has ``success`` False, a zero
    A and no inliers.  ``torch.cat([A, row], 1)`` with ``row = [[0, 0, 1]]`` is a homography whose transfer error, as
    ``find_homography`` and ``NearestNeighborMatcher(...)(data, H=...)`` test it, equals this inlier test bit for
    bit."""
    return _affine(_cabi.GEO_AFFINE, kpts0, kpts1, matches0, ransac_reproj_threshold, max_iters, confidence,
                   refine_iters, seed)


def estimate_affine_partial_2d(kpts0: torch.Tensor, kpts1: torch.Tensor, matches0: torch.Tensor,
                               ransac_reproj_threshold: float = 3.0, max_iters: int = 2000, confidence: float = 0.99,
                               refine_iters: int = 10, seed: int = 0) -> dict:
    """RANSAC similarity transform per pair (rotation, uniform scale and translation: 4 degrees of freedom) from
    2-point samples, then ``refine_iters`` Levenberg-Marquardt steps on the best sample's inliers.  Defaults of
    ``cv2.estimateAffinePartial2D(method=cv2.RANSAC)``.

    Returns the keys of ``estimate_affine_2d``, with ``A`` exactly [[a, -b, tx], [b, a, ty]]: ``A[:, 0, 0]`` equals
    ``A[:, 1, 1]`` and ``A[:, 0, 1]`` equals ``-A[:, 1, 0]`` bit for bit.  A pair with fewer than 2 valid matches or
    only degenerate samples (coincident points in either image) fails as in ``estimate_affine_2d``."""
    return _affine(_cabi.GEO_AFFINE_PARTIAL, kpts0, kpts1, matches0, ransac_reproj_threshold, max_iters, confidence,
                   refine_iters, seed)


def _rigid(kind: int, points0, points1, matches0, threshold, max_iters, confidence, seed) -> dict:
    _check_inputs(points0, points1, matches0, "points1", 3, "points0", 3)
    _check_params(threshold, max_iters, confidence, seed, "ransac_threshold", "a positive distance in points1's units")
    device = points0.device
    b, m, n = points0.shape[0], points0.shape[1], points1.shape[1]
    p0 = points0.detach().to(torch.float32).contiguous()
    p1 = points1.detach().to(torch.float32).contiguous()
    m0 = matches0.detach().contiguous()
    f64, i32, bl = torch.float64, torch.int32, torch.bool
    shapes = {"R": ((b, 3, 3), f64), "t": ((b, 3), f64), "scale": ((b,), f64), "inliers": ((b, m), bl),
              "num_inliers": ((b,), i32), "success": ((b,), bl), "best_hypothesis": ((b,), i32),
              "num_hypotheses": ((b,), i32)}

    def make_args(out):
        cfg = _cabi.GeoConfig(_cabi.GEO_ABI_VERSION, kind, max_iters, seed, float(threshold), float(confidence))
        ins = _cabi.GeoInputs(b, m, n, p0.data_ptr(), p1.data_ptr(), m0.data_ptr())
        return cfg, ins, _cabi.GeoRigidOutputs(*(out[k].data_ptr() for k in shapes))

    return _run("geo_estimate_rigid", "geo_rigid_workspace_bytes", shapes, device, b, m, max_iters, make_args)


def estimate_rigid_3d(points0: torch.Tensor, points1: torch.Tensor, matches0: torch.Tensor, ransac_threshold: float,
                      max_iters: int = 1000, confidence: float = 0.99, seed: int = 0) -> dict:
    """RANSAC rigid transform (SE(3)) per pair between matched 3D points: x1 = R x0 + t from 3-point samples by Horn's
    closed-form quaternion method, then the same closed form (the least-squares Kabsch fit) on the best sample's
    inliers.  ``points0`` [B, M, 3] and ``points1`` [B, N, 3] are floating point, read as float32; a point with a
    non-finite coordinate (NaN for a missing depth) makes its matches invalid.  An inlier's squared distance
    |R x0 + t - x1|^2 is below ``ransac_threshold ** 2``, in the units of ``points1``; there is no default, since no
    single value fits both metres and millimetres.  ``max_iters`` and ``confidence`` default to those of
    ``cv2.estimateAffine3D``.

    Returns ``R`` [B, 3, 3] float64, a proper rotation; ``t`` [B, 3] float64; ``scale`` [B] float64, exactly 1.0 on
    success; ``inliers`` [B, M] bool and ``num_inliers`` [B] int32 of the final transform; ``success`` [B] bool; and
    the diagnostics ``best_hypothesis`` [B] int32 (-1 without one) and ``num_hypotheses`` [B] int32.  A pair with
    fewer than 3 valid matches or only degenerate (collinear or coincident) samples has ``success`` False, zero R, t
    and scale, and no inliers."""
    return _rigid(_cabi.GEO_RIGID_3D, points0, points1, matches0, ransac_threshold, max_iters, confidence, seed)


def estimate_similarity_3d(points0: torch.Tensor, points1: torch.Tensor, matches0: torch.Tensor,
                           ransac_threshold: float, max_iters: int = 1000, confidence: float = 0.99,
                           seed: int = 0) -> dict:
    """RANSAC similarity transform (Sim(3)) per pair between matched 3D points: x1 = scale R x0 + t, with Umeyama's
    least-squares scale, for maps or reconstructions that each have their own scale.  Arguments, outputs and failures
    are those of ``estimate_rigid_3d``, with ``scale`` > 0 free; ``ransac_threshold`` is measured in the frame of
    ``points1``.  On a fixed inlier set the fit equals ``cv2.estimateAffine3D(src, dst, force_rotation=True)``."""
    return _rigid(_cabi.GEO_SIMILARITY_3D, points0, points1, matches0, ransac_threshold, max_iters, confidence, seed)
