"""The fisheye camera without a GPU: the header's new exports and constants, the struct layouts they reuse, and the
argument checks of lightglue_b200.camera's fisheye functions, of the fisheye absolute pose and of their C entry points
(include/geometry_b200.h, steps FE1-FE4 and AE1-AE4)."""
import ctypes
import inspect
import os
import re

import pytest
import torch

from lightglue_b200 import _cabi
from lightglue_b200.camera import dist_coeffs, fisheye_distort_points, fisheye_undistort_points
from lightglue_b200.geometry import estimate_absolute_pose_fisheye, estimate_absolute_pose_lo_fisheye

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("geo_fisheye_undistort_points", "geo_fisheye_distort_points", "geo_absolute_pose_fisheye",
       "geo_absolute_pose_lo_fisheye")


def _header():
    with open(os.path.join(ROOT, "include", "geometry_b200.h")) as f:
        return f.read()


def test_entry_points_are_exported():
    assert set(NEW) <= set(_cabi.GEO_EXPORTS)
    lib = _cabi.load()
    for s in NEW:
        assert getattr(lib, s).argtypes is not None, s
        assert f"LG_API int {s}(" in _header(), s


def test_constants_match_the_header():
    h = _header()
    assert int(re.search(r"#define GEO_FISHEYE_ITERS (\S+)", h).group(1)) == _cabi.GEO_FISHEYE_ITERS == 10
    assert float(re.search(r"#define GEO_FISHEYE_EPS (\S+)", h).group(1)) == _cabi.GEO_FISHEYE_EPS == 1e-8
    assert re.search(r"#define GEO_ABI_VERSION (\S+)", h).group(1) == "1"


def test_struct_layouts_are_the_lens_distortion_ones():
    assert ctypes.sizeof(_cabi.GeoCameraConfig) == 24 and _cabi.GeoCameraConfig.eps.offset == 16
    assert ctypes.sizeof(_cabi.GeoCameraInputs) == 32 and ctypes.sizeof(_cabi.GeoPnpDistInputs) == 64


def test_defaults_are_opencvs():
    p = inspect.signature(fisheye_undistort_points).parameters
    assert (p["max_iters"].default, p["eps"].default) == (10, 1e-8)
    for f in (estimate_absolute_pose_fisheye, estimate_absolute_pose_lo_fisheye):
        p = inspect.signature(f).parameters
        assert list(p)[:5] == ["kpts0", "points3d1", "matches0", "K0", "D0"]
        assert (p["ransac_reproj_threshold"].default, p["max_iters"].default, p["confidence"].default) == (8.0, 100,
                                                                                                           0.99)


@pytest.mark.parametrize("k", [0, 1, 3, 5, 8, 12, 14])
def test_coefficient_counts_other_than_4_are_refused(k):
    with pytest.raises(ValueError, match="exactly 4"):
        dist_coeffs("D", torch.zeros(k), 2, None, fisheye=True)


@pytest.mark.parametrize("max_iters,eps", [(-1, 1e-8), (1001, 1e-8), (2.0, 1e-8), (True, 1e-8), (10, -1e-9),
                                           (10, float("inf")), (10, float("nan"))])
def test_max_iters_and_eps_bounds(max_iters, eps):
    with pytest.raises(ValueError):
        fisheye_undistort_points(torch.zeros(1, 2, 2), torch.eye(3), torch.zeros(4), max_iters=max_iters, eps=eps)


def test_keypoints_must_be_cuda():
    with pytest.raises(RuntimeError, match="CUDA"):
        fisheye_distort_points(torch.zeros(1, 2, 2), torch.eye(3), torch.zeros(4))
    with pytest.raises(RuntimeError, match="CUDA"):
        fisheye_undistort_points(torch.zeros(1, 2, 2), torch.eye(3), torch.zeros(4))


@pytest.mark.parametrize("D0", [None, torch.zeros(5), torch.zeros(12), torch.zeros(2, 5), torch.zeros(0)],
                         ids=["none", "5", "12", "2x5", "empty"])
@pytest.mark.parametrize("f", [estimate_absolute_pose_fisheye, estimate_absolute_pose_lo_fisheye],
                         ids=["plain", "lo"])
def test_pose_refuses_missing_or_wrong_coefficient_counts(f, D0):
    # refused before any keypoint or device check: never a silent pinhole or rational-lens run
    z = torch.zeros
    with pytest.raises(ValueError, match="not None" if D0 is None else "exactly 4"):
        f(z(2, 8, 2), z(2, 8, 3), z(2, 8, dtype=torch.int64), torch.eye(3), D0)
    with pytest.raises(TypeError):
        f(z(2, 8, 2), z(2, 8, 3), z(2, 8, dtype=torch.int64), torch.eye(3))  # D0 is required


def _cfg(nd=4, max_iters=10, dtype=0, eps=1e-8):
    return _cabi.GeoCameraConfig(_cabi.GEO_ABI_VERSION, nd, max_iters, dtype, eps)


def _err(rc):
    assert rc != 0
    return _cabi.load().lg_last_error().decode()


def test_c_abi_checks():
    lib = _cabi.load()
    ins = _cabi.GeoCameraInputs(1, 4, 1, 1, 1)
    outs = _cabi.GeoCameraOutputs(1)
    C = ctypes.byref
    for entry in ("geo_fisheye_undistort_points", "geo_fisheye_distort_points"):
        f = getattr(lib, entry)
        for nd in (5, 8, 12, 0):
            msg = _err(f(C(_cfg(nd=nd)), C(ins), C(outs), None))
            assert msg.startswith(entry) and "num_dist must be 4" in msg
        assert "null argument" in _err(f(None, C(ins), C(outs), None))
        assert "null input or output" in _err(f(C(_cfg()), C(_cabi.GeoCameraInputs(1, 4, 0, 1, 1)), C(outs), None))
        assert "null input or output" in _err(f(C(_cfg()), C(_cabi.GeoCameraInputs(1, 4, 1, 1, 0)), C(outs), None))
        assert f(C(_cfg()), C(_cabi.GeoCameraInputs(0, 4, 0, 0, 0)), C(outs), None) == 0
    u = lib.geo_fisheye_undistort_points
    assert "max_iters" in _err(u(C(_cfg(max_iters=-1)), C(ins), C(outs), None))
    assert "max_iters" in _err(u(C(_cfg(max_iters=1001)), C(ins), C(outs), None))
    for eps in (-1.0, float("inf"), float("nan")):
        assert "eps" in _err(u(C(_cfg(eps=eps)), C(ins), C(outs), None))
    cfg = _cabi.GeoPnpConfig(_cabi.GEO_ABI_VERSION, 100, 0, 0, 8.0, 0.99)
    pin = _cabi.GeoPnpInputs(1, 8, 8, 1, 1, 1, 1)
    for entry, out in (("geo_absolute_pose_fisheye", _cabi.GeoPnpOutputs(*[1] * 8)),
                       ("geo_absolute_pose_lo_fisheye",
                        _cabi.GeoLoPnpOutputs(_cabi.GeoPnpOutputs(*[1] * 8), 1, 1))):
        f = getattr(lib, entry)
        for nd in (5, 8, 12):
            msg = _err(f(C(cfg), C(_cabi.GeoPnpDistInputs(pin, nd, 1)), C(out), 1, 1 << 30, None))
            assert msg.startswith(entry) and "num_dist must be 4" in msg
        assert "null intrinsics" in _err(f(C(cfg), C(_cabi.GeoPnpDistInputs(pin, 4, 0)), C(out), 1, 1 << 30, None))
        assert "null argument" in _err(f(C(cfg), None, C(out), 1, 1 << 30, None))
