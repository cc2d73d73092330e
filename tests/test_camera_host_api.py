"""Lens distortion without a GPU: the header's new exports, constants and struct layouts, and the argument checks of
lightglue_b200.camera and of the distortion-aware absolute pose (include/geometry_b200.h, steps D1-D3 and AD1-AD4)."""
import ctypes
import inspect
import os
import re

import pytest
import torch

from lightglue_b200 import _cabi
from lightglue_b200.camera import dist_coeffs, distort_points, undistort_points
from lightglue_b200.geometry import estimate_absolute_pose, estimate_absolute_pose_lo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("geo_undistort_points", "geo_distort_points", "geo_absolute_pose_dist", "geo_absolute_pose_lo_dist")


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
    for name in ("GEO_CAMERA_FLOAT32", "GEO_CAMERA_FLOAT64", "GEO_UNDISTORT_MAX_ITERS"):
        value = getattr(_cabi, name)
        m = re.search(rf"#define {name} (\S+)", h)
        assert m and int(m.group(1)) == value, name


def test_struct_layouts():
    assert [f for f, _ in _cabi.GeoCameraConfig._fields_] == ["abi_version", "num_dist", "max_iters", "dtype", "eps"]
    assert _cabi.GeoCameraConfig.eps.offset == 16 and ctypes.sizeof(_cabi.GeoCameraConfig) == 24
    assert _cabi.GeoCameraInputs.pts.offset == 8 and _cabi.GeoCameraInputs.dist.offset == 24
    assert ctypes.sizeof(_cabi.GeoCameraInputs) == 32 and ctypes.sizeof(_cabi.GeoCameraOutputs) == 8
    # GeoPnpDistInputs embeds GeoPnpInputs unchanged, as GeoLoPnpOutputs embeds GeoPnpOutputs
    assert ctypes.sizeof(_cabi.GeoPnpInputs) == 48
    assert _cabi.GeoPnpDistInputs.num_dist.offset == 48 and _cabi.GeoPnpDistInputs.dist0.offset == 56
    assert ctypes.sizeof(_cabi.GeoPnpDistInputs) == 64


def test_defaults():
    p = inspect.signature(undistort_points).parameters
    assert (p["max_iters"].default, p["eps"].default) == (5, 0.0)
    for f in (estimate_absolute_pose, estimate_absolute_pose_lo):
        names = list(inspect.signature(f).parameters)
        assert names[-1] == "dist_coeffs0" and names[-2] == "seed"
        assert inspect.signature(f).parameters["dist_coeffs0"].default is None


@pytest.mark.parametrize("k", [0, 1, 3, 6, 7, 9, 13, 14, 15])
def test_coefficient_lengths_other_than_4_5_8_12_are_refused(k):
    with pytest.raises(ValueError, match="tilted" if k == 14 else "expected 4, 5, 8 or 12"):
        dist_coeffs("d", torch.zeros(k), 2, None)


def test_coefficient_shapes_and_dtypes():
    with pytest.raises(ValueError, match="torch.Tensor"):
        dist_coeffs("d", [0.0] * 4, 2, None)
    with pytest.raises(ValueError, match="floating point"):
        dist_coeffs("d", torch.zeros(4, dtype=torch.int64), 2, None)
    with pytest.raises(ValueError, match=r"\[k\] or \[B, k\]"):
        dist_coeffs("d", torch.zeros(3, 4), 2, None)
    with pytest.raises(ValueError, match=r"\[k\] or \[B, k\]"):
        dist_coeffs("d", torch.zeros(2, 2, 4), 2, None)
    with pytest.raises(RuntimeError, match="CUDA"):
        dist_coeffs("d", torch.zeros(4), 2, None)


@pytest.mark.parametrize("max_iters,eps", [(-1, 0.0), (1001, 0.0), (2.0, 0.0), (True, 0.0), (5, -1e-9),
                                           (5, float("inf")), (5, float("nan"))])
def test_max_iters_and_eps_bounds(max_iters, eps):
    with pytest.raises(ValueError):
        undistort_points(torch.zeros(1, 2, 2), torch.eye(3), torch.zeros(4), max_iters=max_iters, eps=eps)


def test_keypoints_must_be_cuda_float_b_n_2():
    with pytest.raises(RuntimeError, match="CUDA"):
        distort_points(torch.zeros(1, 2, 2), torch.eye(3), torch.zeros(4))
    with pytest.raises(ValueError, match="torch.Tensor"):
        distort_points([[0.0, 0.0]], torch.eye(3), torch.zeros(4))


def _cfg(nd=4, max_iters=5, dtype=0, eps=0.0):
    return _cabi.GeoCameraConfig(_cabi.GEO_ABI_VERSION, nd, max_iters, dtype, eps)


def _err(rc):
    assert rc != 0
    return _cabi.load().lg_last_error().decode()


def test_c_abi_checks():
    lib = _cabi.load()
    ins = _cabi.GeoCameraInputs(1, 4, 1, 1, 1)
    outs = _cabi.GeoCameraOutputs(1)
    C = ctypes.byref
    assert "num_dist" in _err(lib.geo_undistort_points(C(_cfg(nd=6)), C(ins), C(outs), None))
    assert "max_iters" in _err(lib.geo_undistort_points(C(_cfg(max_iters=1001)), C(ins), C(outs), None))
    assert "eps" in _err(lib.geo_undistort_points(C(_cfg(eps=-1.0)), C(ins), C(outs), None))
    assert "dtype" in _err(lib.geo_distort_points(C(_cfg(dtype=2)), C(ins), C(outs), None))
    bad = _cabi.GeoCameraConfig(_cabi.GEO_ABI_VERSION + 1, 4, 5, 0, 0.0)
    assert "ABI" in _err(lib.geo_distort_points(C(bad), C(ins), C(outs), None))
    assert lib.geo_undistort_points(C(_cfg()), C(_cabi.GeoCameraInputs(0, 4, 0, 0, 0)), C(outs), None) == 0
    cfg = _cabi.GeoPnpConfig(_cabi.GEO_ABI_VERSION, 100, 0, 0, 8.0, 0.99)
    pin = _cabi.GeoPnpInputs(1, 8, 8, 1, 1, 1, 1)
    for entry, out in (("geo_absolute_pose_dist", _cabi.GeoPnpOutputs(*[1] * 8)),
                       ("geo_absolute_pose_lo_dist", _cabi.GeoLoPnpOutputs(_cabi.GeoPnpOutputs(*[1] * 8), 1, 1))):
        f = getattr(lib, entry)
        msg = _err(f(C(cfg), C(_cabi.GeoPnpDistInputs(pin, 6, 1)), C(out), 1, 1 << 30, None))
        assert msg.startswith(entry) and "num_dist" in msg
        msg = _err(f(C(cfg), C(_cabi.GeoPnpDistInputs(pin, 8, 0)), C(out), 1, 1 << 30, None))
        assert "null intrinsics" in msg
        assert "null argument" in _err(f(C(cfg), None, C(out), 1, 1 << 30, None))
