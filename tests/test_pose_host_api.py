"""Relative pose without a GPU: the header's new exports, constants and struct layouts, argument checks and OpenCV's
defaults (include/geometry_b200.h, lightglue_b200/geometry.py)."""
import ctypes
import inspect
import os
import re

import pytest
import torch

from lightglue_b200 import _cabi
from lightglue_b200.geometry import estimate_relative_pose

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header():
    with open(os.path.join(ROOT, "include", "geometry_b200.h")) as f:
        return f.read()


def test_pose_entry_points_are_exported():
    assert {"geo_pose_workspace_bytes", "geo_relative_pose"} <= set(_cabi.GEO_EXPORTS)
    lib = _cabi.load()
    for s in ("geo_pose_workspace_bytes", "geo_relative_pose"):
        assert getattr(lib, s).argtypes is not None, s


def test_pose_constants_match_bindings():
    assert re.search(rf"#define GEO_ESSENTIAL {_cabi.GEO_ESSENTIAL}\b", _header())
    assert re.search(r"#define GEO_MAX_SOLUTIONS 10\b", _header())


def test_workspace_does_not_grow_with_the_budget():
    lib = _cabi.load()
    assert lib.geo_pose_workspace_bytes(32, 2048, 1000) == lib.geo_pose_workspace_bytes(32, 2048, 1 << 24) > 0
    assert lib.geo_pose_workspace_bytes(32, 4096, 1000) > lib.geo_pose_workspace_bytes(32, 2048, 1000)


def test_defaults_are_opencvs():
    p = inspect.signature(estimate_relative_pose).parameters
    assert (p["ransac_reproj_threshold"].default, p["max_iters"].default, p["confidence"].default) == (1.0, 1000, 0.999)
    assert p["distance_threshold"].default == 50.0 and p["seed"].default == 0 and p["K1"].default is None


def test_struct_layouts():
    c = _cabi.GeoPoseConfig(_cabi.GEO_ABI_VERSION, 1000, 0xFFFFFFFF, 0, 1.0, 0.999, 50.0)
    assert (c.abi_version, c.max_iters, c.seed, c.threshold, c.confidence, c.distance_threshold) == \
        (1, 1000, 0xFFFFFFFF, 1.0, 0.999, 50.0)
    assert _cabi.GeoPoseConfig.threshold.offset == 16 and ctypes.sizeof(_cabi.GeoPoseConfig) == 40
    assert _cabi.GeoPoseInputs.K0.offset == 40 and ctypes.sizeof(_cabi.GeoPoseInputs) == 56
    assert [f for f, _ in _cabi.GeoPoseOutputs._fields_] == [
        "E", "R", "t", "inliers", "num_inliers", "pose_inliers", "num_pose_inliers", "success", "best_hypothesis",
        "best_solution", "num_hypotheses"]


def _inputs(b=2, m=16, n=12):
    return torch.rand(b, m, 2), torch.rand(b, n, 2), torch.randint(-1, n, (b, m)), torch.eye(3, dtype=torch.float64)


def test_cpu_tensors_raise():
    with pytest.raises(RuntimeError):
        estimate_relative_pose(*_inputs())


@pytest.mark.parametrize("case", ["kpts0_rank", "matches_dtype", "batch", "not_tensor", "K_shape", "K_batch", "K1_shape",
                                  "K_int", "K_not_tensor"])
def test_bad_shapes_and_dtypes_raise_value_error(case, monkeypatch):
    k0, k1, m0, K = _inputs()
    bad = {
        "kpts0_rank": ((k0[0], k1, m0, K), {}),
        "matches_dtype": ((k0, k1, m0.to(torch.int32), K), {}),
        "batch": ((k0, k1[:1], m0, K), {}),
        "not_tensor": ((k0.numpy(), k1, m0, K), {}),
        "K_shape": ((k0, k1, m0, K[:2]), {}),
        "K_batch": ((k0, k1, m0, K.expand(3, 3, 3)), {}),
        "K1_shape": ((k0, k1, m0, K), {"K1": K.reshape(9)}),
        "K_int": ((k0, k1, m0, K.to(torch.int64)), {}),
        "K_not_tensor": ((k0, k1, m0, K.numpy()), {}),
    }[case]
    # shapes and dtypes are checked before any device work: CPU tensors posing as CUDA ones reach those checks
    monkeypatch.setattr(torch.Tensor, "device", property(lambda self: torch.device("cuda", 0)))
    with pytest.raises(ValueError):
        estimate_relative_pose(*bad[0], **bad[1])


@pytest.mark.parametrize("kw", [dict(max_iters=0), dict(max_iters=1.5), dict(max_iters=(1 << 24) + 1),
                                dict(ransac_reproj_threshold=0.0), dict(ransac_reproj_threshold=-1.0),
                                dict(confidence=1.5), dict(confidence=-0.1), dict(seed=-1), dict(seed=1 << 32),
                                dict(distance_threshold=0.0), dict(distance_threshold=float("inf"))])
def test_bad_parameters_raise_value_error(kw, monkeypatch):
    monkeypatch.setattr(torch.Tensor, "device", property(lambda self: torch.device("cuda", 0)))
    with pytest.raises(ValueError):
        estimate_relative_pose(*_inputs(), **kw)
