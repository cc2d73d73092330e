"""Absolute pose without a GPU: the header's new exports, constants and struct layouts, argument checks and OpenCV's
defaults (include/geometry_b200.h, lightglue_b200/geometry.py)."""
import ctypes
import inspect
import os
import re

import pytest
import torch

from lightglue_b200 import _cabi
from lightglue_b200.geometry import estimate_absolute_pose
from oracle import pnp_oracle as pp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header():
    with open(os.path.join(ROOT, "include", "geometry_b200.h")) as f:
        return f.read()


def test_pnp_entry_points_are_exported():
    assert {"geo_pnp_workspace_bytes", "geo_absolute_pose"} <= set(_cabi.GEO_EXPORTS)
    lib = _cabi.load()
    for s in ("geo_pnp_workspace_bytes", "geo_absolute_pose"):
        assert getattr(lib, s).argtypes is not None, s


def test_pnp_constants_match_the_oracle():
    h = _header()
    for name, value in (("MAX_SOLUTIONS", pp.MAX_SOLS), ("COLLINEAR_EPS", pp.COLLINEAR_EPS),
                        ("BISECT_STEPS", pp.BISECT_STEPS), ("NEWTON_STEPS", pp.NEWTON_STEPS),
                        ("GN_STEPS", pp.GN_STEPS), ("LM_STEPS", pp.LM_STEPS), ("LM_LAMBDA0", pp.LM_LAMBDA0),
                        ("REFIT_MIN", pp.REFIT_MIN)):
        m = re.search(rf"#define GEO_PNP_{name} (\S+)", h)
        assert m and float(m.group(1)) == value, name
    assert re.search(r"#define GEO_ABI_VERSION 1\b", h)


def test_workspace_does_not_grow_with_the_budget():
    lib = _cabi.load()
    assert lib.geo_pnp_workspace_bytes(32, 2048, 100) == lib.geo_pnp_workspace_bytes(32, 2048, 1 << 24) > 0
    assert lib.geo_pnp_workspace_bytes(32, 4096, 100) > lib.geo_pnp_workspace_bytes(32, 2048, 100)


def test_defaults_are_opencvs():
    p = inspect.signature(estimate_absolute_pose).parameters
    assert (p["ransac_reproj_threshold"].default, p["max_iters"].default, p["confidence"].default) == (8.0, 100, 0.99)
    assert p["seed"].default == 0


def test_struct_layouts():
    c = _cabi.GeoPnpConfig(_cabi.GEO_ABI_VERSION, 100, 0xFFFFFFFF, 0, 8.0, 0.99)
    assert (c.abi_version, c.max_iters, c.seed, c.threshold, c.confidence) == (1, 100, 0xFFFFFFFF, 8.0, 0.99)
    assert _cabi.GeoPnpConfig.threshold.offset == 16 and ctypes.sizeof(_cabi.GeoPnpConfig) == 32
    assert _cabi.GeoPnpInputs.points3d1.offset == 24 and _cabi.GeoPnpInputs.K0.offset == 40
    assert ctypes.sizeof(_cabi.GeoPnpInputs) == 48
    assert [f for f, _ in _cabi.GeoPnpOutputs._fields_] == [
        "R", "t", "inliers", "num_inliers", "success", "best_hypothesis", "best_solution", "num_hypotheses"]
    assert ctypes.sizeof(_cabi.GeoPnpOutputs) == 64


def _inputs(b=2, m=16, n=12):
    return torch.rand(b, m, 2), torch.rand(b, n, 3), torch.randint(-1, n, (b, m)), torch.eye(3, dtype=torch.float64)


def test_cpu_tensors_raise():
    with pytest.raises(RuntimeError):
        estimate_absolute_pose(*_inputs())


@pytest.mark.parametrize("case", ["kpts0_rank", "points_dim", "points_rank", "matches_dtype", "batch", "not_tensor",
                                  "points_int", "K_shape", "K_batch", "K_int", "K_not_tensor"])
def test_bad_shapes_and_dtypes_raise_value_error(case, monkeypatch):
    k0, p3, m0, K = _inputs()
    bad = {
        "kpts0_rank": (k0[0], p3, m0, K),
        "points_dim": (k0, p3[..., :2], m0, K),
        "points_rank": (k0, p3[0], m0, K),
        "matches_dtype": (k0, p3, m0.to(torch.int32), K),
        "batch": (k0, p3[:1], m0, K),
        "not_tensor": (k0, p3.numpy(), m0, K),
        "points_int": (k0, p3.to(torch.int64), m0, K),
        "K_shape": (k0, p3, m0, K[:2]),
        "K_batch": (k0, p3, m0, K.expand(3, 3, 3)),
        "K_int": (k0, p3, m0, K.to(torch.int64)),
        "K_not_tensor": (k0, p3, m0, K.numpy()),
    }[case]
    # shapes and dtypes are checked before any device work: CPU tensors posing as CUDA ones reach those checks
    monkeypatch.setattr(torch.Tensor, "device", property(lambda self: torch.device("cuda", 0)))
    with pytest.raises(ValueError):
        estimate_absolute_pose(*bad)


def test_messages_name_the_3d_points(monkeypatch):
    k0, p3, m0, K = _inputs()
    monkeypatch.setattr(torch.Tensor, "device", property(lambda self: torch.device("cuda", 0)))
    with pytest.raises(ValueError, match=r"points3d1 \(2, 12, 2\): expected \[B, M, 2\] and \[B, N, 3\]"):
        estimate_absolute_pose(k0, p3[..., :2], m0, K)


@pytest.mark.parametrize("kw", [dict(max_iters=0), dict(max_iters=1.5), dict(max_iters=(1 << 24) + 1),
                                dict(ransac_reproj_threshold=0.0), dict(ransac_reproj_threshold=-1.0),
                                dict(ransac_reproj_threshold=float("inf")), dict(confidence=1.5),
                                dict(confidence=-0.1), dict(seed=-1), dict(seed=1 << 32)])
def test_bad_parameters_raise_value_error(kw, monkeypatch):
    monkeypatch.setattr(torch.Tensor, "device", property(lambda self: torch.device("cuda", 0)))
    with pytest.raises(ValueError):
        estimate_absolute_pose(*_inputs(), **kw)
