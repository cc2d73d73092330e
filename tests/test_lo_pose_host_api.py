"""LO-RANSAC relative pose without a GPU: the header's new exports, constants and struct layouts, argument checks,
the shared defaults and B = 0 (include/geometry_b200.h, lightglue_b200/geometry.py)."""
import ctypes
import inspect
import os
import re

import pytest
import torch

from lightglue_b200 import _cabi
from lightglue_b200.geometry import estimate_relative_pose, estimate_relative_pose_lo
from oracle import lo_pose_oracle as lo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header():
    with open(os.path.join(ROOT, "include", "geometry_b200.h")) as f:
        return f.read()


def test_lo_entry_points_are_exported():
    assert {"geo_lo_pose_workspace_bytes", "geo_relative_pose_lo"} <= set(_cabi.GEO_EXPORTS)
    lib = _cabi.load()
    for s in ("geo_lo_pose_workspace_bytes", "geo_relative_pose_lo"):
        assert getattr(lib, s).argtypes is not None, s


def test_lo_constants_and_row_bound_match_the_oracle_and_bindings():
    h = _header()
    for name, value in (("GEO_LO_QSCALE", lo.QSCALE), ("GEO_LO_STEPS", lo.STEPS),
                        ("GEO_LO_FINAL_STEPS", lo.FINAL_STEPS)):
        assert re.search(rf"#define {name} {value}\b", h), name
    assert re.search(r"#define GEO_LO_LAMBDA0 1e-3\b", h) and lo.LAMBDA0 == 1e-3
    # the row bound keeps the largest score, QSCALE * M, below 2^36: the bits above h in the (score, h) key
    assert re.search(r"#define GEO_LO_MAX_MATCHES \(\(1 << 20\) - 1\)", h) and _cabi.GEO_LO_MAX_MATCHES == (1 << 20) - 1
    assert lo.QSCALE * _cabi.GEO_LO_MAX_MATCHES < 1 << 36
    assert _cabi.GEO_LO_QSCALE == lo.QSCALE
    assert re.search(r"#define GEO_ABI_VERSION 1\b", h)


def test_workspace_does_not_grow_with_the_budget():
    lib = _cabi.load()
    assert lib.geo_lo_pose_workspace_bytes(32, 2048, 1000) == lib.geo_lo_pose_workspace_bytes(32, 2048, 1 << 24) > 0
    assert lib.geo_lo_pose_workspace_bytes(32, 4096, 1000) > lib.geo_lo_pose_workspace_bytes(32, 2048, 1000)
    assert lib.geo_lo_pose_workspace_bytes(32, 2048, 1000) > lib.geo_pose_workspace_bytes(32, 2048, 1000)


def test_defaults_equal_the_plain_estimators():
    a = inspect.signature(estimate_relative_pose).parameters
    b = inspect.signature(estimate_relative_pose_lo).parameters
    assert list(a) == list(b)
    assert all(a[k].default == b[k].default for k in a)


def test_struct_layouts():
    c = _cabi.GeoLoPoseConfig(_cabi.GEO_ABI_VERSION, 1000, 0xFFFFFFFF, 0, 1.0, 0.999, 50.0)
    assert (c.abi_version, c.max_iters, c.seed, c.threshold, c.confidence, c.distance_threshold) == \
        (1, 1000, 0xFFFFFFFF, 1.0, 0.999, 50.0)
    assert _cabi.GeoLoPoseConfig.threshold.offset == 16 and ctypes.sizeof(_cabi.GeoLoPoseConfig) == 40
    assert _cabi.GeoLoPoseOutputs.num_local_optimizations.offset == ctypes.sizeof(_cabi.GeoPoseOutputs) == 88
    assert ctypes.sizeof(_cabi.GeoLoPoseOutputs) == 104


def _call(lib, b=0, m=16, n=12, **cfg_kw):
    kw = dict(max_iters=1000, seed=0, reserved=0, threshold=1.0, confidence=0.999, distance_threshold=50.0)
    kw.update(cfg_kw)
    cfg = _cabi.GeoLoPoseConfig(_cabi.GEO_ABI_VERSION, *kw.values())
    ins = _cabi.GeoPoseInputs(b, m, n, None, None, None, None, None)
    outs = _cabi.GeoLoPoseOutputs()
    return lib.geo_relative_pose_lo(ctypes.byref(cfg), ctypes.byref(ins), ctypes.byref(outs), None, 0, None)


def test_an_empty_batch_is_a_no_op():
    lib = _cabi.load()
    assert _call(lib, b=0) == 0


@pytest.mark.parametrize("kw", [dict(max_iters=0), dict(threshold=0.0), dict(confidence=1.5),
                                dict(distance_threshold=float("inf")), dict(b=-1), dict(m=(1 << 20) + 1)])
def test_the_c_abi_rejects_bad_arguments(kw):
    lib = _cabi.load()
    assert _call(lib, **kw) != 0
    assert lib.lg_last_error().decode().startswith("geo_relative_pose_lo")


def _inputs(b=2, m=16, n=12):
    return torch.rand(b, m, 2), torch.rand(b, n, 2), torch.randint(-1, n, (b, m)), torch.eye(3, dtype=torch.float64)


def test_cpu_tensors_raise():
    with pytest.raises(RuntimeError):
        estimate_relative_pose_lo(*_inputs())


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
        estimate_relative_pose_lo(*bad[0], **bad[1])


@pytest.mark.parametrize("kw", [dict(max_iters=0), dict(max_iters=1.5), dict(max_iters=(1 << 24) + 1),
                                dict(ransac_reproj_threshold=0.0), dict(ransac_reproj_threshold=-1.0),
                                dict(confidence=1.5), dict(confidence=-0.1), dict(seed=-1), dict(seed=1 << 32),
                                dict(distance_threshold=0.0), dict(distance_threshold=float("inf"))])
def test_bad_parameters_raise_value_error(kw, monkeypatch):
    monkeypatch.setattr(torch.Tensor, "device", property(lambda self: torch.device("cuda", 0)))
    with pytest.raises(ValueError):
        estimate_relative_pose_lo(*_inputs(), **kw)


def test_too_many_rows_raise_value_error(monkeypatch):
    monkeypatch.setattr(torch.Tensor, "device", property(lambda self: torch.device("cuda", 0)))
    m = (1 << 20) + 1
    with pytest.raises(ValueError):
        estimate_relative_pose_lo(torch.zeros(1, m, 2), torch.zeros(1, 4, 2), torch.full((1, m), -1),
                                  torch.eye(3, dtype=torch.float64))
