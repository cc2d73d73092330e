"""Geometric verification without a GPU: the header's export table, argument checks and OpenCV's defaults
(include/geometry_b200.h, lightglue_b200/geometry.py)."""
import ctypes
import inspect
import os
import re

import pytest
import torch

from lightglue_b200 import _cabi
from lightglue_b200.geometry import find_fundamental, find_homography

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_symbols_equal_exports_and_are_exported():
    with open(os.path.join(ROOT, "include", "geometry_b200.h")) as f:
        hdr = f.read()
    syms = tuple(re.findall(r"LG_API\s+[\w\s\*]+?\b(geo_\w+)\s*\(", hdr))
    assert sorted(syms) == sorted(_cabi.GEO_EXPORTS)
    lib = _cabi.load()
    for s in _cabi.GEO_EXPORTS:
        assert hasattr(lib, s), s
        assert getattr(lib, s).argtypes is not None, s


def test_header_constants_match_bindings():
    with open(os.path.join(ROOT, "include", "geometry_b200.h")) as f:
        hdr = f.read()
    for name, value in (("GEO_ABI_VERSION", _cabi.GEO_ABI_VERSION), ("GEO_HOMOGRAPHY", _cabi.GEO_HOMOGRAPHY),
                        ("GEO_FUNDAMENTAL", _cabi.GEO_FUNDAMENTAL)):
        assert re.search(rf"#define {name} {value}\b", hdr), name


def test_workspace_does_not_grow_with_the_budget():
    lib = _cabi.load()
    assert lib.geo_workspace_bytes(32, 2048, 2000) == lib.geo_workspace_bytes(32, 2048, 100000) > 0
    assert lib.geo_workspace_bytes(32, 4096, 2000) > lib.geo_workspace_bytes(32, 2048, 2000)


def test_defaults_are_opencvs():
    h = inspect.signature(find_homography).parameters
    f = inspect.signature(find_fundamental).parameters
    assert (h["ransac_reproj_threshold"].default, h["max_iters"].default, h["confidence"].default) == (3.0, 2000, 0.995)
    assert (f["ransac_reproj_threshold"].default, f["max_iters"].default, f["confidence"].default) == (3.0, 1000, 0.99)
    assert h["seed"].default == f["seed"].default == 0


def _inputs(b=2, m=16, n=12):
    return torch.rand(b, m, 2), torch.rand(b, n, 2), torch.randint(-1, n, (b, m))


@pytest.mark.parametrize("fn", [find_homography, find_fundamental])
def test_cpu_tensors_raise(fn):
    with pytest.raises(RuntimeError):
        fn(*_inputs())


@pytest.mark.parametrize("fn", [find_homography, find_fundamental])
@pytest.mark.parametrize("case", ["kpts0_rank", "kpts1_last", "matches_shape", "matches_dtype", "batch", "kpts_int",
                                  "not_tensor"])
def test_bad_shapes_and_dtypes_raise_value_error(fn, case, monkeypatch):
    k0, k1, m0 = _inputs()
    bad = {
        "kpts0_rank": (k0[0], k1, m0),
        "kpts1_last": (k0, k1[..., :1], m0),
        "matches_shape": (k0, k1, m0[:, :-1]),
        "matches_dtype": (k0, k1, m0.to(torch.int32)),
        "batch": (k0, k1[:1], m0),
        "kpts_int": (k0.to(torch.int64), k1, m0),
        "not_tensor": (k0.numpy(), k1, m0),
    }[case]
    # shapes and dtypes are checked before any device work: CPU tensors posing as CUDA ones reach those checks
    monkeypatch.setattr(torch.Tensor, "device", property(lambda self: torch.device("cuda", 0)))
    with pytest.raises(ValueError):
        fn(*bad)


@pytest.mark.parametrize("kw", [dict(max_iters=0), dict(max_iters=1.5), dict(max_iters=(1 << 24) + 1),
                                dict(ransac_reproj_threshold=0.0), dict(ransac_reproj_threshold=-1.0),
                                dict(confidence=1.5), dict(confidence=-0.1), dict(seed=-1), dict(seed=1 << 32)])
def test_bad_parameters_raise_value_error(kw, monkeypatch):
    monkeypatch.setattr(torch.Tensor, "device", property(lambda self: torch.device("cuda", 0)))
    with pytest.raises(ValueError):
        find_homography(*_inputs(), **kw)


def test_config_struct_layout():
    c = _cabi.GeoConfig(_cabi.GEO_ABI_VERSION, _cabi.GEO_FUNDAMENTAL, 1000, 0xFFFFFFFF, 3.0, 0.99)
    assert (c.abi_version, c.model, c.max_iters, c.seed, c.threshold, c.confidence) == (1, 1, 1000, 0xFFFFFFFF, 3.0, 0.99)
    assert _cabi.GeoConfig.threshold.offset == 16 and ctypes.sizeof(_cabi.GeoConfig) == 32
    assert [f for f, _ in _cabi.GeoOutputs._fields_] == ["model", "inliers", "num_inliers", "success", "best_hypothesis",
                                                         "num_hypotheses"]
