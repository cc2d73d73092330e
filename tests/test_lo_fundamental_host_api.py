"""LO-RANSAC fundamental matrix without a GPU: the header's new exports, argument checks, the shared constants and
defaults, and B = 0 (include/geometry_b200.h, lightglue_b200/geometry.py)."""
import ctypes
import inspect
import os
import re

import pytest
import torch

from lightglue_b200 import _cabi
from lightglue_b200.geometry import find_fundamental, find_fundamental_lo
from oracle import lo_fundamental_oracle as lf

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header():
    with open(os.path.join(ROOT, "include", "geometry_b200.h")) as f:
        return f.read()


def test_lo_fundamental_entry_points_are_exported():
    h = _header()
    for s in ("geo_lo_fundamental_workspace_bytes", "geo_fundamental_lo"):
        assert s in _cabi.GEO_EXPORTS and re.search(rf"LG_API \w+ {s}\(", h), s
    assert re.search(r"LG_API int geo_fundamental_lo\(const GeoConfig\* cfg, const GeoInputs\* in, GeoLoOutputs\* out,",
                     h)
    lib = _cabi.load()
    for s in ("geo_lo_fundamental_workspace_bytes", "geo_fundamental_lo"):
        assert getattr(lib, s).argtypes is not None, s


def test_constants_are_shared_with_the_other_lo_estimators():
    h = _header()
    for name, value in (("GEO_LO_QSCALE", lf.QSCALE), ("GEO_LO_STEPS", lf.STEPS), ("GEO_LO_FINAL_STEPS", lf.FINAL_STEPS)):
        assert re.search(rf"#define {name} {value}\b", h), name
    assert lf.LAMBDA0 == 1e-3 and re.search(r"#define GEO_LO_LAMBDA0 1e-3\b", h)
    assert re.search(r"#define GEO_ABI_VERSION 1\b", h) and _cabi.GEO_ABI_VERSION == 1
    assert _cabi.GEO_LO_MAX_MATCHES == (1 << 20) - 1


def test_workspace_does_not_grow_with_the_budget():
    lib = _cabi.load()
    ws = lib.geo_lo_fundamental_workspace_bytes
    assert ws(32, 2048, 1000) == ws(32, 2048, 1 << 24) > 0
    assert ws(32, 4096, 1000) > ws(32, 2048, 1000) > lib.geo_workspace_bytes(32, 2048, 1000)
    assert ws(32, 2048, 1000) == lib.geo_lo_homography_workspace_bytes(32, 2048, 1000)


def test_defaults_equal_the_plain_estimator():
    a = inspect.signature(find_fundamental).parameters
    b = inspect.signature(find_fundamental_lo).parameters
    assert list(a) == list(b)
    assert all(a[k].default == b[k].default for k in a)


def _call(lib, b=0, m=16, n=12, model=_cabi.GEO_FUNDAMENTAL, max_iters=1000, threshold=3.0, confidence=0.99):
    cfg = _cabi.GeoConfig(_cabi.GEO_ABI_VERSION, model, max_iters, 0, threshold, confidence)
    ins = _cabi.GeoInputs(b, m, n, None, None, None)
    outs = _cabi.GeoLoOutputs()
    return lib.geo_fundamental_lo(ctypes.byref(cfg), ctypes.byref(ins), ctypes.byref(outs), None, 0, None)


def test_an_empty_batch_is_a_no_op():
    assert _call(_cabi.load(), b=0) == 0


@pytest.mark.parametrize("kw", [dict(model=_cabi.GEO_HOMOGRAPHY), dict(model=_cabi.GEO_ESSENTIAL), dict(model=7),
                                dict(max_iters=0), dict(max_iters=(1 << 24) + 1), dict(threshold=0.0),
                                dict(threshold=float("inf")), dict(threshold=float("nan")), dict(confidence=1.5),
                                dict(confidence=float("nan")), dict(b=-1), dict(m=-1),
                                dict(m=_cabi.GEO_LO_MAX_MATCHES + 1)])
def test_the_c_abi_rejects_bad_arguments(kw):
    lib = _cabi.load()
    assert _call(lib, **kw) != 0
    assert lib.lg_last_error().decode().startswith("geo_fundamental_lo")


def test_the_c_abi_names_the_model_it_needs():
    lib = _cabi.load()
    assert _call(lib, model=_cabi.GEO_HOMOGRAPHY) != 0
    assert "GEO_FUNDAMENTAL" in lib.lg_last_error().decode()


def test_the_c_abi_accepts_the_row_bound_and_checks_the_outputs():
    # M = GEO_LO_MAX_MATCHES passes the size checks and stops at the null outputs
    lib = _cabi.load()
    assert _call(lib, b=1, m=_cabi.GEO_LO_MAX_MATCHES) != 0
    assert "null output" in lib.lg_last_error().decode()


def _inputs(b=2, m=16, n=12):
    return torch.rand(b, m, 2), torch.rand(b, n, 2), torch.randint(-1, n, (b, m))


def test_cpu_tensors_raise():
    with pytest.raises(RuntimeError):
        find_fundamental_lo(*_inputs())


@pytest.mark.parametrize("case", ["kpts0_rank", "matches_dtype", "batch", "not_tensor", "kpts1_width"])
def test_bad_shapes_and_dtypes_raise_value_error(case, monkeypatch):
    k0, k1, m0 = _inputs()
    bad = {
        "kpts0_rank": (k0[0], k1, m0),
        "matches_dtype": (k0, k1, m0.to(torch.int32)),
        "batch": (k0, k1[:1], m0),
        "not_tensor": (k0.numpy(), k1, m0),
        "kpts1_width": (k0, torch.rand(2, 12, 3), m0),
    }[case]
    # shapes and dtypes are checked before any device work: CPU tensors posing as CUDA ones reach those checks
    monkeypatch.setattr(torch.Tensor, "device", property(lambda self: torch.device("cuda", 0)))
    with pytest.raises(ValueError):
        find_fundamental_lo(*bad)


@pytest.mark.parametrize("kw", [dict(max_iters=0), dict(max_iters=1.5), dict(max_iters=(1 << 24) + 1),
                                dict(ransac_reproj_threshold=0.0), dict(ransac_reproj_threshold=-1.0),
                                dict(ransac_reproj_threshold=float("inf")), dict(confidence=1.5),
                                dict(confidence=-0.1), dict(seed=-1), dict(seed=1 << 32), dict(seed=1.0)])
def test_bad_parameters_raise_value_error(kw, monkeypatch):
    monkeypatch.setattr(torch.Tensor, "device", property(lambda self: torch.device("cuda", 0)))
    with pytest.raises(ValueError):
        find_fundamental_lo(*_inputs(), **kw)


def test_too_many_rows_raise_value_error(monkeypatch):
    monkeypatch.setattr(torch.Tensor, "device", property(lambda self: torch.device("cuda", 0)))
    m = _cabi.GEO_LO_MAX_MATCHES + 1
    with pytest.raises(ValueError, match="rows per pair"):
        find_fundamental_lo(torch.zeros(1, m, 2), torch.zeros(1, 4, 2), torch.full((1, m), -1))
