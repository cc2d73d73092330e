"""LO-RANSAC homography without a GPU: the header's new exports and struct layout, argument checks, the shared defaults
and B = 0 (include/geometry_b200.h, lightglue_b200/geometry.py)."""
import ctypes
import inspect
import os
import re

import pytest
import torch

from lightglue_b200 import _cabi
from lightglue_b200.geometry import find_homography, find_homography_lo
from oracle import lo_homography_oracle as lh

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header():
    with open(os.path.join(ROOT, "include", "geometry_b200.h")) as f:
        return f.read()


def test_lo_homography_entry_points_are_exported():
    h = _header()
    for s in ("geo_lo_homography_workspace_bytes", "geo_homography_lo"):
        assert s in _cabi.GEO_EXPORTS and re.search(rf"LG_API \w+ {s}\(", h), s
    lib = _cabi.load()
    for s in ("geo_lo_homography_workspace_bytes", "geo_homography_lo"):
        assert getattr(lib, s).argtypes is not None, s


def test_constants_are_shared_with_the_lo_pose():
    h = _header()
    for name, value in (("GEO_LO_QSCALE", lh.QSCALE), ("GEO_LO_STEPS", lh.STEPS), ("GEO_LO_FINAL_STEPS", lh.FINAL_STEPS)):
        assert re.search(rf"#define {name} {value}\b", h), name
    assert lh.LAMBDA0 == 1e-3 and re.search(r"#define GEO_LO_LAMBDA0 1e-3\b", h)
    assert re.search(r"#define GEO_ABI_VERSION 1\b", h) and _cabi.GEO_ABI_VERSION == 1


def test_workspace_does_not_grow_with_the_budget():
    lib = _cabi.load()
    ws = lib.geo_lo_homography_workspace_bytes
    assert ws(32, 2048, 2000) == ws(32, 2048, 1 << 24) > 0
    assert ws(32, 4096, 2000) > ws(32, 2048, 2000) > lib.geo_workspace_bytes(32, 2048, 2000)


def test_defaults_equal_the_plain_estimator():
    a = inspect.signature(find_homography).parameters
    b = inspect.signature(find_homography_lo).parameters
    assert list(a) == list(b)
    assert all(a[k].default == b[k].default for k in a)


def test_struct_layout():
    assert re.search(r"typedef struct GeoLoOutputs \{\s*GeoOutputs geo;[^}]*int32_t\* num_local_optimizations;[^}]*"
                     r"int64_t\* cost;[^}]*\} GeoLoOutputs;", _header())
    assert _cabi.GeoLoOutputs.num_local_optimizations.offset == ctypes.sizeof(_cabi.GeoOutputs) == 48
    assert _cabi.GeoLoOutputs.cost.offset == 56 and ctypes.sizeof(_cabi.GeoLoOutputs) == 64


def _call(lib, b=0, m=16, n=12, model=_cabi.GEO_HOMOGRAPHY, max_iters=2000, threshold=3.0, confidence=0.995):
    cfg = _cabi.GeoConfig(_cabi.GEO_ABI_VERSION, model, max_iters, 0, threshold, confidence)
    ins = _cabi.GeoInputs(b, m, n, None, None, None)
    outs = _cabi.GeoLoOutputs()
    return lib.geo_homography_lo(ctypes.byref(cfg), ctypes.byref(ins), ctypes.byref(outs), None, 0, None)


def test_an_empty_batch_is_a_no_op():
    assert _call(_cabi.load(), b=0) == 0


@pytest.mark.parametrize("kw", [dict(model=_cabi.GEO_FUNDAMENTAL), dict(model=_cabi.GEO_ESSENTIAL), dict(model=7),
                                dict(max_iters=0), dict(threshold=0.0), dict(confidence=1.5), dict(b=-1),
                                dict(m=(1 << 20) + 1)])
def test_the_c_abi_rejects_bad_arguments(kw):
    lib = _cabi.load()
    assert _call(lib, **kw) != 0
    assert lib.lg_last_error().decode().startswith("geo_homography_lo")


def test_the_c_abi_names_the_model_it_needs():
    lib = _cabi.load()
    assert _call(lib, model=_cabi.GEO_FUNDAMENTAL) != 0
    assert "GEO_HOMOGRAPHY" in lib.lg_last_error().decode()


def _inputs(b=2, m=16, n=12):
    return torch.rand(b, m, 2), torch.rand(b, n, 2), torch.randint(-1, n, (b, m))


def test_cpu_tensors_raise():
    with pytest.raises(RuntimeError):
        find_homography_lo(*_inputs())


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
        find_homography_lo(*bad)


@pytest.mark.parametrize("kw", [dict(max_iters=0), dict(max_iters=1.5), dict(max_iters=(1 << 24) + 1),
                                dict(ransac_reproj_threshold=0.0), dict(ransac_reproj_threshold=-1.0),
                                dict(confidence=1.5), dict(confidence=-0.1), dict(seed=-1), dict(seed=1 << 32)])
def test_bad_parameters_raise_value_error(kw, monkeypatch):
    monkeypatch.setattr(torch.Tensor, "device", property(lambda self: torch.device("cuda", 0)))
    with pytest.raises(ValueError):
        find_homography_lo(*_inputs(), **kw)


def test_too_many_rows_raise_value_error(monkeypatch):
    monkeypatch.setattr(torch.Tensor, "device", property(lambda self: torch.device("cuda", 0)))
    m = (1 << 20) + 1
    with pytest.raises(ValueError):
        find_homography_lo(torch.zeros(1, m, 2), torch.zeros(1, 4, 2), torch.full((1, m), -1))
