"""MAGSAC++ homography and fundamental matrix without a GPU: the header's new exports, constants and struct layout,
argument checks, defaults and B = 0 (include/geometry_b200.h, lightglue_b200/geometry.py)."""
import ctypes
import inspect
import os
import re

import pytest
import torch

from lightglue_b200 import _cabi
from lightglue_b200.geometry import (find_fundamental_lo, find_fundamental_magsac, find_homography_lo,
                                     find_homography_magsac)
from oracle import magsac_oracle as mo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRIES = {"geo_homography_magsac": (_cabi.GEO_HOMOGRAPHY, "GEO_HOMOGRAPHY", find_homography_magsac,
                                     find_homography_lo),
           "geo_fundamental_magsac": (_cabi.GEO_FUNDAMENTAL, "GEO_FUNDAMENTAL", find_fundamental_magsac,
                                      find_fundamental_lo)}


def _header():
    with open(os.path.join(ROOT, "include", "geometry_b200.h")) as f:
        return f.read()


def test_entry_points_are_exported():
    h = _header()
    lib = _cabi.load()
    for s in ENTRIES:
        assert s in _cabi.GEO_EXPORTS and re.search(rf"LG_API \w+ {s}\(", h), s
        assert getattr(lib, s).argtypes is not None, s


def test_constants_and_struct_layout():
    h = _header()
    assert re.search(rf"#define GEO_MAGSAC_KNOTS {mo.KNOTS}\b", h) and _cabi.GEO_MAGSAC_KNOTS == mo.KNOTS
    assert re.search(rf"#define GEO_MAGSAC_K {_cabi.GEO_MAGSAC_K!r}\b", h)
    assert re.search(r"typedef struct GeoMagsacConfig \{\s*GeoConfig geo;[^}]*double max_threshold;[^}]*\} "
                     r"GeoMagsacConfig;", h)
    assert _cabi.GeoMagsacConfig.max_threshold.offset == ctypes.sizeof(_cabi.GeoConfig) == 32
    assert ctypes.sizeof(_cabi.GeoMagsacConfig) == 40
    assert re.search(r"#define GEO_ABI_VERSION 1\b", h) and _cabi.GEO_ABI_VERSION == 1


@pytest.mark.parametrize("entry", list(ENTRIES))
def test_defaults_extend_the_lo_estimator(entry):
    a = inspect.signature(ENTRIES[entry][3]).parameters
    b = inspect.signature(ENTRIES[entry][2]).parameters
    assert [k for k in b if k != "max_threshold"] == list(a)
    assert all(a[k].default == b[k].default for k in a) and b["max_threshold"].default == 7.5


def _call(entry, b=0, m=16, n=12, model=None, max_iters=2000, threshold=3.0, confidence=0.995, max_threshold=7.5,
          abi=_cabi.GEO_ABI_VERSION):
    lib = _cabi.load()
    model = ENTRIES[entry][0] if model is None else model
    cfg = _cabi.GeoMagsacConfig(_cabi.GeoConfig(abi, model, max_iters, 0, threshold, confidence), max_threshold)
    ins = _cabi.GeoInputs(b, m, n, None, None, None)
    outs = _cabi.GeoLoOutputs()
    return getattr(lib, entry)(ctypes.byref(cfg), ctypes.byref(ins), ctypes.byref(outs), None, 0, None)


@pytest.mark.parametrize("entry", list(ENTRIES))
def test_an_empty_batch_is_a_no_op(entry):
    assert _call(entry, b=0) == 0


@pytest.mark.parametrize("entry", list(ENTRIES))
@pytest.mark.parametrize("kw", [dict(model=_cabi.GEO_ESSENTIAL), dict(model=7), dict(abi=2), dict(max_iters=0),
                                dict(threshold=0.0), dict(confidence=1.5), dict(max_threshold=0.0),
                                dict(max_threshold=-1.0), dict(max_threshold=float("inf")),
                                dict(max_threshold=float("nan")), dict(b=-1), dict(m=(1 << 20) + 1)])
def test_the_c_abi_rejects_bad_arguments(entry, kw):
    assert _call(entry, **kw) != 0
    assert _cabi.load().lg_last_error().decode().startswith(entry)


@pytest.mark.parametrize("entry", list(ENTRIES))
def test_the_c_abi_names_the_model_it_needs(entry):
    other = _cabi.GEO_FUNDAMENTAL if ENTRIES[entry][0] == _cabi.GEO_HOMOGRAPHY else _cabi.GEO_HOMOGRAPHY
    assert _call(entry, model=other) != 0
    assert ENTRIES[entry][1] in _cabi.load().lg_last_error().decode()


def test_a_null_config_is_rejected():
    lib = _cabi.load()
    for entry in ENTRIES:
        ins, outs = _cabi.GeoInputs(0, 0, 0, None, None, None), _cabi.GeoLoOutputs()
        assert getattr(lib, entry)(None, ctypes.byref(ins), ctypes.byref(outs), None, 0, None) != 0


def _inputs(b=2, m=16, n=12):
    return torch.rand(b, m, 2), torch.rand(b, n, 2), torch.randint(-1, n, (b, m))


@pytest.mark.parametrize("fn", [find_homography_magsac, find_fundamental_magsac])
def test_cpu_tensors_raise(fn):
    with pytest.raises(RuntimeError):
        fn(*_inputs())


@pytest.mark.parametrize("fn", [find_homography_magsac, find_fundamental_magsac])
@pytest.mark.parametrize("kw", [dict(max_threshold=0.0), dict(max_threshold=-2.0), dict(max_threshold=float("inf")),
                                dict(max_threshold=float("nan")), dict(max_iters=0), dict(ransac_reproj_threshold=0.0),
                                dict(confidence=1.5), dict(seed=-1)])
def test_bad_parameters_raise_value_error(fn, kw, monkeypatch):
    monkeypatch.setattr(torch.Tensor, "device", property(lambda self: torch.device("cuda", 0)))
    with pytest.raises(ValueError):
        fn(*_inputs(), **kw)


@pytest.mark.parametrize("fn", [find_homography_magsac, find_fundamental_magsac])
def test_too_many_rows_raise_value_error(fn, monkeypatch):
    monkeypatch.setattr(torch.Tensor, "device", property(lambda self: torch.device("cuda", 0)))
    m = (1 << 20) + 1
    with pytest.raises(ValueError):
        fn(torch.zeros(1, m, 2), torch.zeros(1, 4, 2), torch.full((1, m), -1))
