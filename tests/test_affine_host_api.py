"""Affine and partial affine estimation without a GPU: the header's new constants, exports and ``GeoAffineConfig``
layout, the workspace size, every argument check of ``geo_estimate_affine`` with its exact message, and the Python
validation of ``estimate_affine_2d`` and ``estimate_affine_partial_2d`` (include/geometry_b200.h,
lightglue_b200/geometry.py)."""
import ctypes as C
import os
import re

import pytest
import torch

from lightglue_b200 import _cabi
from lightglue_b200.geometry import estimate_affine_2d, estimate_affine_partial_2d

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PTR = 4096  # any non-null address: every call below fails or returns before it is dereferenced
B, M, N = 2, 16, 12
ENTRY = "geo_estimate_affine"


def _header():
    with open(os.path.join(ROOT, "include", "geometry_b200.h")) as f:
        return f.read()


def test_constants_match_the_header():
    h = _header()
    for name in ("GEO_AFFINE", "GEO_AFFINE_PARTIAL", "GEO_AFFINE_MAX_REFINE"):
        m = re.search(rf"#define {name} (\d+)", h)
        assert m and int(m.group(1)) == getattr(_cabi, name), name
    assert (_cabi.GEO_AFFINE, _cabi.GEO_AFFINE_PARTIAL) == (3, 4)


def test_config_layout_matches_the_header():
    body = re.search(r"typedef struct GeoAffineConfig \{(.*?)\} GeoAffineConfig;", _header(), re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = [d.split()[-1] for d in body.split(";") if d.strip()]
    assert [f for f, _ in _cabi.GeoAffineConfig._fields_] == names
    assert _cabi.GeoAffineConfig.threshold.offset == 24 and C.sizeof(_cabi.GeoAffineConfig) == 40


def test_entry_points_are_declared_last_and_exported():
    declared = re.findall(r"LG_API \w+\*? (geo_\w+)\(", _header())
    assert declared[-2:] == ["geo_affine_workspace_bytes", ENTRY]
    assert list(_cabi.GEO_EXPORTS)[-2:] == declared[-2:]
    lib = _cabi.load()
    assert lib.geo_estimate_affine.argtypes[0] is C.POINTER(_cabi.GeoAffineConfig)
    assert lib.geo_estimate_affine.argtypes[1:3] == [C.POINTER(_cabi.GeoInputs), C.POINTER(_cabi.GeoOutputs)]


def test_workspace_matches_the_carve():
    lib = _cabi.load()
    for b, m in ((1, 0), (1, 100), (32, 2048), (265, 300), (1, (1 << 17) + 37)):
        # the H/F workspace of geo_hf.cuh: 72-byte pair records, compacted points (float4) and rows (int), one chunk
        # of 9-float models and int counts, each 256-byte aligned, plus 256 bytes of base alignment
        up = lambda x: (x + 255) // 256 * 256  # noqa: E731
        want = up(b * 72) + up(b * m * 16) + up(b * m * 4) + up(b * 256 * 9 * 4) + up(b * 256 * 4) + 256
        got = lib.geo_affine_workspace_bytes(b, m, 2000)
        assert got == want == lib.geo_workspace_bytes(b, m, 2000), (b, m, got, want)
    assert lib.geo_affine_workspace_bytes(-1, 10, 1) == 0 and lib.geo_affine_workspace_bytes(1, -1, 1) == 0


def _call(fault=lambda cfg, ins, outs: None, ws_short=False):
    lib = _cabi.load()
    cfg = _cabi.GeoAffineConfig(_cabi.GEO_ABI_VERSION, _cabi.GEO_AFFINE, 1000, 0, 10, 0, 3.0, 0.99)
    ins = _cabi.GeoInputs(B, M, N, PTR, PTR, PTR)
    outs = _cabi.GeoOutputs(*([PTR] * len(_cabi.GeoOutputs._fields_)))
    fault(cfg, ins, outs)
    bytes_ = lib.geo_affine_workspace_bytes(max(ins.B, 0), max(ins.M, 0), cfg.max_iters) - (1 if ws_short else 0)
    rc = lib.geo_estimate_affine(C.byref(cfg), C.byref(ins), C.byref(outs), PTR, bytes_, None)
    return rc, lib.lg_last_error().decode()


def _set(obj, field, value):
    return lambda cfg, ins, outs: setattr({"cfg": cfg, "in": ins, "out": outs}[obj], field, value)


def _faults():
    yield "ABI version", _set("cfg", "abi_version", _cabi.GEO_ABI_VERSION + 1), "ABI version mismatch"
    for v in (_cabi.GEO_HOMOGRAPHY, _cabi.GEO_FUNDAMENTAL, _cabi.GEO_ESSENTIAL, 5, -1):
        yield f"model={v}", _set("cfg", "model", v), "unknown model"
    for v in (0, (1 << 24) + 1):
        yield f"max_iters={v}", _set("cfg", "max_iters", v), "max_iters outside [1, 2^24]"
    for v in (0.0, -1.0, float("inf"), float("nan")):
        yield f"threshold={v}", _set("cfg", "threshold", v), "threshold must be positive"
    for v in (-0.1, 1.5, float("nan")):
        yield f"confidence={v}", _set("cfg", "confidence", v), "confidence outside [0, 1]"
    for v in (-1, _cabi.GEO_AFFINE_MAX_REFINE + 1):
        yield f"refine_iters={v}", _set("cfg", "refine_iters", v), "refine_iters outside [0, GEO_AFFINE_MAX_REFINE]"
    for f in ("B", "M", "N"):
        yield f"{f}<0", _set("in", f, -1), "negative size"
    for f, _ in _cabi.GeoOutputs._fields_:
        yield f"out.{f}", _set("out", f, None), "null output"
    for f in ("kpts0", "kpts1", "matches0"):
        yield f"in.{f}", _set("in", f, None), "null input"


CASES = list(_faults())


@pytest.mark.parametrize("label,fault,what", CASES, ids=[c[0] for c in CASES])
def test_single_fault_gives_its_message(label, fault, what):
    rc, msg = _call(fault)
    assert rc != 0 and msg == f"{ENTRY}: {what}"


def test_valid_models_and_refinement_bounds_reach_the_workspace_check():
    for model in (_cabi.GEO_AFFINE, _cabi.GEO_AFFINE_PARTIAL):
        for r in (0, _cabi.GEO_AFFINE_MAX_REFINE):
            def fault(cfg, ins, outs, model=model, r=r):
                cfg.model, cfg.refine_iters = model, r
            assert _call(fault, ws_short=True)[1] == f"{ENTRY}: workspace too small"


def test_null_arguments():
    lib = _cabi.load()
    cfg, ins, outs = _cabi.GeoAffineConfig(), _cabi.GeoInputs(), _cabi.GeoOutputs()
    for args in ((None, C.byref(ins), C.byref(outs)), (C.byref(cfg), None, C.byref(outs)),
                 (C.byref(cfg), C.byref(ins), None)):
        assert lib.geo_estimate_affine(*args, PTR, 1 << 30, None) != 0
        assert lib.lg_last_error().decode() == f"{ENTRY}: null argument"


def test_workspace_one_byte_short():
    rc, msg = _call(ws_short=True)
    assert rc != 0 and msg == f"{ENTRY}: workspace too small"


def test_empty_masks_may_have_no_storage():
    def fault(cfg, ins, outs):
        ins.M, ins.kpts0, ins.matches0, outs.inliers = 0, None, None, None
    assert _call(fault, ws_short=True)[1] == f"{ENTRY}: workspace too small"


def test_empty_batch_returns_zero():
    assert _call(_set("in", "B", 0))[0] == 0


FNS = [estimate_affine_2d, estimate_affine_partial_2d]


@pytest.mark.parametrize("fn", FNS)
def test_cpu_tensors_raise_runtime_error(fn):
    k = torch.zeros(1, 4, 2)
    with pytest.raises(RuntimeError, match="CUDA"):
        fn(k, k, torch.zeros(1, 4, dtype=torch.int64))


@pytest.mark.parametrize("fn", FNS)
@pytest.mark.parametrize("kw, match", [
    ({"max_iters": 0}, "max_iters"), ({"max_iters": 2.0}, "max_iters"), ({"ransac_reproj_threshold": 0.0}, "threshold"),
    ({"confidence": 1.5}, "confidence"), ({"seed": -1}, "seed"), ({"refine_iters": -1}, "refine_iters"),
    ({"refine_iters": _cabi.GEO_AFFINE_MAX_REFINE + 1}, "refine_iters"), ({"refine_iters": True}, "refine_iters"),
    ({"refine_iters": 1.0}, "refine_iters")])
def test_parameters_are_checked(fn, kw, match, monkeypatch):
    # the input checks pass on tensors that claim a CUDA device; the parameter checks must raise before any launch
    monkeypatch.setattr("lightglue_b200.geometry._check_inputs", lambda *a, **k: None)
    k = torch.zeros(1, 4, 2)
    with pytest.raises(ValueError, match=match):
        fn(k, k, torch.zeros(1, 4, dtype=torch.int64), **kw)


@pytest.mark.parametrize("fn", FNS)
def test_inputs_are_checked(fn):
    k = torch.zeros(1, 4, 2)
    with pytest.raises(ValueError):
        fn("x", k, torch.zeros(1, 4, dtype=torch.int64))
