"""3D rigid and similarity estimation without a GPU: the header's new constants, exports and ``GeoRigidOutputs``
layout, the workspace size, every argument check of ``geo_estimate_rigid`` with its exact message, and the Python
validation of ``estimate_rigid_3d`` and ``estimate_similarity_3d`` (include/geometry_b200.h,
lightglue_b200/geometry.py)."""
import ctypes as C
import os
import re

import pytest
import torch

from lightglue_b200 import _cabi
from lightglue_b200.geometry import estimate_rigid_3d, estimate_similarity_3d
from oracle import rigid_oracle as ro

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PTR = 4096  # any non-null address: every call below fails or returns before it is dereferenced
B, M, N = 2, 16, 12
ENTRY = "geo_estimate_rigid"


def _header():
    with open(os.path.join(ROOT, "include", "geometry_b200.h")) as f:
        return f.read()


def test_constants_match_the_header_and_the_oracle():
    h = _header()
    for name in ("GEO_RIGID_3D", "GEO_SIMILARITY_3D"):
        m = re.search(rf"#define {name} (\d+)\b", h)
        assert m and int(m.group(1)) == getattr(_cabi, name), name
    assert (_cabi.GEO_RIGID_3D, _cabi.GEO_SIMILARITY_3D) == (ro.RIGID, ro.SIMILARITY) == (5, 6)
    m = re.search(r"#define GEO_RIGID_COLLINEAR_EPS (\S+)", h)
    assert m and float(m.group(1)) == ro.COLLINEAR_EPS
    assert re.search(r"#define GEO_ABI_VERSION 1\b", h) and _cabi.GEO_ABI_VERSION == 1


def test_outputs_layout_matches_the_header():
    body = re.search(r"typedef struct GeoRigidOutputs \{(.*?)\} GeoRigidOutputs;", _header(), re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = [d.split()[-1].lstrip("*") for d in body.split(";") if d.strip()]
    assert [f for f, _ in _cabi.GeoRigidOutputs._fields_] == names
    assert names == ["R", "t", "scale", "inliers", "num_inliers", "success", "best_hypothesis", "num_hypotheses"]
    assert C.sizeof(_cabi.GeoRigidOutputs) == 64 and _cabi.GeoRigidOutputs.scale.offset == 16


def test_entry_points_are_declared_and_exported():
    declared = re.findall(r"LG_API \w+\*? (geo_\w+)\(", _header())
    assert "geo_rigid_workspace_bytes" in declared and ENTRY in declared
    assert {"geo_rigid_workspace_bytes", ENTRY} <= set(_cabi.GEO_EXPORTS)
    lib = _cabi.load()
    assert lib.geo_estimate_rigid.argtypes[:3] == [C.POINTER(_cabi.GeoConfig), C.POINTER(_cabi.GeoInputs),
                                                   C.POINTER(_cabi.GeoRigidOutputs)]


def test_workspace_matches_the_carve_and_is_monotone():
    lib = _cabi.load()
    up = lambda x: (x + 255) // 256 * 256  # noqa: E731
    for b, m in ((1, 0), (1, 100), (32, 2048), (265, 300), (1, (1 << 17) + 37)):
        # 24-byte pair records, two compacted float4 points and an int row per match, one chunk of 12-float models
        # and int counts, each 256-byte aligned, plus 256 bytes of base alignment
        want = up(b * 24) + 2 * up(b * m * 16) + up(b * m * 4) + up(b * 256 * 12 * 4) + up(b * 256 * 4) + 256
        got = lib.geo_rigid_workspace_bytes(b, m, 1000)
        assert got == want, (b, m, got, want)
        assert lib.geo_rigid_workspace_bytes(b, m, 1) == lib.geo_rigid_workspace_bytes(b, m, 1 << 24) == got
    for b in (1, 2, 7, 64):
        sizes = [lib.geo_rigid_workspace_bytes(b, m, 1000) for m in (0, 1, 100, 1000, 5000)]
        assert sizes == sorted(sizes), (b, sizes)
    for m in (0, 10, 2048):
        sizes = [lib.geo_rigid_workspace_bytes(b, m, 1000) for b in (0, 1, 2, 33, 500)]
        assert sizes == sorted(sizes), (m, sizes)
    assert lib.geo_rigid_workspace_bytes(-1, 10, 1) == 0 and lib.geo_rigid_workspace_bytes(1, -1, 1) == 0


def _call(fault=lambda cfg, ins, outs: None, ws_short=False):
    lib = _cabi.load()
    cfg = _cabi.GeoConfig(_cabi.GEO_ABI_VERSION, _cabi.GEO_RIGID_3D, 1000, 0, 0.05, 0.99)
    ins = _cabi.GeoInputs(B, M, N, PTR, PTR, PTR)
    outs = _cabi.GeoRigidOutputs(*([PTR] * len(_cabi.GeoRigidOutputs._fields_)))
    fault(cfg, ins, outs)
    bytes_ = lib.geo_rigid_workspace_bytes(max(ins.B, 0), max(ins.M, 0), cfg.max_iters) - (1 if ws_short else 0)
    rc = lib.geo_estimate_rigid(C.byref(cfg), C.byref(ins), C.byref(outs), PTR, bytes_, None)
    return rc, lib.lg_last_error().decode()


def _set(obj, field, value):
    return lambda cfg, ins, outs: setattr({"cfg": cfg, "in": ins, "out": outs}[obj], field, value)


def _faults():
    yield "ABI version", _set("cfg", "abi_version", _cabi.GEO_ABI_VERSION + 1), "ABI version mismatch"
    for v in (_cabi.GEO_HOMOGRAPHY, _cabi.GEO_FUNDAMENTAL, _cabi.GEO_ESSENTIAL, _cabi.GEO_AFFINE,
              _cabi.GEO_AFFINE_PARTIAL, 7, -1):
        yield f"model={v}", _set("cfg", "model", v), "unknown model"
    for v in (0, (1 << 24) + 1):
        yield f"max_iters={v}", _set("cfg", "max_iters", v), "max_iters outside [1, 2^24]"
    for v in (0.0, -1.0, float("inf"), float("nan")):
        yield f"threshold={v}", _set("cfg", "threshold", v), "threshold must be positive"
    for v in (-0.1, 1.5, float("nan")):
        yield f"confidence={v}", _set("cfg", "confidence", v), "confidence outside [0, 1]"
    for f in ("B", "M", "N"):
        yield f"{f}<0", _set("in", f, -1), "negative size"
    for f, _ in _cabi.GeoRigidOutputs._fields_:
        yield f"out.{f}", _set("out", f, None), "null output"
    for f in ("kpts0", "kpts1", "matches0"):
        yield f"in.{f}", _set("in", f, None), "null input"


CASES = list(_faults())


@pytest.mark.parametrize("label,fault,what", CASES, ids=[c[0] for c in CASES])
def test_single_fault_gives_its_message(label, fault, what):
    rc, msg = _call(fault)
    assert rc != 0 and msg == f"{ENTRY}: {what}"


def test_both_models_reach_the_workspace_check():
    for model in (_cabi.GEO_RIGID_3D, _cabi.GEO_SIMILARITY_3D):
        assert _call(_set("cfg", "model", model), ws_short=True)[1] == f"{ENTRY}: workspace too small"


def test_null_arguments():
    lib = _cabi.load()
    cfg, ins, outs = _cabi.GeoConfig(), _cabi.GeoInputs(), _cabi.GeoRigidOutputs()
    for args in ((None, C.byref(ins), C.byref(outs)), (C.byref(cfg), None, C.byref(outs)),
                 (C.byref(cfg), C.byref(ins), None)):
        assert lib.geo_estimate_rigid(*args, PTR, 1 << 30, None) != 0
        assert lib.lg_last_error().decode() == f"{ENTRY}: null argument"


def test_workspace_one_byte_short_or_missing():
    rc, msg = _call(ws_short=True)
    assert rc != 0 and msg == f"{ENTRY}: workspace too small"
    lib = _cabi.load()
    cfg = _cabi.GeoConfig(_cabi.GEO_ABI_VERSION, _cabi.GEO_SIMILARITY_3D, 1000, 0, 0.05, 0.99)
    ins = _cabi.GeoInputs(B, M, N, PTR, PTR, PTR)
    outs = _cabi.GeoRigidOutputs(*([PTR] * 8))
    assert lib.geo_estimate_rigid(C.byref(cfg), C.byref(ins), C.byref(outs), None, 1 << 30, None) != 0
    assert lib.lg_last_error().decode() == f"{ENTRY}: workspace too small"


def test_empty_masks_and_image_1_may_have_no_storage():
    def fault(cfg, ins, outs):
        ins.M, ins.kpts0, ins.matches0, outs.inliers = 0, None, None, None
    assert _call(fault, ws_short=True)[1] == f"{ENTRY}: workspace too small"

    def no_points1(cfg, ins, outs):
        ins.N, ins.kpts1 = 0, None
    assert _call(no_points1, ws_short=True)[1] == f"{ENTRY}: workspace too small"


def test_empty_batch_returns_zero():
    assert _call(_set("in", "B", 0))[0] == 0


FNS = [estimate_rigid_3d, estimate_similarity_3d]


def _args(dim0=3, dim1=3, dtype=torch.float32):
    return torch.zeros(1, 4, dim0, dtype=dtype), torch.zeros(1, 5, dim1, dtype=dtype), torch.zeros(1, 4,
                                                                                                    dtype=torch.int64)


@pytest.mark.parametrize("fn", FNS)
def test_cpu_tensors_raise_runtime_error(fn):
    with pytest.raises(RuntimeError, match="CUDA"):
        fn(*_args(), 0.05)


@pytest.mark.parametrize("fn", FNS)
def test_threshold_is_required(fn):
    with pytest.raises(TypeError, match="ransac_threshold"):
        fn(*_args())


@pytest.mark.parametrize("fn", FNS)
@pytest.mark.parametrize("kw, match", [
    ({"ransac_threshold": 0.0}, r"ransac_threshold=0\.0: a positive distance in points1's units"),
    ({"ransac_threshold": -1.0}, "ransac_threshold"), ({"ransac_threshold": float("inf")}, "ransac_threshold"),
    ({"ransac_threshold": float("nan")}, "ransac_threshold"),
    ({"max_iters": 0}, "max_iters"), ({"max_iters": 2.0}, "max_iters"), ({"confidence": 1.5}, "confidence"),
    ({"seed": -1}, "seed"), ({"seed": 1 << 32}, "seed")])
def test_parameters_are_checked(fn, kw, match, monkeypatch):
    # the input checks pass on tensors that claim a CUDA device; the parameter checks must raise before any launch
    monkeypatch.setattr("lightglue_b200.geometry._check_inputs", lambda *a, **k: None)
    kw = {"ransac_threshold": 0.05, **kw}
    with pytest.raises(ValueError, match=match):
        fn(*_args(), **kw)


class _Cuda0(torch.Tensor):
    """A CPU tensor that reports a CUDA device, so the shape, dtype and device checks can run without a GPU."""

    @property
    def device(self):
        return torch.device("cuda", 0)


class _Cuda1(_Cuda0):
    @property
    def device(self):
        return torch.device("cuda", 1)


@pytest.mark.parametrize("fn", FNS)
@pytest.mark.parametrize("case, match", [
    ("2d0", r"points0 \(1, 4, 2\) and points1 \(1, 5, 3\): expected \[B, M, 3\] and \[B, N, 3\]"),
    ("2d1", r"points0 \(1, 4, 3\) and points1 \(1, 5, 2\): expected \[B, M, 3\] and \[B, N, 3\]"),
    ("int", "points0 and points1 must be floating point$"),
    ("m32", "matches0 must be int64"),
    ("rows", r"matches0 \(1, 3\): expected \[B, M\] of points0"),
    ("device", "points0, points1 and matches0 must be on one device"),
    ("type", "points1 must be a torch.Tensor")])
def test_inputs_are_checked(fn, case, match):
    p0, p1, m0 = _args(2 if case == "2d0" else 3, 2 if case == "2d1" else 3)
    if case == "int":
        p0 = p0.to(torch.int32)
    if case == "m32":
        m0 = m0.to(torch.int32)
    if case == "rows":
        m0 = m0[:, :3]
    p0, p1 = p0.as_subclass(_Cuda0), p1.as_subclass(_Cuda0)
    m0 = m0.as_subclass(_Cuda1 if case == "device" else _Cuda0)
    if case == "type":
        p1 = p1.numpy()
    with pytest.raises(ValueError, match=match):
        fn(p0, p1, m0, 0.05)
