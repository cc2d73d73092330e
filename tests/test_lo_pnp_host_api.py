"""LO-RANSAC absolute pose without a GPU: the header's new exports and struct, the shared constants and defaults, the
workspace, every single argument fault with its exact C message, and the Python checks (include/geometry_b200.h,
lightglue_b200/geometry.py)."""
import ctypes as C
import inspect
import os
import re

import pytest
import torch

from lightglue_b200 import _cabi
from lightglue_b200.geometry import estimate_absolute_pose, estimate_absolute_pose_lo
from oracle import lo_pnp_oracle as la

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRY = "geo_absolute_pose_lo"
PTR = 4096  # any non-null address: every call below fails or returns before it is dereferenced
B, M, N = 2, 16, 12


def _header():
    with open(os.path.join(ROOT, "include", "geometry_b200.h")) as f:
        return f.read()


def test_entry_points_are_exported():
    h = _header()
    for s in ("geo_lo_pnp_workspace_bytes", ENTRY):
        assert s in _cabi.GEO_EXPORTS and re.search(rf"LG_API \w+ {s}\(", h), s
    assert re.search(r"LG_API int geo_absolute_pose_lo\(const GeoPnpConfig\* cfg, const GeoPnpInputs\* in, "
                     r"GeoLoPnpOutputs\* out,", h)
    lib = _cabi.load()
    for s in ("geo_lo_pnp_workspace_bytes", ENTRY):
        assert getattr(lib, s).argtypes is not None, s


def test_outputs_struct_matches_the_header():
    body = re.search(r"typedef struct GeoLoPnpOutputs \{(.*?)\} GeoLoPnpOutputs;", _header(), re.S).group(1)
    fields = re.findall(r"^\s*[\w ]+?\**\s*\**(\w+);", body, re.M)
    assert fields == [f for f, _ in _cabi.GeoLoPnpOutputs._fields_] == ["pnp", "num_local_optimizations", "cost"]
    assert re.search(r"GeoPnpOutputs pnp;", body) and re.search(r"int32_t\* num_local_optimizations;", body)
    assert re.search(r"int64_t\* cost;", body)
    assert _cabi.GeoLoPnpOutputs._fields_[0][1] is _cabi.GeoPnpOutputs
    assert C.sizeof(_cabi.GeoLoPnpOutputs) == C.sizeof(_cabi.GeoPnpOutputs) + 2 * C.sizeof(C.c_void_p)
    assert _cabi.GeoLoPnpOutputs.cost.offset == C.sizeof(_cabi.GeoPnpOutputs) + C.sizeof(C.c_void_p)


def test_constants_are_shared_with_the_other_lo_estimators():
    h = _header()
    for name, value in (("GEO_LO_QSCALE", la.QSCALE), ("GEO_LO_STEPS", la.STEPS), ("GEO_LO_FINAL_STEPS", la.FINAL_STEPS)):
        assert re.search(rf"#define {name} {value}\b", h), name
    assert la.LAMBDA0 == 1e-3 and re.search(r"#define GEO_LO_LAMBDA0 1e-3\b", h)
    assert re.search(r"#define GEO_ABI_VERSION 1\b", h) and _cabi.GEO_ABI_VERSION == 1
    for s in ("LA1", "LA2", "LA3", "LA4", "LA5", "LA6", "LA7", "LA8"):
        assert re.search(rf"\* {s}\. ", h), s


def test_workspace_does_not_grow_with_the_budget():
    ws = _cabi.load().geo_lo_pnp_workspace_bytes
    assert ws(32, 2048, 100) == ws(32, 2048, 1000) == ws(32, 2048, 1 << 24) > 0
    assert ws(32, 4096, 1000) > ws(32, 2048, 1000) > _cabi.load().geo_pnp_workspace_bytes(32, 2048, 1000)
    assert ws(-1, 16, 100) == 0 and ws(2, -1, 100) == 0


def test_defaults_equal_the_plain_estimator():
    a = inspect.signature(estimate_absolute_pose).parameters
    b = inspect.signature(estimate_absolute_pose_lo).parameters
    assert list(a) == list(b)
    assert all(a[k].default == b[k].default for k in a)


# ------------------------------------------------------------------------------------------------- C argument checks


def _call(fault=lambda cfg, ins, outs, lo: None, ws_short=False):
    """Calls geo_absolute_pose_lo on valid arguments changed by fault; returns (rc, error message)."""
    lib = _cabi.load()
    cfg = _cabi.GeoPnpConfig(_cabi.GEO_ABI_VERSION, 1000, 0, 0, 8.0, 0.99)
    ins = _cabi.GeoPnpInputs(B, M, N, PTR, PTR, PTR, PTR)
    outs = _cabi.GeoPnpOutputs(*([PTR] * len(_cabi.GeoPnpOutputs._fields_)))
    lo = _cabi.GeoLoPnpOutputs(outs, PTR, PTR)
    fault(cfg, ins, lo.pnp, lo)
    bytes_ = lib.geo_lo_pnp_workspace_bytes(max(ins.B, 0), max(ins.M, 0), cfg.max_iters) - (1 if ws_short else 0)
    rc = getattr(lib, ENTRY)(C.byref(cfg), C.byref(ins), C.byref(lo), PTR, bytes_, None)
    return rc, lib.lg_last_error().decode()


def _set(obj, field, value):
    return lambda cfg, ins, outs, lo: setattr({"cfg": cfg, "in": ins, "out": outs, "lo": lo}[obj], field, value)


def _faults():
    yield "ABI version", _set("cfg", "abi_version", _cabi.GEO_ABI_VERSION + 1), "ABI version mismatch"
    for v in (0, -1, (1 << 24) + 1):
        yield f"max_iters={v}", _set("cfg", "max_iters", v), "max_iters outside [1, 2^24]"
    for v in (0.0, -1.0, float("inf"), float("nan")):
        yield f"threshold={v}", _set("cfg", "threshold", v), "threshold must be positive"
    for v in (1.5, -0.1, float("nan")):
        yield f"confidence={v}", _set("cfg", "confidence", v), "confidence outside [0, 1]"
    for f in ("B", "M", "N"):
        yield f"{f}<0", _set("in", f, -1), "negative size"
    yield "M>GEO_LO_MAX_MATCHES", _set("in", "M", _cabi.GEO_LO_MAX_MATCHES + 1), "M above GEO_LO_MAX_MATCHES"
    for f, _ in _cabi.GeoPnpOutputs._fields_:
        yield f"out.{f}", _set("out", f, None), "null output"
    for f in ("num_local_optimizations", "cost"):
        yield f"out.{f}", _set("lo", f, None), "null output"
    yield "in.K0", _set("in", "K0", None), "null intrinsics"
    for f in ("kpts0", "points3d1", "matches0"):
        yield f"in.{f}", _set("in", f, None), "null input"


CASES = list(_faults())


@pytest.mark.parametrize("label,fault,what", CASES, ids=[c[0] for c in CASES])
def test_single_fault_gives_its_message(label, fault, what):
    rc, msg = _call(fault)
    assert rc != 0 and msg == f"{ENTRY}: {what}"


def test_null_arguments():
    lib = _cabi.load()
    cfg, ins, outs = _cabi.GeoPnpConfig(), _cabi.GeoPnpInputs(), _cabi.GeoLoPnpOutputs()
    for args in ((None, C.byref(ins), C.byref(outs)), (C.byref(cfg), None, C.byref(outs)),
                 (C.byref(cfg), C.byref(ins), None)):
        assert getattr(lib, ENTRY)(*args, PTR, 1 << 30, None) != 0
        assert lib.lg_last_error().decode() == f"{ENTRY}: null argument"


def test_workspace_one_byte_short():
    rc, msg = _call(ws_short=True)
    assert rc != 0 and msg == f"{ENTRY}: workspace too small"


def test_the_row_bound_passes_the_size_checks():
    # M = GEO_LO_MAX_MATCHES passes the size checks and the pointer checks, and stops at the workspace
    rc, msg = _call(_set("in", "M", _cabi.GEO_LO_MAX_MATCHES), ws_short=True)
    assert rc != 0 and msg == f"{ENTRY}: workspace too small"


def test_empty_masks_and_points_may_have_no_storage():
    # with M = 0 the null mask and inputs pass, and with N = 0 the null points3d1: the call reaches the workspace check
    def fault(cfg, ins, outs, lo):
        ins.M, ins.N = 0, 0
        outs.inliers = ins.kpts0 = ins.matches0 = ins.points3d1 = None
    rc, msg = _call(fault, ws_short=True)
    assert rc != 0 and msg == f"{ENTRY}: workspace too small"


def test_empty_batch_returns_zero():
    assert _call(_set("in", "B", 0))[0] == 0


# ------------------------------------------------------------------------------------------------------ Python checks


def _inputs(b=2, m=16, n=12):
    return torch.rand(b, m, 2), torch.rand(b, n, 3), torch.randint(-1, n, (b, m)), torch.eye(3, dtype=torch.float64)


def test_cpu_tensors_raise():
    with pytest.raises(RuntimeError):
        estimate_absolute_pose_lo(*_inputs())


@pytest.mark.parametrize("case", ["kpts0_rank", "matches_dtype", "batch", "not_tensor", "points_width", "k_shape",
                                  "k_dtype"])
def test_bad_shapes_and_dtypes_raise_value_error(case, monkeypatch):
    k0, p3, m0, K = _inputs()
    bad = {
        "kpts0_rank": (k0[0], p3, m0, K),
        "matches_dtype": (k0, p3, m0.to(torch.int32), K),
        "batch": (k0, p3[:1], m0, K),
        "not_tensor": (k0.numpy(), p3, m0, K),
        "points_width": (k0, torch.rand(2, 12, 2), m0, K),
        "k_shape": (k0, p3, m0, torch.eye(3, dtype=torch.float64).expand(3, 3, 3)),
        "k_dtype": (k0, p3, m0, torch.eye(3, dtype=torch.int64)),
    }[case]
    # shapes and dtypes are checked before any device work: CPU tensors posing as CUDA ones reach those checks
    monkeypatch.setattr(torch.Tensor, "device", property(lambda self: torch.device("cuda", 0)))
    with pytest.raises(ValueError):
        estimate_absolute_pose_lo(*bad)


@pytest.mark.parametrize("kw", [dict(max_iters=0), dict(max_iters=1.5), dict(max_iters=(1 << 24) + 1),
                                dict(ransac_reproj_threshold=0.0), dict(ransac_reproj_threshold=-1.0),
                                dict(ransac_reproj_threshold=float("inf")), dict(confidence=1.5),
                                dict(confidence=-0.1), dict(seed=-1), dict(seed=1 << 32), dict(seed=1.0)])
def test_bad_parameters_raise_value_error(kw, monkeypatch):
    monkeypatch.setattr(torch.Tensor, "device", property(lambda self: torch.device("cuda", 0)))
    with pytest.raises(ValueError):
        estimate_absolute_pose_lo(*_inputs(), **kw)


def test_too_many_rows_raise_value_error(monkeypatch):
    monkeypatch.setattr(torch.Tensor, "device", property(lambda self: torch.device("cuda", 0)))
    m = _cabi.GEO_LO_MAX_MATCHES + 1
    with pytest.raises(ValueError, match="rows per pair"):
        estimate_absolute_pose_lo(torch.zeros(1, m, 2), torch.zeros(1, 4, 3), torch.full((1, m), -1),
                                  torch.eye(3, dtype=torch.float64))
