"""The argument checks of the six geometry C entry points, without a GPU: every single fault fails with its exact
``"<entry>: <what>"`` message, an empty mask may have no storage, and B = 0 returns 0 (include/geometry_b200.h)."""
import ctypes as C

import pytest

from lightglue_b200 import _cabi

PTR = 4096  # any non-null address: every call below fails or returns before it is dereferenced
B, M, N = 2, 16, 12

# entry -> (workspace function, config, inputs, outputs, wrapper of the outputs (LO), model, checks distance_threshold,
#           intrinsics, name of image 1's input)
ENTRIES = {
    "geo_estimate": ("geo_workspace_bytes", _cabi.GeoConfig, _cabi.GeoInputs, _cabi.GeoOutputs, None,
                     _cabi.GEO_HOMOGRAPHY, False, (), "kpts1"),
    "geo_homography_lo": ("geo_lo_homography_workspace_bytes", _cabi.GeoConfig, _cabi.GeoInputs, _cabi.GeoOutputs,
                          _cabi.GeoLoOutputs, _cabi.GEO_HOMOGRAPHY, False, (), "kpts1"),
    "geo_fundamental_lo": ("geo_lo_fundamental_workspace_bytes", _cabi.GeoConfig, _cabi.GeoInputs, _cabi.GeoOutputs,
                           _cabi.GeoLoOutputs, _cabi.GEO_FUNDAMENTAL, False, (), "kpts1"),
    "geo_relative_pose": ("geo_pose_workspace_bytes", _cabi.GeoPoseConfig, _cabi.GeoPoseInputs, _cabi.GeoPoseOutputs,
                          None, None, True, ("K0", "K1"), "kpts1"),
    "geo_relative_pose_lo": ("geo_lo_pose_workspace_bytes", _cabi.GeoLoPoseConfig, _cabi.GeoPoseInputs,
                             _cabi.GeoPoseOutputs, _cabi.GeoLoPoseOutputs, None, True, ("K0", "K1"), "kpts1"),
    "geo_absolute_pose": ("geo_pnp_workspace_bytes", _cabi.GeoPnpConfig, _cabi.GeoPnpInputs, _cabi.GeoPnpOutputs,
                          None, None, False, ("K0",), "points3d1"),
}
WRONG_MODEL = {"geo_estimate": (7, "unknown model"),
               "geo_homography_lo": (_cabi.GEO_FUNDAMENTAL, "model must be GEO_HOMOGRAPHY"),
               "geo_fundamental_lo": (_cabi.GEO_HOMOGRAPHY, "model must be GEO_FUNDAMENTAL")}
LO = ("geo_homography_lo", "geo_fundamental_lo", "geo_relative_pose_lo")


def _call(entry, fault=lambda cfg, ins, outs, lo: None, ws_short=False):
    """Calls entry on valid arguments changed by fault; returns (rc, error message)."""
    ws_fn, cfg_t, in_t, out_t, lo_t, model, _, intr, name1 = ENTRIES[entry]
    lib = _cabi.load()
    cfg = cfg_t()
    cfg.abi_version, cfg.max_iters, cfg.seed, cfg.threshold, cfg.confidence = _cabi.GEO_ABI_VERSION, 1000, 0, 1.0, 0.99
    if model is not None:
        cfg.model = model
    if hasattr(cfg, "distance_threshold"):
        cfg.distance_threshold = 50.0
    ins = in_t(B, M, N)
    for f in ("kpts0", name1, "matches0") + intr:
        setattr(ins, f, PTR)
    outs = out_t(*([PTR] * len(out_t._fields_)))
    lo = lo_t(outs, PTR, PTR) if lo_t else None
    fault(cfg, ins, lo.pose if lo_t is _cabi.GeoLoPoseOutputs else lo.geo if lo else outs, lo)
    bytes_ = getattr(lib, ws_fn)(max(ins.B, 0), max(ins.M, 0), cfg.max_iters) - (1 if ws_short else 0)
    args = [C.byref(cfg), C.byref(ins), C.byref(lo if lo else outs), PTR, bytes_, None]
    rc = getattr(lib, entry)(*args)
    return rc, lib.lg_last_error().decode()


def _set(obj, field, value):
    return lambda cfg, ins, outs, lo: setattr({"cfg": cfg, "in": ins, "out": outs, "lo": lo}[obj], field, value)


def _faults(entry):
    _, _, in_t, out_t, lo_t, model, distance, intr, name1 = ENTRIES[entry]
    yield "ABI version", _set("cfg", "abi_version", _cabi.GEO_ABI_VERSION + 1), "ABI version mismatch"
    if entry in WRONG_MODEL:
        yield "model", _set("cfg", "model", WRONG_MODEL[entry][0]), WRONG_MODEL[entry][1]
    for v in (0, (1 << 24) + 1):
        yield f"max_iters={v}", _set("cfg", "max_iters", v), "max_iters outside [1, 2^24]"
    for v in (0.0, float("inf"), float("nan")):
        yield f"threshold={v}", _set("cfg", "threshold", v), "threshold must be positive"
    for v in (1.5, float("nan")):
        yield f"confidence={v}", _set("cfg", "confidence", v), "confidence outside [0, 1]"
    if distance:
        for v in (0.0, float("inf"), float("nan")):
            yield (f"distance_threshold={v}", _set("cfg", "distance_threshold", v),
                   "distance_threshold must be positive")
    for f in ("B", "M", "N"):
        yield f"{f}<0", _set("in", f, -1), "negative size"
    if entry in LO:
        yield "M>GEO_LO_MAX_MATCHES", _set("in", "M", _cabi.GEO_LO_MAX_MATCHES + 1), "M above GEO_LO_MAX_MATCHES"
    for f, _ in out_t._fields_:
        yield f"out.{f}", _set("out", f, None), "null output"
    if lo_t:
        for f in ("num_local_optimizations", "cost"):
            yield f"out.{f}", _set("lo", f, None), "null output"
    for f in intr:
        yield f"in.{f}", _set("in", f, None), "null intrinsics"
    for f in ("kpts0", name1, "matches0"):
        yield f"in.{f}", _set("in", f, None), "null input"


CASES = [(e, label, fault, what) for e in ENTRIES for label, fault, what in _faults(e)]


@pytest.mark.parametrize("entry,label,fault,what", CASES, ids=[f"{e}-{label}" for e, label, _, _ in CASES])
def test_single_fault_gives_its_message(entry, label, fault, what):
    rc, msg = _call(entry, fault)
    assert rc != 0 and msg == f"{entry}: {what}"


@pytest.mark.parametrize("entry", ENTRIES)
def test_null_arguments(entry):
    lib = _cabi.load()
    ws_fn, cfg_t, in_t, out_t, lo_t = ENTRIES[entry][:5]
    cfg, ins, outs = cfg_t(), in_t(), (lo_t or out_t)()
    for args in ((None, C.byref(ins), C.byref(outs)), (C.byref(cfg), None, C.byref(outs)),
                 (C.byref(cfg), C.byref(ins), None)):
        assert getattr(lib, entry)(*args, PTR, 1 << 30, None) != 0
        assert lib.lg_last_error().decode() == f"{entry}: null argument"


@pytest.mark.parametrize("entry", ENTRIES)
def test_workspace_one_byte_short(entry):
    rc, msg = _call(entry, ws_short=True)
    assert rc != 0 and msg == f"{entry}: workspace too small"


@pytest.mark.parametrize("entry", ENTRIES)
def test_empty_masks_may_have_no_storage(entry):
    # with M = 0 the null masks and inputs pass, and the call reaches the workspace check
    def fault(cfg, ins, outs, lo):
        ins.M = 0
        for f in ("inliers", "pose_inliers", "kpts0", "matches0"):
            for o in (ins, outs):
                if hasattr(o, f):
                    setattr(o, f, None)
    rc, msg = _call(entry, fault, ws_short=True)
    assert rc != 0 and msg == f"{entry}: workspace too small"


@pytest.mark.parametrize("entry", ENTRIES)
def test_empty_batch_returns_zero(entry):
    assert _call(entry, _set("in", "B", 0))[0] == 0
