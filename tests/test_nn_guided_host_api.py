"""Guided nearest-neighbour matching without a GPU: the header's new exports, constants and ``NnGuide`` layout, the
argument checks of ``nn_match_guided`` and of ``NearestNeighborMatcher.forward(..., F= / H=)``, and the guided
workspace size (include/nn_b200.h, lightglue_b200/nn_matcher.py)."""
import ctypes
import os
import re

import pytest
import torch

from lightglue_b200 import NearestNeighborMatcher, _cabi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header():
    with open(os.path.join(ROOT, "include", "nn_b200.h")) as f:
        return f.read()


def test_guided_entry_points_follow_the_existing_ones_in_header_order():
    declared = re.findall(r"LG_API \w+\*? (nn_\w+)\(", _header())
    assert declared[-2:] == ["nn_guided_workspace_bytes", "nn_match_guided"]
    assert list(_cabi.NN_EXPORTS)[-2:] == declared[-2:]
    lib = _cabi.load()
    assert lib.nn_match_guided.argtypes[3] is ctypes.POINTER(_cabi.NnGuide)


def test_guide_constants_match_the_header_and_the_estimators():
    h = _header()
    for name, value in (("NN_GUIDE_H", _cabi.NN_GUIDE_H), ("NN_GUIDE_F", _cabi.NN_GUIDE_F)):
        m = re.search(rf"#define {name} (\d+)", h)
        assert m and int(m.group(1)) == value, name
    assert (_cabi.NN_GUIDE_H, _cabi.NN_GUIDE_F) == (_cabi.GEO_HOMOGRAPHY, _cabi.GEO_FUNDAMENTAL)
    assert re.search(r"#define NN_ABI_VERSION 1\b", h)


def test_guide_layout_matches_the_header():
    body = re.search(r"typedef struct NnGuide \{(.*?)\} NnGuide;", _header(), re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = [n for decl in body.split(";") for n in re.findall(r"\**(\w+)\s*(?:,|$)", decl.strip())]
    assert [f for f, _ in _cabi.NnGuide._fields_] == names
    assert _cabi.NnGuide.model.offset == 8 and _cabi.NnGuide.max_error.offset == 40
    assert ctypes.sizeof(_cabi.NnGuide) == 48


def test_guided_workspace_adds_the_gate_records():
    lib = _cabi.load()
    for b, m, n, d in ((1, 100, 100, 128), (32, 2048, 2048, 128), (8, 8192, 8192, 256), (3, 300, 5000, 64)):
        plain, guided = lib.nn_workspace_bytes(b, m, n, d), lib.nn_guided_workspace_bytes(b, m, n, d)
        lp = (max(m, n) + 127) // 128 * 128
        g_max = max(_cabi.NN_GROUP_ROWS // lp, 1)
        groups = -(-b // g_max)
        g = -(-b // groups)
        # six fp32 fields per row of both sides of one group, one flag per pair, alignment padding
        assert 24 * 2 * g * lp + 4 * g <= guided - plain <= 24 * 2 * g * lp + 4 * g + 512
    big = lib.nn_guided_workspace_bytes(32, 8192, 8192, 256)
    assert 0 < big < 32 * 8192 * 8192 * 4 // 32


@pytest.mark.parametrize("d", [0, 32, 96, 576])
def test_guided_workspace_rejects_a_bad_dim(d):
    assert _cabi.load().nn_guided_workspace_bytes(4, 100, 100, d) == 0


def _fake_call(guide, cfg=None, ins=None):
    lib = _cabi.load()
    cfg = cfg or _cabi.NnConfig(_cabi.NN_ABI_VERSION, 128, 1, 0.8, 0.0)
    # never dereferenced: every call below fails a check before any launch
    ins = ins or _cabi.NnInputs(1, 10, 10, 1024, 2048, None, None)
    outs = _cabi.NnOutputs(*([4096] * 7))
    g = None if guide is None else ctypes.byref(guide)
    rc = lib.nn_match_guided(ctypes.c_void_p(1), ctypes.byref(cfg), ctypes.byref(ins), g, ctypes.byref(outs), None, 0,
                             None)
    return rc, lib.lg_last_error()


def _guide(**kw):
    args = {"kind": _cabi.NN_GUIDE_F, "model": 8192, "valid": None, "kpts0": 16384, "kpts1": 32768, "max_error": 4.0}
    args.update(kw)
    return _cabi.NnGuide(**args)


@pytest.mark.parametrize("guide, what", [
    (None, b"null"),
    (_guide(kind=2), b"kind"),
    (_guide(kind=-1), b"kind"),
    (_guide(max_error=0.0), b"max_error"),
    (_guide(max_error=-1.0), b"max_error"),
    (_guide(max_error=float("inf")), b"max_error"),
    (_guide(max_error=float("nan")), b"max_error"),
    (_guide(model=None), b"null"),
    (_guide(kpts0=None), b"null"),
    (_guide(kpts1=None), b"null"),
    (_guide(model=8196), b"aligned"),
    (_guide(kpts0=16388), b"aligned"),
    (_guide(kpts1=32772), b"aligned"),
    (_guide(), b"workspace"),
])
def test_nn_match_guided_rejects_bad_arguments_before_any_launch(guide, what):
    rc, msg = _fake_call(guide)
    assert rc != 0 and what in msg and msg.startswith(b"nn_match_guided: "), msg


def test_nn_match_guided_shares_nn_matchs_checks():
    for cfg, what in ((_cabi.NnConfig(_cabi.NN_ABI_VERSION + 1, 128, 1, 0.8, 0.0), b"ABI"),
                      (_cabi.NnConfig(_cabi.NN_ABI_VERSION, 96, 1, 0.8, 0.0), b"dim"),
                      (_cabi.NnConfig(_cabi.NN_ABI_VERSION, 128, 1, 1.5, 0.0), b"ratio"),
                      (_cabi.NnConfig(_cabi.NN_ABI_VERSION, 128, 1, 0.8, float("nan")), b"distance")):
        rc, msg = _fake_call(_guide(), cfg=cfg)
        assert rc != 0 and what in msg, msg
    rc, msg = _fake_call(_guide(), ins=_cabi.NnInputs(1, 10, 10, 1032, 2048, None, None))
    assert rc != 0 and b"16-byte" in msg
    # an empty batch is a no-op once the arguments pass; an empty image needs no keypoints of its own
    rc, _ = _fake_call(_guide(kpts0=None, kpts1=None), ins=_cabi.NnInputs(0, 10, 10, None, None, None, None))
    assert rc == 0
    rc, msg = _fake_call(_guide(kpts1=None), ins=_cabi.NnInputs(1, 10, 0, 1024, None, None, None))
    assert rc != 0 and b"workspace" in msg


def _data(b=2, m=10, n=12, d=128, kp=True):
    data = {"image0": {"descriptors": torch.zeros(b, m, d)}, "image1": {"descriptors": torch.zeros(b, n, d)}}
    if kp:
        data["image0"]["keypoints"] = torch.zeros(b, m, 2)
        data["image1"]["keypoints"] = torch.zeros(b, n, 2)
    return data


@pytest.mark.parametrize("kw, what", [
    ({"F": torch.eye(3).expand(2, 3, 3), "H": torch.eye(3).expand(2, 3, 3)}, "at most one"),
    ({"F": torch.eye(3)}, r"\(3, 3\)"),
    ({"H": torch.eye(3).expand(3, 3, 3)}, r"\(3, 3, 3\)"),
    ({"H": torch.zeros(2, 9)}, r"\(2, 9\)"),
    ({"F": torch.zeros(2, 3, 3, dtype=torch.int64)}, "float"),
    ({"F": [[0.0] * 3] * 3}, "list"),
    ({"H": torch.eye(3).expand(2, 3, 3), "max_error": 0.0}, "max_error=0.0"),
    ({"H": torch.eye(3).expand(2, 3, 3), "max_error": -2}, "max_error=-2"),
    ({"H": torch.eye(3).expand(2, 3, 3), "max_error": float("inf")}, "max_error=inf"),
    ({"H": torch.eye(3).expand(2, 3, 3), "max_error": float("nan")}, "max_error=nan"),
    ({"H": torch.eye(3).expand(2, 3, 3), "max_error": "far"}, "max_error='far'"),
    ({"H": torch.eye(3).expand(2, 3, 3), "valid": torch.ones(3)}, r"valid \(3,\)"),
    ({"H": torch.eye(3).expand(2, 3, 3), "valid": torch.ones(2, 1)}, r"valid \(2, 1\)"),
])
def test_bad_guided_arguments_are_a_value_error(kw, what):
    with pytest.raises(ValueError, match=what):
        NearestNeighborMatcher()(_data(), **kw)


@pytest.mark.parametrize("image, shape", [("image0", None), ("image1", None), ("image0", (2, 10, 3)),
                                          ("image1", (2, 11, 2)), ("image1", (1, 12, 2))])
def test_guided_matching_needs_the_keypoints(image, shape):
    data = _data()
    if shape is None:
        del data[image]["keypoints"]
    else:
        data[image]["keypoints"] = torch.zeros(shape)
    with pytest.raises(ValueError, match=image):
        NearestNeighborMatcher()(data, H=torch.eye(3).expand(2, 3, 3))


def test_guided_cpu_tensors_are_a_runtime_error():
    with pytest.raises(RuntimeError, match="CUDA"):
        NearestNeighborMatcher()(_data(), F=torch.zeros(2, 3, 3, dtype=torch.float64), valid=torch.ones(2))


def test_unguided_call_needs_no_keypoints():
    with pytest.raises(RuntimeError, match="CUDA"):  # past every check: the CPU tensors are the only objection
        NearestNeighborMatcher()(_data(kp=False))
