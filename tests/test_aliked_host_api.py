"""Host-side contract of the ALIKED extractor (include/aliked_b200.h, lightglue_b200/aliked.py); no GPU needed."""
import ctypes as C
import os
import re

import pytest
import torch

from lightglue_b200 import _cabi
from lightglue_b200.aliked import ALIKED
from oracle import aliked_synth as als

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "aliked")


def test_header_symbols_equal_exports_and_are_exported():
    with open(os.path.join(ROOT, "include", "aliked_b200.h")) as f:
        hdr = f.read()
    syms = tuple(re.findall(r"LG_API\s+[\w\s\*]+?\b(al_\w+)\s*\(", hdr))
    assert sorted(syms) == sorted(_cabi.AL_EXPORTS)
    lib = _cabi.load()
    for s in _cabi.AL_EXPORTS:
        assert hasattr(lib, s), s
        assert getattr(lib, s).argtypes is not None, s


@pytest.mark.parametrize("model_name", sorted(ALIKED.cfgs))
def test_blob_size_is_parameters_plus_bn_statistics(model_name):
    m = ALIKED(model_name=model_name, weights=None)
    n_param = sum(p.numel() for p in m.parameters())
    n_stats = sum(b.numel() for k, b in m.named_buffers() if k.endswith(("running_mean", "running_var")))
    cfg = m._config()
    assert _cabi.load().al_weight_blob_floats(C.byref(cfg)) == n_param + n_stats == m._blob().numel()


@pytest.mark.parametrize("model_name", sorted(ALIKED.cfgs))
def test_state_dict_keys_equal_the_reference(model_name):
    fixtures = {"aliked-t16": "al_t16", "aliked-n32": "al_n32"}
    fix = torch.load(os.path.join(GOLDEN, fixtures.get(model_name, "al_240x320") + ".pt"), weights_only=False)
    ref = [(k, tuple(s)) for k, s in fix["state_dict_layout"]]
    if model_name in fixtures:
        ours = [(k, tuple(v.shape)) for k, v in ALIKED(model_name=model_name, weights=None).state_dict().items()]
        assert ours == ref
    else:  # aliked-n16 / n16rot share the fixture's (n16) layout
        assert [k for k, _ in ALIKED(model_name=model_name, weights=None).state_dict().items()] == [k for k, _ in ref]
    # the synthetic weights load strictly
    ALIKED(model_name=model_name, weights=None).load_state_dict(als.make_aliked_state_dict(model_name), strict=True)


def test_cpu_tensor_raises():
    m = ALIKED(weights=None)
    with pytest.raises(RuntimeError):
        m({"image": torch.rand(1, 3, 32, 32)})


def test_missing_weights_raise(tmp_path, monkeypatch):
    monkeypatch.setenv("LIGHTGLUE_WEIGHTS_DIR", str(tmp_path))
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path))
    with pytest.raises(FileNotFoundError):
        ALIKED(model_name="aliked-n16")


def test_weights_found_in_weights_dir(tmp_path, monkeypatch):
    torch.save(als.make_aliked_state_dict("aliked-t16"), tmp_path / "aliked-t16.pth")
    monkeypatch.setenv("LIGHTGLUE_WEIGHTS_DIR", str(tmp_path))
    m = ALIKED(model_name="aliked-t16")
    assert torch.equal(m.desc_head.agg_weights, als.make_aliked_state_dict("aliked-t16")["desc_head.agg_weights"])


def test_unknown_model_name_raises():
    with pytest.raises(ValueError):
        ALIKED(model_name="aliked-x99", weights=None)


# ---------------------------------------------------------------------------------------------- workspace layout
LAYOUT_NAMES = ["img", "ta", "x1", "s1", "invn", "p1", "t2", "d2", "x2", "a2", "p2", "o3", "t3", "d3", "x3", "a3",
                "p3", "o4", "t4", "d4", "x4", "a4", "score", "nms", "kpn", "mean", "cnt", "sel_pos", "sel_score", "n_sel"]


def al_layout(cfg, b, h, w):
    """{name: (byte offset, bytes)} of al_workspace_layout and its total."""
    n = _cabi.AL_LAYOUT_BUFFERS
    off, size = (C.c_int64 * n)(), (C.c_int64 * n)()
    total = _cabi.load().al_workspace_layout(C.byref(cfg), b, h, w, off, size)
    return {k: (off[i], size[i]) for i, k in enumerate(LAYOUT_NAMES)}, total


def _expected_floats(model_name, b, h, w, cap):
    c1, c2, c3, c4, dim, _, _ = ALIKED.cfgs[model_name]
    hp, wp = -(-h // 32) * 32, -(-w // 32) * 32
    p0, q, px = b * hp * wp, dim // 4, b * h * w
    p1, p2, p3 = p0 // 4, p0 // 64, p0 // 1024
    return {"img": 3 * p0, "ta": max(c1, 8) * p0, "x1": c1 * p0, "s1": 8 * p0, "invn": p0,
            "p1": c1 * p1, "t2": c2 * p1, "d2": c2 * p1, "x2": c2 * p1, "a2": q * p1,
            "p2": c2 * p2, "o3": 18 * p2, "t3": c3 * p2, "d3": c3 * p2, "x3": c3 * p2, "a3": q * p2,
            "p3": c3 * p3, "o4": 18 * p3, "t4": c4 * p3, "d4": c4 * p3, "x4": c4 * p3, "a4": q * p3,
            "score": px, "nms": px, "kpn": 2 * b * cap, "mean": b, "cnt": b, "sel_pos": b * cap, "sel_score": b * cap,
            "n_sel": b}


# (model, conf, B, H, W): t16 / n16 / n32, odd pads, a 1x1 level 3, top-k and threshold capacities
LAYOUT_CASES = [("aliked-t16", {}, 1, 8, 8), ("aliked-t16", dict(max_num_keypoints=100), 2, 33, 47),
                ("aliked-n16", {}, 3, 240, 320), ("aliked-n16", dict(max_num_keypoints=50, detection_threshold=-1), 1, 100, 37),
                ("aliked-n32", {}, 1, 203, 317), ("aliked-n32", {}, 2, 768, 1024)]


@pytest.mark.parametrize("model_name,conf,b,h,w", LAYOUT_CASES)
def test_workspace_layout_buffers(model_name, conf, b, h, w):
    """Every buffer 256-aligned, of its shape's size and disjoint from the others; the total is the bump carve of the
    listed buffers plus DKD's scratch (three NMS planes, the candidate list and the row scan), 256-aligned."""
    cfg = ALIKED(model_name=model_name, weights=None, **conf)._config()
    lay, total = al_layout(cfg, b, h, w)
    k = conf.get("max_num_keypoints", -1)
    cap = min(k if k > 0 else 20000, h * w)
    want = _expected_floats(model_name, b, h, w, cap)
    for name, (o, n) in lay.items():
        assert o % 256 == 0, name
        assert n == 4 * want[name], (name, n, 4 * want[name])
    spans = sorted(lay.values())
    for (o0, n0), (o1, _) in zip(spans, spans[1:]):
        assert o0 + n0 <= o1
    # the carve's order, scratch (None: its float count) between the listed buffers
    px = b * h * w
    order = LAYOUT_NAMES[:24] + [px, px, px, "kpn", "mean", "cnt", px, px, "sel_score", "sel_pos", b * h, b * h, b,
                                 "n_sel"]
    at = 0
    for item in order:
        at = -(-at // 256) * 256
        if isinstance(item, str):
            assert lay[item][0] == at, item
            at += lay[item][1]
        else:
            at += 4 * item
    assert total == -(-at // 256) * 256


def test_workspace_layout_rejects_bad_arguments():
    cfg = ALIKED(weights=None)._config()
    assert _cabi.load().al_workspace_layout(C.byref(cfg), 0, 64, 64, None, None) == 0
    assert _cabi.load().al_workspace_layout(C.byref(cfg), 1, 64, 0, None, None) == 0
    bad = ALIKED(weights=None)._config()
    bad.M = 33
    assert _cabi.load().al_workspace_layout(C.byref(bad), 1, 64, 64, None, None) == 0
    assert _cabi.load().al_workspace_layout(C.byref(cfg), 1, 64, 64, None, None) > 0
