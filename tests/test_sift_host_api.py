"""Host-side contract of the SIFT extractor (include/sift_b200.h, lightglue_b200/sift.py); no GPU needed."""
import ctypes as C
import os
import re

import pytest
import torch

from lightglue_b200 import _cabi
from lightglue_b200.sift import SIFT

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_symbols_equal_exports_and_are_exported():
    with open(os.path.join(ROOT, "include", "sift_b200.h")) as f:
        hdr = f.read()
    syms = tuple(re.findall(r"LG_API\s+[\w\s\*]+?\b(sift_\w+)\s*\(", hdr))
    assert sorted(syms) == sorted(_cabi.SIFT_EXPORTS)
    lib = _cabi.load()
    for s in _cabi.SIFT_EXPORTS:
        assert hasattr(lib, s), s
        assert getattr(lib, s).argtypes is not None, s


def test_conf_defaults_equal_the_reference():
    assert SIFT.default_conf == {
        "rootsift": True,
        "nms_radius": 0,
        "max_num_keypoints": 4096,
        "backend": "opencv",
        "detection_threshold": 0.0066667,
        "edge_threshold": 10,
        "first_octave": -1,
        "num_octaves": 4,
    }
    assert SIFT.preprocess_conf == {"resize": 1024}
    assert SIFT.required_data_keys == ["image"]


@pytest.mark.parametrize("backend", ["pycolmap", "pycolmap_cpu", "pycolmap_cuda", "vlfeat"])
def test_other_backends_raise_value_error(backend):
    with pytest.raises(ValueError):
        SIFT(backend=backend)


def test_cpu_tensor_raises_runtime_error():
    with pytest.raises(RuntimeError):
        SIFT()({"image": torch.rand(1, 1, 64, 64)})


def test_package_exports_sift():
    import lightglue_b200

    assert lightglue_b200.SIFT is SIFT


# ---------------------------------------------------------------------------------------------- workspace layout
@pytest.mark.parametrize("conf,H,W,h,w", [({}, 8, 8, 8, 8), (dict(num_octaves=1), 17, 23, 17, 23),
                                          (dict(num_octaves=8, max_num_keypoints=7), 203, 317, 150, 301),
                                          ({}, 32, 1024, 32, 1024), ({}, 768, 1024, 768, 1024)])
def test_workspace_layout(conf, H, W, h, w):
    """Buffers 256-aligned, disjoint and inside sift_workspace_bytes; the pyramid of the crop inside `pyr`, octave o of
    size (2h >> o, 2w >> o) with cvRound(log2(2 min(h, w)) - 2) + 1 octaves, its layers disjoint and in carve order."""
    import numpy as np

    from oracle import sift_oracle as so

    m = SIFT(**conf)
    cfg = m._config()
    lay = so.layout(cfg, H, W, h, w)
    L = cfg.num_octave_layers
    lib = _cabi.load()
    handle = C.c_void_p()
    _cabi.check(lib.sift_create(C.byref(cfg), None, C.byref(handle)), "sift_create")
    try:
        assert lay["total"] == lib.sift_workspace_bytes(handle, 2, H, W) > 0
    finally:
        lib.sift_destroy(handle)
    raw = H * W // 4 + 4096
    want = {"counters": 32, "q": 4 * H * W, "tmp": 16 * H * W, "cand": 32 * raw, "kpt": 32 * raw, "order": 4 * raw,
            "flags": 4 * raw, "pix": 4 * raw, "out_src": 4 * cfg.max_num_keypoints}
    spans = []
    for name, o, n in zip(so.BUFFERS, lay["off"], lay["bytes"]):
        assert o % 256 == 0, name
        assert name not in want or n == want[name], (name, n)
        spans.append((o, n))
    spans.sort()
    for (o0, n0), (o1, _) in zip(spans, spans[1:]):
        assert o0 + n0 <= o1
    assert spans[-1][0] + spans[-1][1] + 256 <= lay["total"]
    assert lay["n_oct"] == max(1, int(np.rint(np.log2(2 * min(h, w)) - 2)) + 1)
    pyr = so.BUFFERS.index("pyr")
    at = lay["off"][pyr]
    for o, (hh, ww) in enumerate(lay["dims"]):
        assert (hh, ww) == ((2 * h) >> o, (2 * w) >> o)
        for off in lay["gauss"][o] + lay["dog"][o]:
            assert off == at
            at += 4 * hh * ww
    assert at <= lay["off"][pyr] + lay["bytes"][pyr]
    assert len(lay["gauss"][0]) == L + 3 and len(lay["dog"][0]) == L + 2


def test_workspace_layout_rejects_bad_arguments():
    from oracle import sift_oracle as so

    cfg = SIFT()._config()
    lib = _cabi.load()
    assert lib.sift_workspace_layout(C.byref(cfg), 64, 64, 64, 65, None, None, None, None, None, None) == 0
    assert lib.sift_workspace_layout(C.byref(cfg), 64, 64, 0, 64, None, None, None, None, None, None) == 0
    bad = SIFT()._config()
    bad.num_octave_layers = 9
    assert lib.sift_workspace_layout(C.byref(bad), 64, 64, 64, 64, None, None, None, None, None, None) == 0
    assert so.layout(cfg, 64, 64, 64, 64)["total"] > 0


def test_record_dtypes_match_the_structs():
    import numpy as np

    assert np.dtype(_cabi.SIFT_CAND_DTYPE).itemsize == 32 and np.dtype(_cabi.SIFT_KPT_DTYPE).itemsize == 32
    assert np.dtype(_cabi.SIFT_CAND_DTYPE).fields["octave_packed"][1] == 28
    assert np.dtype(_cabi.SIFT_KPT_DTYPE).fields["angle"][1] == 12
