"""Host-side contract of the SIFT extractor (include/sift_b200.h, lightglue_b200/sift.py); no GPU needed."""
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
