"""The SuperPoint CUDA path, executed on the host.

``lightglue_b200/csrc/sp_pipeline.h`` holds every stage of the extractor as a functor (the body of one GPU thread)
plus the orchestration; ``oracle/sp_emul.cpp`` compiles that header with g++ and runs each functor over its index
space in a loop.  Here that library is checked against the fixtures produced by the reference's own superpoint.py
(tests/golden/sp_*.pt): identical keypoints in the reference's order, scores within 2e-5, descriptors within 2e-6.
The GPU run of the very same code is tests/test_gpu_superpoint.py.  CPU only; test infrastructure."""
import ctypes as C
import os
import subprocess

import pytest
import torch

from lightglue_b200 import synth
from lightglue_b200.superpoint import LAYERS
from oracle import superpoint_synth as sps

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
CASES = ["sp_240x320", "sp_b2_top256", "sp_nms2_thr01", "sp_480x640_top512", "sp_odd_203x317"]


@pytest.fixture(scope="module")
def emul():
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle")])
    lib = C.CDLL(os.path.join(ROOT, "oracle", "_build", "libsp_emul.so"))
    lib.sp_emul_forward.restype = C.c_int
    lib.sp_emul_max_keypoints.restype = C.c_long
    lib.sp_emul_blob_floats.restype = C.c_size_t
    return lib


def weight_blob(w):
    return torch.cat([torch.cat([w[f"{n}.weight"].reshape(-1), w[f"{n}.bias"].reshape(-1)]) for n, *_ in LAYERS]).contiguous()


def run_emulated(lib, w, image, conf):
    b, _, h, ww = image.shape
    k = conf["max_num_keypoints"] or 0
    cap = lib.sp_emul_max_keypoints(conf["nms_radius"], k, h, ww)
    kp, sc = torch.zeros(b, cap, 2), torch.zeros(b, cap)
    de, cnt = torch.zeros(b, cap, 256), torch.zeros(b, dtype=torch.int32)
    blob = weight_blob(w)
    assert blob.numel() == lib.sp_emul_blob_floats()
    image = image.contiguous()
    rc = lib.sp_emul_forward(
        C.c_void_p(blob.data_ptr()), conf["nms_radius"], k, conf["remove_borders"], C.c_float(conf["detection_threshold"]),
        C.c_void_p(image.data_ptr()), b, h, ww, C.c_long(cap), C.c_void_p(kp.data_ptr()), C.c_void_p(sc.data_ptr()),
        C.c_void_p(de.data_ptr()), C.c_void_p(cnt.data_ptr()),
    )
    assert rc == 0
    return kp, sc, de, cnt


@pytest.mark.parametrize("name", CASES)
def test_cuda_functors_on_host_match_reference_fixture(emul, name):
    fix = torch.load(os.path.join(GOLDEN, name + ".pt"), weights_only=False)
    rc, conf, gold = fix["recipe"], fix["conf"], fix["out"]
    w = sps.make_superpoint_state_dict(0)
    image = sps.make_image(rc["h"], rc["w"], rc["b"], rc["seed"])
    assert synth.checksum(image) == fix["image_checksum"]
    kp, sc, de, cnt = run_emulated(emul, w, image, conf)
    for b in range(rc["b"]):
        n = int(cnt[b])
        assert n == gold["keypoints"][b].shape[0]
        assert torch.equal(kp[b, :n], gold["keypoints"][b]), "keypoint set / order differs from the reference"
        assert float((sc[b, :n] - gold["keypoint_scores"][b]).abs().max()) <= 2e-5
        st = gold["desc_stride"][b]
        assert float((de[b, :n][::st] - gold["descriptors"][b]).abs().max()) <= 2e-6
        assert float(kp[b, n:].abs().sum()) == 0.0 and float(de[b, n:].abs().sum()) == 0.0  # padding slots are zero


def test_superpoint_header_symbols_are_exported_and_host_mirror_contract():
    import re

    from lightglue_b200 import _cabi
    from lightglue_b200.superpoint import SuperPoint

    lib = _cabi.load()
    header = open(os.path.join(ROOT, "include", "superpoint_b200.h")).read()
    declared = re.findall(r"LG_API\s+[\w\s\*]+?\b(sp_\w+)\s*\(", header)
    assert sorted(declared) == sorted(_cabi.SP_EXPORTS)
    for name in declared:
        assert hasattr(lib, name), name
        assert getattr(lib, name).argtypes is not None, name
    m = SuperPoint(weights=None, max_num_keypoints=512)
    assert lib.sp_weight_blob_floats() == m._blob().numel() == sum(p.numel() for p in m.parameters())
    ref_keys = {f"{n}.{s}" for n, *_ in LAYERS for s in ("weight", "bias")}  # superpoint.py:137-153
    assert set(m.state_dict().keys()) == ref_keys
    assert m.conf.nms_radius == 4 and m.conf.detection_threshold == 0.0005 and m.conf.remove_borders == 4
    assert SuperPoint.preprocess_conf == {"resize": 1024} and SuperPoint.required_data_keys == ["image"]
    with pytest.raises(ValueError):
        SuperPoint(weights=None, max_num_keypoints=0)
    with pytest.raises(FileNotFoundError):
        SuperPoint()  # no network, no cached superpoint_v1.pth
    with pytest.raises(RuntimeError):
        m({"image": torch.zeros(1, 1, 64, 64)})  # CPU tensor: no CPU path
    m.load_state_dict(sps.make_superpoint_state_dict(0))


@pytest.mark.parametrize("h,w,conf", [
    (8, 8, dict(remove_borders=0)),                       # one detector cell
    (9, 15, dict(remove_borders=1, nms_radius=1)),        # neither extent a multiple of 8, one cell row
    (17, 33, dict(remove_borders=2)),
    (67, 45, {}),                                         # portrait, odd at every pooling level
    (24, 131, dict(max_num_keypoints=20)),
])
def test_cuda_functors_on_host_any_image_size_vs_oracle(emul, h, w, conf):
    """Image extents that are not multiples of 8 (floor poolings, superpoint.py:173-179; score map over the 8-aligned
    top-left area, 188-190): the CUDA functors against the Python oracle, which is pinned to the reference on the
    fixtures (among them the odd-sized sp_odd_203x317)."""
    from oracle import superpoint_oracle as spo

    torch.set_grad_enabled(False)
    wts = sps.make_superpoint_state_dict(0)
    image = sps.make_image(h, w, 1, 100 + h)
    full = dict(nms_radius=4, max_num_keypoints=None, detection_threshold=0.0005, remove_borders=4)
    full.update(conf)
    ref = spo.forward(wts, image, **full)
    kp, sc, de, cnt = run_emulated(emul, wts, image, full)
    n = int(cnt[0])
    assert n == ref["keypoints"][0].shape[0] and n > 0
    assert torch.equal(kp[0, :n], ref["keypoints"][0])
    assert float((sc[0, :n] - ref["keypoint_scores"][0]).abs().max()) <= 2e-5
    assert float((de[0, :n] - ref["descriptors"][0]).abs().max()) <= 2e-6
