"""ctypes front of oracle/_build/libsift_emul.so (the host build of the SIFT CUDA path's functors, sift_emul.cpp), with
the reference's conf and outputs.  Test infrastructure only."""
from __future__ import annotations

import ctypes as C
import os

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "_build", "libsift_emul.so")
_lib = None


def available() -> bool:
    return os.path.exists(LIB)


def _load():
    global _lib
    if _lib is None:
        lib = C.CDLL(LIB)
        lib.sift_emul_forward.restype = C.c_int
        lib.sift_emul_forward.argtypes = [C.c_int, C.c_double, C.c_double, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                          C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_long] + [C.c_void_p] * 6
        _lib = lib
    return _lib


def forward(conf: dict, image: torch.Tensor, image_size=None) -> list:
    """Per image, a dict of keypoints, scales, oris, keypoint_scores and descriptors (the first counts[b] rows)."""
    image = image.detach().to(torch.float32).contiguous().cpu()
    B, Ch, H, W = image.shape
    k = int(conf["max_num_keypoints"])
    nms = -1 if conf["nms_radius"] is None else int(conf["nms_radius"])
    sizes = None
    if image_size is not None:
        sizes = torch.as_tensor(image_size).to(torch.int32).contiguous()
    kp = torch.zeros(B, k, 2)
    sc, ori, scr = torch.zeros(B, k), torch.zeros(B, k), torch.zeros(B, k)
    desc = torch.zeros(B, k, 128)
    counts = torch.zeros(B, dtype=torch.int32)
    rc = _load().sift_emul_forward(
        int(conf["num_octaves"]), float(conf["detection_threshold"]), float(conf["edge_threshold"]), nms, k,
        int(bool(conf["rootsift"])), image.data_ptr(), Ch, sizes.data_ptr() if sizes is not None else None, B, H, W, k,
        kp.data_ptr(), sc.data_ptr(), ori.data_ptr(), scr.data_ptr(), desc.data_ptr(), counts.data_ptr())
    assert rc == 0, rc
    out = []
    for b in range(B):
        n = int(counts[b])
        assert n >= 0, "raw keypoint list overflowed"
        out.append({"keypoints": kp[b, :n], "scales": sc[b, :n], "oris": ori[b, :n], "keypoint_scores": scr[b, :n],
                    "descriptors": desc[b, :n]})
    return out
