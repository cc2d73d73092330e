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
        lib.sift_emul_forward_ws.restype = C.c_int
        lib.sift_emul_forward_ws.argtypes = lib.sift_emul_forward.argtypes + [C.c_void_p, C.c_size_t]
        lib.sift_emul_workspace_bytes.restype = C.c_size_t
        lib.sift_emul_workspace_bytes.argtypes = [C.c_int] * 4
        lib.sift_emul_filter.restype = C.c_int
        lib.sift_emul_filter.argtypes = [C.c_void_p] + [C.c_int] * 5 + [C.c_void_p] * 5
        _lib = lib
    return _lib


def forward(conf: dict, image: torch.Tensor, image_size=None) -> list:
    """Per image, a dict of keypoints, scales, oris, keypoint_scores and descriptors (the first counts[b] rows)."""
    out = []
    for b, o in enumerate(forward_ws(conf, image, image_size)[0]):
        n = int(o["count"])
        assert n >= 0, "raw keypoint list overflowed"
        out.append({k: o[k][:n] for k in ("keypoints", "scales", "oris", "keypoint_scores", "descriptors")})
    return out


def forward_ws(conf: dict, image: torch.Tensor, image_size=None):
    """-> (per image a dict of all `cap` rows of keypoints, scales, oris, keypoint_scores, descriptors and its count,
    the workspace as a uint8 tensor from the carve's 256-byte-aligned base).  The workspace holds the last image's
    intermediates where sift_workspace_layout says."""
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
    L = int(conf["num_octaves"])
    nbytes = _load().sift_emul_workspace_bytes(L, k, H, W)
    assert nbytes > 0
    ws = torch.zeros(nbytes + 256, dtype=torch.uint8)
    rc = _load().sift_emul_forward_ws(
        L, float(conf["detection_threshold"]), float(conf["edge_threshold"]), nms, k,
        int(bool(conf["rootsift"])), image.data_ptr(), Ch, sizes.data_ptr() if sizes is not None else None, B, H, W, k,
        kp.data_ptr(), sc.data_ptr(), ori.data_ptr(), scr.data_ptr(), desc.data_ptr(), counts.data_ptr(), ws.data_ptr(),
        nbytes + 256)
    assert rc == 0, rc
    out = [{"keypoints": kp[b], "scales": sc[b], "oris": ori[b], "keypoint_scores": scr[b], "descriptors": desc[b],
            "count": int(counts[b])} for b in range(B)]
    return out, ws[(-ws.data_ptr()) % 256:]


def filter_records(kpt, w: int, nms_radius, max_kpts: int) -> dict:
    """The ordering and filtering functors on raw keypoint records kpt (numpy, _cabi.SIFT_KPT_DTYPE) of an image of
    width w -> {"order", "flags", "pix", "out_src", "counters"} as the workspace holds them."""
    import numpy as np

    from lightglue_b200 import _cabi

    kpt = np.ascontiguousarray(kpt, dtype=np.dtype(_cabi.SIFT_KPT_DTYPE))
    n = len(kpt)
    cap = max(n, 1)
    out = {k: np.zeros(cap, np.int32) for k in ("order", "flags", "pix")}
    out["out_src"], out["counters"] = np.zeros(max_kpts, np.int32), np.zeros(8, np.int32)
    rc = _load().sift_emul_filter(kpt.ctypes.data, n, cap, w, -1 if nms_radius is None else int(nms_radius), max_kpts,
                                  *(out[k].ctypes.data for k in ("order", "flags", "pix", "out_src", "counters")))
    assert rc == 0, rc
    return out
