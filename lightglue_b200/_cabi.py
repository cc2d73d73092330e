"""ctypes binding of include/*.h -- the thin layer between Python and the C ABI."""
from __future__ import annotations

import ctypes as C
import os

from . import build as _build

PREC = {"fp32": 0, "bf16": 1, "bf16x3": 2}
K_ATTENTION, K_LINEAR, K_ASSIGN, K_OTHER = 0, 1, 2, 3
ABI_VERSION = 3

# include/superpoint_b200.h, include/aliked_b200.h and include/sift_b200.h: same library
SP_ABI_VERSION = 2
SP_TC_BUFFERS = 9  # buffers of the tensor-core backbone's workspace plan (sp_tc_layout)
AL_ABI_VERSION = 1
SIFT_ABI_VERSION = 1


class LgConfig(C.Structure):
    _fields_ = [
        ("abi_version", C.c_int32), ("input_dim", C.c_int32), ("pos_dim", C.c_int32), ("n_layers", C.c_int32),
        ("precision", C.c_int32), ("depth_confidence", C.c_float), ("width_confidence", C.c_float),
        ("filter_threshold", C.c_float),
    ]


class SpConfig(C.Structure):
    _fields_ = [
        ("abi_version", C.c_int32), ("nms_radius", C.c_int32), ("max_num_keypoints", C.c_int32),
        ("remove_borders", C.c_int32), ("detection_threshold", C.c_float), ("precision", C.c_int32),
    ]


class AlConfig(C.Structure):
    _fields_ = [
        ("abi_version", C.c_int32), ("c1", C.c_int32), ("c2", C.c_int32), ("c3", C.c_int32), ("c4", C.c_int32),
        ("dim", C.c_int32), ("K", C.c_int32), ("M", C.c_int32), ("nms_radius", C.c_int32),
        ("max_num_keypoints", C.c_int32), ("detection_threshold", C.c_float),
    ]


class SiftConfig(C.Structure):
    _fields_ = [
        ("abi_version", C.c_int32), ("num_octave_layers", C.c_int32), ("nms_radius", C.c_int32),
        ("max_num_keypoints", C.c_int32), ("rootsift", C.c_int32), ("reserved", C.c_int32),
        ("detection_threshold", C.c_double), ("edge_threshold", C.c_double),
    ]


class LgInputs(C.Structure):
    _fields_ = [
        ("B", C.c_int32), ("M", C.c_int32), ("N", C.c_int32),
        ("kpts0", C.c_void_p), ("kpts1", C.c_void_p), ("desc0", C.c_void_p), ("desc1", C.c_void_p),
        ("size0", C.c_void_p), ("size1", C.c_void_p),
        ("scales0", C.c_void_p), ("oris0", C.c_void_p), ("scales1", C.c_void_p), ("oris1", C.c_void_p),
        ("pruning_threshold", C.c_int32),
        ("lens0", C.c_void_p), ("lens1", C.c_void_p),
    ]


class LgOutputs(C.Structure):
    _fields_ = [
        ("matches0", C.c_void_p), ("matches1", C.c_void_p), ("matching_scores0", C.c_void_p),
        ("matching_scores1", C.c_void_p), ("stop", C.c_void_p), ("prune0", C.c_void_p), ("prune1", C.c_void_p),
        ("n_matches", C.c_void_p), ("matches", C.c_void_p), ("match_scores", C.c_void_p),
        ("log_assignment", C.c_void_p),
    ]



# name: (restype, argtypes), one table per header.  The export lists are the tables' keys.
_VP, _I32, _I64, _SZ = C.c_void_p, C.c_int32, C.c_int64, C.c_size_t
_HANDLE_OUT = C.POINTER(C.c_void_p)
LG_PROTOTYPES = {  # include/lightglue_b200.h
    "lg_weight_blob_floats": (_SZ, [_I32, _I32, _I32]),
    "lg_create": (C.c_int, [C.POINTER(LgConfig), _VP, _SZ, _VP, _HANDLE_OUT]),
    "lg_destroy": (C.c_int, [_VP]),
    "lg_workspace_bytes": (_SZ, [_VP, _I32, _I32, _I32]),
    "lg_forward": (C.c_int, [_VP, C.POINTER(LgInputs), C.POINTER(LgOutputs), _VP, _SZ, _VP]),
    "lg_assign": (C.c_int, [_VP, _I32, _I32, _I32, _I32, _VP, _VP, C.POINTER(LgOutputs), _VP, _SZ, _VP]),
    "lg_attention": (C.c_int, [_VP] + [_I32] * 4 + [_VP] * 8 + [_VP, _SZ, _VP]),
    "lg_last_launch_count": (_I64, [_VP]),
    "lg_timing_enable": (C.c_int, [_VP, _I32]),
    "lg_kernel_time_ms": (C.c_int, [_VP, _I32, C.POINTER(C.c_double), C.POINTER(C.c_int64)]),
    "lg_last_error": (C.c_char_p, []),
    "lg_build_info": (C.c_char_p, []),
    "lg_debug_timeout_code": (C.c_uint32, [_VP, C.POINTER(C.c_uint32)]),
    "lg_debug_capture_layers": (C.c_int, [_VP, _VP, _SZ]),
    "lg_padded_length": (_I32, [_I32, _I32]),
}
SP_PROTOTYPES = {  # include/superpoint_b200.h
    "sp_weight_blob_floats": (_SZ, []),
    "sp_create": (C.c_int, [C.POINTER(SpConfig), _VP, _SZ, _VP, _HANDLE_OUT]),
    "sp_destroy": (C.c_int, [_VP]),
    "sp_max_keypoints": (_I64, [_VP, _I32, _I32]),
    "sp_workspace_bytes": (_SZ, [_VP, _I32, _I32, _I32]),
    "sp_forward": (C.c_int, [_VP, _VP, _I32, _I32, _I32, _I64] + [_VP] * 5 + [_SZ, _VP]),
    "sp_backbone": (C.c_int, [_VP, _VP, _I32, _I32, _I32, _VP, _VP, _VP, _SZ, _VP]),
    "sp_tc_layout": (_I64, [_I32, _I32, _I32, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
}
AL_PROTOTYPES = {  # include/aliked_b200.h
    "al_weight_blob_floats": (_SZ, [C.POINTER(AlConfig)]),
    "al_create": (C.c_int, [C.POINTER(AlConfig), _VP, _SZ, _VP, _HANDLE_OUT]),
    "al_destroy": (C.c_int, [_VP]),
    "al_max_keypoints": (_I64, [_VP, _I32, _I32]),
    "al_workspace_bytes": (_SZ, [_VP, _I32, _I32, _I32]),
    "al_forward": (C.c_int, [_VP, _VP, _VP, _I32, _I32, _I32, _I64] + [_VP] * 5 + [_SZ, _VP]),
}
SIFT_PROTOTYPES = {  # include/sift_b200.h
    "sift_create": (C.c_int, [C.POINTER(SiftConfig), _VP, _HANDLE_OUT]),
    "sift_destroy": (C.c_int, [_VP]),
    "sift_max_keypoints": (_I64, [_VP, _I32, _I32]),
    "sift_workspace_bytes": (_SZ, [_VP, _I32, _I32, _I32]),
    "sift_forward": (C.c_int, [_VP, _VP, _I32, _VP, _I32, _I32, _I32, _I64] + [_VP] * 7 + [_SZ, _VP]),
}
EXPORTS, SP_EXPORTS, AL_EXPORTS, SIFT_EXPORTS = (
    tuple(t) for t in (LG_PROTOTYPES, SP_PROTOTYPES, AL_PROTOTYPES, SIFT_PROTOTYPES))

_lib = None


def lib_path() -> str:
    return _build.LIB


def load():
    """Load liblightglue_b200.so (building it if the sources are newer).  Raises if it cannot be had:
    there is no fallback implementation."""
    global _lib
    if _lib is not None:
        return _lib
    path = _build.build() if os.environ.get("LIGHTGLUE_B200_NO_BUILD") != "1" else _build.LIB
    if not os.path.exists(path):
        raise RuntimeError(f"{path} is missing: the CUDA library must be built (python -m lightglue_b200.build)")
    lib = C.CDLL(path)
    for table in (LG_PROTOTYPES, SP_PROTOTYPES, AL_PROTOTYPES, SIFT_PROTOTYPES):
        for name, (restype, argtypes) in table.items():
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = restype, argtypes
    _lib = lib
    return lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        raise RuntimeError(f"{what} failed: {load().lg_last_error().decode()}")
