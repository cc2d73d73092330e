"""ctypes binding of include/lightglue_b200.h -- the thin layer between Python and the C ABI."""
from __future__ import annotations

import ctypes as C
import os

from . import build as _build

PREC = {"fp32": 0, "bf16": 1, "bf16x3": 2}
K_ATTENTION, K_LINEAR, K_ASSIGN, K_OTHER = 0, 1, 2, 3
ABI_VERSION = 3

EXPORTS = (
    "lg_weight_blob_floats", "lg_create", "lg_destroy", "lg_workspace_bytes", "lg_forward", "lg_assign", "lg_attention",
    "lg_last_launch_count", "lg_timing_enable", "lg_kernel_time_ms", "lg_last_error", "lg_build_info",
    "lg_debug_timeout_code", "lg_debug_capture_layers", "lg_padded_length",
)
# include/superpoint_b200.h (same library)
SP_ABI_VERSION = 2
SP_EXPORTS = ("sp_weight_blob_floats", "sp_create", "sp_destroy", "sp_max_keypoints", "sp_workspace_bytes", "sp_forward",
              "sp_backbone", "sp_tc_layout")
SP_TC_BUFFERS = 9  # buffers of the tensor-core backbone's workspace plan (sp_tc_layout)
# include/aliked_b200.h (same library)
AL_ABI_VERSION = 1
AL_EXPORTS = ("al_weight_blob_floats", "al_create", "al_destroy", "al_max_keypoints", "al_workspace_bytes", "al_forward")
# include/sift_b200.h (same library)
SIFT_ABI_VERSION = 1
SIFT_EXPORTS = ("sift_create", "sift_destroy", "sift_max_keypoints", "sift_workspace_bytes", "sift_forward")


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
    lib.lg_weight_blob_floats.restype = C.c_size_t
    lib.lg_weight_blob_floats.argtypes = [C.c_int32, C.c_int32, C.c_int32]
    lib.lg_create.restype = C.c_int
    lib.lg_create.argtypes = [C.POINTER(LgConfig), C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_void_p)]
    lib.lg_destroy.restype = C.c_int
    lib.lg_destroy.argtypes = [C.c_void_p]
    lib.lg_workspace_bytes.restype = C.c_size_t
    lib.lg_workspace_bytes.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32]
    lib.lg_forward.restype = C.c_int
    lib.lg_forward.argtypes = [C.c_void_p, C.POINTER(LgInputs), C.POINTER(LgOutputs), C.c_void_p, C.c_size_t, C.c_void_p]
    lib.lg_assign.restype = C.c_int
    lib.lg_assign.argtypes = [
        C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.POINTER(LgOutputs),
        C.c_void_p, C.c_size_t, C.c_void_p,
    ]
    lib.lg_attention.restype = C.c_int
    lib.lg_attention.argtypes = [C.c_void_p] + [C.c_int32] * 4 + [C.c_void_p] * 8 + [C.c_void_p, C.c_size_t, C.c_void_p]
    lib.sp_weight_blob_floats.restype = C.c_size_t
    lib.sp_weight_blob_floats.argtypes = []
    lib.sp_create.restype = C.c_int
    lib.sp_create.argtypes = [C.POINTER(SpConfig), C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_void_p)]
    lib.sp_destroy.restype = C.c_int
    lib.sp_destroy.argtypes = [C.c_void_p]
    lib.sp_max_keypoints.restype = C.c_int64
    lib.sp_max_keypoints.argtypes = [C.c_void_p, C.c_int32, C.c_int32]
    lib.sp_workspace_bytes.restype = C.c_size_t
    lib.sp_workspace_bytes.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32]
    lib.sp_forward.restype = C.c_int
    lib.sp_forward.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int64] + [C.c_void_p] * 5 + [
        C.c_size_t, C.c_void_p]
    lib.sp_backbone.restype = C.c_int
    lib.sp_backbone.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                C.c_size_t, C.c_void_p]
    lib.sp_tc_layout.restype = C.c_int64
    lib.sp_tc_layout.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
    lib.al_weight_blob_floats.restype = C.c_size_t
    lib.al_weight_blob_floats.argtypes = [C.POINTER(AlConfig)]
    lib.al_create.restype = C.c_int
    lib.al_create.argtypes = [C.POINTER(AlConfig), C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_void_p)]
    lib.al_destroy.restype = C.c_int
    lib.al_destroy.argtypes = [C.c_void_p]
    lib.al_max_keypoints.restype = C.c_int64
    lib.al_max_keypoints.argtypes = [C.c_void_p, C.c_int32, C.c_int32]
    lib.al_workspace_bytes.restype = C.c_size_t
    lib.al_workspace_bytes.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32]
    lib.al_forward.restype = C.c_int
    lib.al_forward.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int64] + [
        C.c_void_p] * 5 + [C.c_size_t, C.c_void_p]
    lib.sift_create.restype = C.c_int
    lib.sift_create.argtypes = [C.POINTER(SiftConfig), C.c_void_p, C.POINTER(C.c_void_p)]
    lib.sift_destroy.restype = C.c_int
    lib.sift_destroy.argtypes = [C.c_void_p]
    lib.sift_max_keypoints.restype = C.c_int64
    lib.sift_max_keypoints.argtypes = [C.c_void_p, C.c_int32, C.c_int32]
    lib.sift_workspace_bytes.restype = C.c_size_t
    lib.sift_workspace_bytes.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32]
    lib.sift_forward.restype = C.c_int
    lib.sift_forward.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int64] + [
        C.c_void_p] * 6 + [C.c_void_p, C.c_size_t, C.c_void_p]
    lib.lg_last_launch_count.restype = C.c_int64
    lib.lg_last_launch_count.argtypes = [C.c_void_p]
    lib.lg_timing_enable.restype = C.c_int
    lib.lg_timing_enable.argtypes = [C.c_void_p, C.c_int32]
    lib.lg_kernel_time_ms.restype = C.c_int
    lib.lg_kernel_time_ms.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_double), C.POINTER(C.c_int64)]
    lib.lg_last_error.restype = C.c_char_p
    lib.lg_debug_timeout_code.restype = C.c_uint32
    lib.lg_debug_timeout_code.argtypes = [C.c_void_p, C.POINTER(C.c_uint32)]
    lib.lg_build_info.restype = C.c_char_p
    lib.lg_debug_capture_layers.restype = C.c_int
    lib.lg_debug_capture_layers.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    lib.lg_padded_length.restype = C.c_int32
    lib.lg_padded_length.argtypes = [C.c_int32, C.c_int32]
    _lib = lib
    return lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        raise RuntimeError(f"{what} failed: {load().lg_last_error().decode()}")
