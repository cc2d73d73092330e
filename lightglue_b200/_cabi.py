"""ctypes binding of include/*.h -- the thin layer between Python and the C ABI."""
from __future__ import annotations

import ctypes as C
import os

from . import build as _build

PREC = {"fp32": 0, "bf16": 1, "bf16x3": 2}
K_ATTENTION, K_LINEAR, K_ASSIGN, K_OTHER = 0, 1, 2, 3
ABI_VERSION = 3

# include/superpoint_b200.h, include/aliked_b200.h, include/sift_b200.h, include/disk_b200.h,
# include/doghardnet_b200.h, include/geometry_b200.h and include/nn_b200.h: same library
SP_ABI_VERSION = 2
SP_TC_BUFFERS = 9  # buffers of the tensor-core backbone's workspace plan (sp_tc_layout)
SP_LAYOUT_BUFFERS = 13  # buffers of sp_workspace_layout
AL_ABI_VERSION = 1
AL_LAYOUT_BUFFERS = 30  # buffers of al_workspace_layout
SIFT_ABI_VERSION = 1
SIFT_LAYOUT_BUFFERS, SIFT_LAYOUT_MAX_OCTAVES = 10, 16  # sift_workspace_layout
DISK_ABI_VERSION = 1
DISK_LAYOUT_BUFFERS = 13  # buffers of disk_workspace_layout
DHN_ABI_VERSION = 1
DHN_LAYOUT_BUFFERS = 16  # buffers of dhn_workspace_layout
GEO_ABI_VERSION = 1  # include/geometry_b200.h
GEO_HOMOGRAPHY, GEO_FUNDAMENTAL, GEO_ESSENTIAL = 0, 1, 2
GEO_LO_QSCALE, GEO_LO_MAX_MATCHES = 65536, (1 << 20) - 1
GEO_AFFINE, GEO_AFFINE_PARTIAL, GEO_AFFINE_MAX_REFINE = 3, 4, 100
GEO_CAMERA_FLOAT32, GEO_CAMERA_FLOAT64, GEO_UNDISTORT_MAX_ITERS = 0, 1, 1000
GEO_RIGID_3D, GEO_SIMILARITY_3D = 5, 6
NN_ABI_VERSION = 1  # include/nn_b200.h
NN_MIN_DIM, NN_MAX_DIM, NN_GROUP_ROWS = 64, 512, 32768
NN_GUIDE_H, NN_GUIDE_F = 0, 1


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


# numpy dtypes of the SIFT list records in the workspace (SiftCand, SiftKpt in csrc/sift_pipeline.h, 32 bytes each)
SIFT_CAND_DTYPE = [("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("response", "<f4"), ("r", "<i4"), ("c", "<i4"),
                   ("layer", "<i4"), ("octave_packed", "<i4")]
SIFT_KPT_DTYPE = [("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("angle", "<f4"), ("response", "<f4"),
                  ("octave_packed", "<i4"), ("o", "<i4"), ("layer", "<i4")]


class DiskConfig(C.Structure):
    _fields_ = [
        ("abi_version", C.c_int32), ("max_num_keypoints", C.c_int32), ("nms_window_size", C.c_int32),
        ("pad_if_not_divisible", C.c_int32), ("detection_threshold", C.c_float),
    ]


class DhnConfig(C.Structure):
    _fields_ = [
        ("abi_version", C.c_int32), ("num_octave_layers", C.c_int32), ("nms_radius", C.c_int32),
        ("max_num_keypoints", C.c_int32), ("detection_threshold", C.c_double), ("edge_threshold", C.c_double),
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


class GeoConfig(C.Structure):
    _fields_ = [
        ("abi_version", C.c_int32), ("model", C.c_int32), ("max_iters", C.c_int32), ("seed", C.c_uint32),
        ("threshold", C.c_double), ("confidence", C.c_double),
    ]


class GeoInputs(C.Structure):
    _fields_ = [
        ("B", C.c_int32), ("M", C.c_int32), ("N", C.c_int32),
        ("kpts0", C.c_void_p), ("kpts1", C.c_void_p), ("matches0", C.c_void_p),
    ]


class GeoOutputs(C.Structure):
    _fields_ = [
        ("model", C.c_void_p), ("inliers", C.c_void_p), ("num_inliers", C.c_void_p), ("success", C.c_void_p),
        ("best_hypothesis", C.c_void_p), ("num_hypotheses", C.c_void_p),
    ]


class GeoPoseConfig(C.Structure):
    _fields_ = [
        ("abi_version", C.c_int32), ("max_iters", C.c_int32), ("seed", C.c_uint32), ("reserved", C.c_int32),
        ("threshold", C.c_double), ("confidence", C.c_double), ("distance_threshold", C.c_double),
    ]


class GeoPoseInputs(C.Structure):
    _fields_ = [
        ("B", C.c_int32), ("M", C.c_int32), ("N", C.c_int32),
        ("kpts0", C.c_void_p), ("kpts1", C.c_void_p), ("matches0", C.c_void_p), ("K0", C.c_void_p), ("K1", C.c_void_p),
    ]


class GeoPoseOutputs(C.Structure):
    _fields_ = [
        ("E", C.c_void_p), ("R", C.c_void_p), ("t", C.c_void_p), ("inliers", C.c_void_p), ("num_inliers", C.c_void_p),
        ("pose_inliers", C.c_void_p), ("num_pose_inliers", C.c_void_p), ("success", C.c_void_p),
        ("best_hypothesis", C.c_void_p), ("best_solution", C.c_void_p), ("num_hypotheses", C.c_void_p),
    ]


class GeoLoPoseConfig(C.Structure):
    _fields_ = GeoPoseConfig._fields_


class GeoLoPoseOutputs(C.Structure):
    _fields_ = [("pose", GeoPoseOutputs), ("num_local_optimizations", C.c_void_p), ("cost", C.c_void_p)]


class GeoLoOutputs(C.Structure):
    _fields_ = [("geo", GeoOutputs), ("num_local_optimizations", C.c_void_p), ("cost", C.c_void_p)]


class GeoPnpConfig(C.Structure):
    _fields_ = [
        ("abi_version", C.c_int32), ("max_iters", C.c_int32), ("seed", C.c_uint32), ("reserved", C.c_int32),
        ("threshold", C.c_double), ("confidence", C.c_double),
    ]


class GeoPnpInputs(C.Structure):
    _fields_ = [
        ("B", C.c_int32), ("M", C.c_int32), ("N", C.c_int32),
        ("kpts0", C.c_void_p), ("points3d1", C.c_void_p), ("matches0", C.c_void_p), ("K0", C.c_void_p),
    ]


class GeoPnpOutputs(C.Structure):
    _fields_ = [
        ("R", C.c_void_p), ("t", C.c_void_p), ("inliers", C.c_void_p), ("num_inliers", C.c_void_p),
        ("success", C.c_void_p), ("best_hypothesis", C.c_void_p), ("best_solution", C.c_void_p),
        ("num_hypotheses", C.c_void_p),
    ]


class GeoLoPnpOutputs(C.Structure):
    _fields_ = [("pnp", GeoPnpOutputs), ("num_local_optimizations", C.c_void_p), ("cost", C.c_void_p)]


class GeoAffineConfig(C.Structure):
    _fields_ = [
        ("abi_version", C.c_int32), ("model", C.c_int32), ("max_iters", C.c_int32), ("seed", C.c_uint32),
        ("refine_iters", C.c_int32), ("reserved", C.c_int32), ("threshold", C.c_double), ("confidence", C.c_double),
    ]


class GeoCameraConfig(C.Structure):
    _fields_ = [
        ("abi_version", C.c_int32), ("num_dist", C.c_int32), ("max_iters", C.c_int32), ("dtype", C.c_int32),
        ("eps", C.c_double),
    ]


class GeoCameraInputs(C.Structure):
    _fields_ = [("B", C.c_int32), ("N", C.c_int32), ("pts", C.c_void_p), ("K", C.c_void_p), ("dist", C.c_void_p)]


class GeoCameraOutputs(C.Structure):
    _fields_ = [("pts", C.c_void_p)]


class GeoPnpDistInputs(C.Structure):
    _fields_ = [("pnp", GeoPnpInputs), ("num_dist", C.c_int32), ("dist0", C.c_void_p)]


class GeoRigidOutputs(C.Structure):
    _fields_ = [
        ("R", C.c_void_p), ("t", C.c_void_p), ("scale", C.c_void_p), ("inliers", C.c_void_p),
        ("num_inliers", C.c_void_p), ("success", C.c_void_p), ("best_hypothesis", C.c_void_p),
        ("num_hypotheses", C.c_void_p),
    ]


class NnConfig(C.Structure):
    _fields_ = [
        ("abi_version", C.c_int32), ("dim", C.c_int32), ("mutual_check", C.c_int32), ("ratio_thresh", C.c_float),
        ("distance_thresh", C.c_float),
    ]


class NnInputs(C.Structure):
    _fields_ = [
        ("B", C.c_int32), ("M", C.c_int32), ("N", C.c_int32),
        ("desc0", C.c_void_p), ("desc1", C.c_void_p), ("lens0", C.c_void_p), ("lens1", C.c_void_p),
    ]


class NnOutputs(C.Structure):
    _fields_ = [
        ("matches0", C.c_void_p), ("matches1", C.c_void_p), ("matching_scores0", C.c_void_p),
        ("matching_scores1", C.c_void_p), ("n_matches", C.c_void_p), ("matches", C.c_void_p),
        ("match_scores", C.c_void_p),
    ]


class NnGuide(C.Structure):
    _fields_ = [
        ("kind", C.c_int32), ("model", C.c_void_p), ("valid", C.c_void_p), ("kpts0", C.c_void_p), ("kpts1", C.c_void_p),
        ("max_error", C.c_double),
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
    "sp_post": (C.c_int, [_VP, _VP, _VP, _I32, _I32, _I32, _I64] + [_VP] * 5 + [_SZ, _VP]),
    "sp_workspace_layout": (_I64, [C.POINTER(SpConfig), _I32, _I32, _I32, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "sp_tc_layout": (_I64, [_I32, _I32, _I32, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
}
AL_PROTOTYPES = {  # include/aliked_b200.h
    "al_weight_blob_floats": (_SZ, [C.POINTER(AlConfig)]),
    "al_create": (C.c_int, [C.POINTER(AlConfig), _VP, _SZ, _VP, _HANDLE_OUT]),
    "al_destroy": (C.c_int, [_VP]),
    "al_max_keypoints": (_I64, [_VP, _I32, _I32]),
    "al_workspace_bytes": (_SZ, [_VP, _I32, _I32, _I32]),
    "al_forward": (C.c_int, [_VP, _VP, _VP, _I32, _I32, _I32, _I64] + [_VP] * 5 + [_SZ, _VP]),
    "al_workspace_layout": (_I64, [C.POINTER(AlConfig), _I32, _I32, _I32, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
}
SIFT_PROTOTYPES = {  # include/sift_b200.h
    "sift_create": (C.c_int, [C.POINTER(SiftConfig), _VP, _HANDLE_OUT]),
    "sift_destroy": (C.c_int, [_VP]),
    "sift_max_keypoints": (_I64, [_VP, _I32, _I32]),
    "sift_workspace_bytes": (_SZ, [_VP, _I32, _I32, _I32]),
    "sift_forward": (C.c_int, [_VP, _VP, _I32, _VP, _I32, _I32, _I32, _I64] + [_VP] * 7 + [_SZ, _VP]),
    "sift_workspace_layout": (_I64, [C.POINTER(SiftConfig), _I32, _I32, _I32, _I32, C.POINTER(C.c_int64),
                                     C.POINTER(C.c_int64), C.POINTER(C.c_int32), C.POINTER(C.c_int32),
                                     C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
}
DISK_PROTOTYPES = {  # include/disk_b200.h
    "disk_weight_blob_floats": (_SZ, []),
    "disk_create": (C.c_int, [C.POINTER(DiskConfig), _VP, _SZ, _VP, _HANDLE_OUT]),
    "disk_destroy": (C.c_int, [_VP]),
    "disk_max_keypoints": (_I64, [_VP, _I32, _I32]),
    "disk_workspace_bytes": (_SZ, [_VP, _I32, _I32, _I32]),
    "disk_forward": (C.c_int, [_VP, _VP, _I32, _I32, _I32, _I32, _I64] + [_VP] * 5 + [_SZ, _VP]),
    "disk_heads": (C.c_int, [_VP, _VP, _I32, _I32, _I32, _I32, _VP, _I32, _VP, _VP, _VP, _SZ, _VP]),
    "disk_workspace_layout": (_I64, [_VP, _I32, _I32, _I32, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "disk_detect": (C.c_int, [_VP, _VP, _I32, _I32, _I32, _I64] + [_VP] * 4 + [_SZ, _VP]),
}
DHN_PROTOTYPES = {  # include/doghardnet_b200.h
    "dhn_weight_blob_floats": (_SZ, []),
    "dhn_create": (C.c_int, [C.POINTER(DhnConfig), _VP, _SZ, _VP, _HANDLE_OUT]),
    "dhn_destroy": (C.c_int, [_VP]),
    "dhn_max_keypoints": (_I64, [_VP, _I32, _I32]),
    "dhn_workspace_bytes": (_SZ, [_VP, _I32, _I32, _I32]),
    "dhn_forward": (C.c_int, [_VP, _VP, _I32, _VP, _I32, _I32, _I32, _I64] + [_VP] * 7 + [_SZ, _VP]),
    "dhn_describe": (C.c_int, [_VP, _VP, _I32, _VP, _I32, _I32, _I32, _I64] + [_VP] * 6 + [_SZ, _VP]),
    "dhn_workspace_layout": (_I64, [_VP, _I32, _I32, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
}
GEO_PROTOTYPES = {  # include/geometry_b200.h
    "geo_workspace_bytes": (_SZ, [_I32, _I32, _I32]),
    "geo_estimate": (C.c_int, [C.POINTER(GeoConfig), C.POINTER(GeoInputs), C.POINTER(GeoOutputs), _VP, _SZ, _VP]),
    "geo_pose_workspace_bytes": (_SZ, [_I32, _I32, _I32]),
    "geo_relative_pose": (C.c_int, [C.POINTER(GeoPoseConfig), C.POINTER(GeoPoseInputs), C.POINTER(GeoPoseOutputs), _VP,
                                    _SZ, _VP]),
    "geo_lo_pose_workspace_bytes": (_SZ, [_I32, _I32, _I32]),
    "geo_relative_pose_lo": (C.c_int, [C.POINTER(GeoLoPoseConfig), C.POINTER(GeoPoseInputs),
                                       C.POINTER(GeoLoPoseOutputs), _VP, _SZ, _VP]),
    "geo_lo_homography_workspace_bytes": (_SZ, [_I32, _I32, _I32]),
    "geo_homography_lo": (C.c_int, [C.POINTER(GeoConfig), C.POINTER(GeoInputs), C.POINTER(GeoLoOutputs), _VP, _SZ,
                                    _VP]),
    "geo_lo_fundamental_workspace_bytes": (_SZ, [_I32, _I32, _I32]),
    "geo_fundamental_lo": (C.c_int, [C.POINTER(GeoConfig), C.POINTER(GeoInputs), C.POINTER(GeoLoOutputs), _VP, _SZ,
                                     _VP]),
    "geo_pnp_workspace_bytes": (_SZ, [_I32, _I32, _I32]),
    "geo_absolute_pose": (C.c_int, [C.POINTER(GeoPnpConfig), C.POINTER(GeoPnpInputs), C.POINTER(GeoPnpOutputs), _VP,
                                    _SZ, _VP]),
    "geo_lo_pnp_workspace_bytes": (_SZ, [_I32, _I32, _I32]),
    "geo_absolute_pose_lo": (C.c_int, [C.POINTER(GeoPnpConfig), C.POINTER(GeoPnpInputs), C.POINTER(GeoLoPnpOutputs),
                                       _VP, _SZ, _VP]),
    "geo_undistort_points": (C.c_int, [C.POINTER(GeoCameraConfig), C.POINTER(GeoCameraInputs),
                                       C.POINTER(GeoCameraOutputs), _VP]),
    "geo_distort_points": (C.c_int, [C.POINTER(GeoCameraConfig), C.POINTER(GeoCameraInputs),
                                     C.POINTER(GeoCameraOutputs), _VP]),
    "geo_absolute_pose_dist": (C.c_int, [C.POINTER(GeoPnpConfig), C.POINTER(GeoPnpDistInputs),
                                         C.POINTER(GeoPnpOutputs), _VP, _SZ, _VP]),
    "geo_absolute_pose_lo_dist": (C.c_int, [C.POINTER(GeoPnpConfig), C.POINTER(GeoPnpDistInputs),
                                            C.POINTER(GeoLoPnpOutputs), _VP, _SZ, _VP]),
    "geo_rigid_workspace_bytes": (_SZ, [_I32, _I32, _I32]),
    "geo_estimate_rigid": (C.c_int, [C.POINTER(GeoConfig), C.POINTER(GeoInputs), C.POINTER(GeoRigidOutputs), _VP,
                                     _SZ, _VP]),
    "geo_affine_workspace_bytes": (_SZ, [_I32, _I32, _I32]),
    "geo_estimate_affine": (C.c_int, [C.POINTER(GeoAffineConfig), C.POINTER(GeoInputs), C.POINTER(GeoOutputs), _VP,
                                      _SZ, _VP]),
}
NN_PROTOTYPES = {  # include/nn_b200.h
    "nn_create": (C.c_int, [_VP, _HANDLE_OUT]),
    "nn_destroy": (C.c_int, [_VP]),
    "nn_workspace_bytes": (_SZ, [_I32, _I32, _I32, _I32]),
    "nn_match": (C.c_int, [_VP, C.POINTER(NnConfig), C.POINTER(NnInputs), C.POINTER(NnOutputs), _VP, _SZ, _VP]),
    "nn_guided_workspace_bytes": (_SZ, [_I32, _I32, _I32, _I32]),
    "nn_match_guided": (C.c_int, [_VP, C.POINTER(NnConfig), C.POINTER(NnInputs), C.POINTER(NnGuide),
                                  C.POINTER(NnOutputs), _VP, _SZ, _VP]),
}
_TABLES = (LG_PROTOTYPES, SP_PROTOTYPES, AL_PROTOTYPES, SIFT_PROTOTYPES, DISK_PROTOTYPES, DHN_PROTOTYPES, GEO_PROTOTYPES,
           NN_PROTOTYPES)
EXPORTS, SP_EXPORTS, AL_EXPORTS, SIFT_EXPORTS, DISK_EXPORTS, DHN_EXPORTS, GEO_EXPORTS, NN_EXPORTS = (
    tuple(t) for t in _TABLES)

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
    for table in _TABLES:
        for name, (restype, argtypes) in table.items():
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = restype, argtypes
    _lib = lib
    return lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        raise RuntimeError(f"{what} failed: {load().lg_last_error().decode()}")
