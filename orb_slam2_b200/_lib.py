"""ctypes binding of libborb.so (the C ABI in include/borb.h).

There is deliberately NO fallback: if the CUDA library is missing or no GPU is visible, the product
raises.  (CPU restatements live only under oracle/ and are test infrastructure.)
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libborb.so")

KP_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("angle", "<f4"), ("response", "<f4"),
                     ("octave", "<i4"), ("class_id", "<i4")])   # == cv::KeyPoint, 28 bytes

BORB_OK = 0
STATUS_NAMES = {0: "BORB_OK", 1: "BORB_ERR_INVALID_ARG", 2: "BORB_ERR_NO_DEVICE", 3: "BORB_ERR_CUDA",
                4: "BORB_ERR_UNSUPPORTED", 5: "BORB_ERR_CAPACITY", 6: "BORB_ERR_STATE"}


class BorbError(RuntimeError):
    def __init__(self, status: int, where: str, detail: str):
        self.status = status
        super().__init__(f"{where}: {STATUS_NAMES.get(status, status)}: {detail}")


class ExtractorCfg(C.Structure):
    _fields_ = [("n_features", C.c_int32), ("scale_factor", C.c_float), ("n_levels", C.c_int32),
                ("ini_th_fast", C.c_int32), ("min_th_fast", C.c_int32)]


u8p = C.POINTER(C.c_uint8)
f32p = C.POINTER(C.c_float)
i32p = C.POINTER(C.c_int32)
vp = C.c_void_p

# name -> (restype, argtypes); mirrors include/borb.h one to one
_SIGNATURES = {
    "borb_last_error": (C.c_char_p, []),
    "borb_status_str": (C.c_char_p, [C.c_int]),
    "borb_version": (C.c_int, []),
    "borb_device_count": (C.c_int, [i32p]),
    "borb_host_alloc": (C.c_int, [C.POINTER(vp), C.c_size_t]),
    "borb_host_free": (C.c_int, [vp]),
    "borb_extractor_create": (C.c_int, [C.POINTER(ExtractorCfg), C.c_int, C.POINTER(vp)]),
    "borb_extractor_destroy": (C.c_int, [vp]),
    "borb_extractor_tables": (C.c_int, [vp, f32p, f32p, f32p, f32p, i32p]),
    "borb_extractor_capacity": (C.c_int, [vp, C.c_int, C.c_int, i32p]),
    "borb_extractor_reserve": (C.c_int, [vp, C.c_int, C.c_int, C.c_int]),
    "borb_extract": (C.c_int, [vp, vp, C.c_int, C.c_int, C.c_int, vp, vp, C.c_int, i32p]),
    "borb_extract_batch": (C.c_int, [vp, C.POINTER(vp), C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, C.c_int, vp]),
    "borb_extract_batch_enqueue": (C.c_int, [vp, C.POINTER(vp), C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, C.c_int, vp]),
    "borb_sync": (C.c_int, [vp]),
    "borb_extract_batch_device": (C.c_int, [vp, vp, C.c_int, C.c_int, C.c_int, C.c_size_t, C.c_size_t, vp, vp, C.c_int, vp]),
    "borb_extractor_pyramid": (C.c_int, [vp, C.c_int, C.c_int, vp, i32p, i32p]),
    "borb_stereo_match": (C.c_int, [vp, C.c_int, vp, vp, C.c_float, C.c_float, vp, vp, C.c_int]),
    "borb_stereo_match2": (C.c_int, [vp, vp, C.c_float, C.c_float, vp, vp, C.c_int]),
    "borb_stereo_frames": (C.c_int, [vp, C.POINTER(vp), C.POINTER(vp), C.c_int, C.c_int, C.c_int, C.c_int, C.c_float,
                                     C.c_float, vp, vp, vp, vp, vp, vp, vp, vp, C.c_int]),
    "borb_stereo_frames_enqueue": (C.c_int, [vp, C.POINTER(vp), C.POINTER(vp), C.c_int, C.c_int, C.c_int, C.c_int,
                                             C.c_float, C.c_float, vp, vp, vp, vp, vp, vp, vp, vp, C.c_int]),
    "borb_stereo_frames_device": (C.c_int, [vp, vp, C.c_int, C.c_int, C.c_int, C.c_size_t, C.c_size_t, C.c_float,
                                            C.c_float, vp, vp, vp, vp, C.c_int]),
    "borb_stereo_frames_device_enqueue": (C.c_int, [vp, vp, C.c_int, C.c_int, C.c_int, C.c_size_t, C.c_size_t, C.c_float,
                                                    C.c_float, vp, vp, vp, vp, C.c_int]),
    "borb_stereo_frames_results": (C.c_int, [vp, C.c_int, vp, vp, vp, vp, vp, vp, vp, vp, C.c_int]),
    "borb_stage_times_total": (C.c_int, [vp, C.POINTER(C.c_double), C.POINTER(C.c_uint64)]),
    "borb_extractor_stream": (C.c_int, [vp, C.POINTER(vp)]),
    "borb_matcher_create": (C.c_int, [C.c_int, C.POINTER(vp)]),
    "borb_extractor_set_input_format": (C.c_int, [vp, C.c_int, C.c_int]),
    "borb_extractor_set_rectify_maps": (C.c_int, [vp, C.c_int, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int]),
    "borb_matcher_destroy": (C.c_int, [vp]),
    "borb_frame_create": (C.c_int, [vp, vp, C.POINTER(vp)]),
    "borb_frame_destroy": (C.c_int, [vp]),
    "borb_frames_from_extractor": (C.c_int, [vp, vp, vp, C.c_int, vp, vp, C.c_int, vp, C.c_int, C.c_float, C.c_int, vp, vp, vp, C.c_int, vp, vp]),
    "borb_frame_from_extractors": (C.c_int, [vp, vp, vp, vp, C.c_int, C.c_float, vp, C.c_int, C.c_float, C.c_int, vp, vp]),
    "borb_frame_info": (C.c_int, [vp, i32p, i32p, i32p]),
    "borb_debug_frame_read": (C.c_int, [vp, vp, vp, vp, vp, vp, vp]),
    "borb_search_by_projection": (C.c_int, [vp, vp, vp, C.c_float, C.c_float, vp, i32p]),
    "borb_search_by_projection_batch": (C.c_int, [vp, vp, vp, C.c_int, C.c_float, C.c_float, vp, vp]),
    "borb_search_by_projection_last": (C.c_int, [vp, vp, vp, vp, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float,
                                                 C.c_int, C.c_int, C.c_int, vp, i32p]),
    "borb_search_by_projection_kf": (C.c_int, [vp, vp, vp, vp, vp, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float,
                                               C.c_int, C.c_int, vp, i32p]),
    "borb_search_by_projection_sim3": (C.c_int, [vp, vp, vp, vp, vp, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int,
                                                 vp, i32p]),
    "borb_search_for_initialization": (C.c_int, [vp, vp, vp, vp, C.c_int, C.c_float, C.c_int, vp, i32p]),
    "borb_search_for_initialization_batch": (C.c_int, [vp, vp, C.c_int, C.c_float, C.c_int, vp]),
    "borb_distinctive_descriptors": (C.c_int, [vp, vp, vp, C.c_int, vp]),
    "borb_distinctive_descriptors_frames": (C.c_int, [vp, vp, C.c_int, vp, vp, vp, C.c_int, vp, vp]),
    "borb_kfdb_create": (C.c_int, [C.c_int, C.POINTER(vp)]),
    "borb_kfdb_destroy": (C.c_int, [vp]),
    "borb_kfdb_clear": (C.c_int, [vp]),
    "borb_kfdb_add": (C.c_int, [vp, vp, vp, vp, C.c_int, i32p]),
    "borb_kfdb_erase": (C.c_int, [vp, C.c_int32]),
    "borb_kfdb_set_has_mp": (C.c_int, [vp, C.c_int32, vp]),
    "borb_kfdb_set_has_mp_batch": (C.c_int, [vp, C.c_int, vp, vp]),
    "borb_kfdb_size": (C.c_int, [vp, i32p, C.POINTER(C.c_uint64)]),
    "borb_kfdb_query": (C.c_int, [vp, vp, vp, vp, C.c_int, vp, vp, vp, C.c_int, i32p]),
    "borb_search_by_bow_db": (C.c_int, [vp, vp, vp, C.c_int, vp, C.c_float, C.c_int, vp, vp]),
    "borb_search_by_bow_db_pairs": (C.c_int, [vp, vp, vp, C.c_int, vp, C.c_float, C.c_int, vp, vp, vp, C.c_int, i32p]),
    "borb_kfdb_query_batch": (C.c_int, [vp, vp, C.c_int]),
    "borb_kfdb_add_frames": (C.c_int, [vp, vp, C.c_int]),
    "borb_bow_score_batch": (C.c_int, [vp, vp, C.c_int]),
    "borb_debug_kfdb_read": (C.c_int, [vp, C.c_int32, vp, C.POINTER(C.c_uint64), vp, vp, vp, vp, vp, vp, vp, vp]),
    "borb_search_by_bow_db_batch": (C.c_int, [vp, vp, C.c_int, C.c_float, C.c_int]),
    "borb_search_by_bow_kf_db_batch": (C.c_int, [vp, vp, C.c_int, C.c_float, C.c_int]),
    "borb_search_by_bow_kf_db_pairs": (C.c_int, [vp, vp, C.c_int32, vp, C.c_int, C.c_float, C.c_int, vp, vp, vp, C.c_int, i32p]),
    "borb_search_local_points": (C.c_int, [vp, vp, vp, vp, vp, vp] + [C.c_float] * 9 + [vp] * 7 + [i32p]),
    "borb_search_local_points_batch": (C.c_int, [vp, vp, C.c_int, C.c_float, C.c_float, vp]),
    "borb_search_by_projection_last_batch": (C.c_int, [vp, vp, C.c_int, C.c_int, vp]),
    "borb_search_by_projection_kf_batch": (C.c_int, [vp, vp, C.c_int, C.c_int, vp]),
    "borb_search_by_projection_sim3_batch": (C.c_int, [vp, vp, C.c_int, vp]),
    "borb_search_by_sim3_batch": (C.c_int, [vp, vp, C.c_int, vp]),
    "borb_fuse": (C.c_int, [vp, vp, vp, vp, vp, vp, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int,
                            vp, i32p]),
    "borb_search_by_sim3": (C.c_int, [vp, vp, vp, vp, vp, vp, vp, vp, vp, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float,
                                      C.c_float, vp, i32p]),
    "borb_search_by_bow": (C.c_int, [vp, vp, C.c_int, vp, C.c_float, C.c_int, vp, vp]),
    "borb_search_by_bow_kf": (C.c_int, [vp, vp, vp, C.c_float, C.c_int, vp, i32p]),
    "borb_search_by_bow_batch": (C.c_int, [vp, vp, C.c_int, C.c_float, C.c_int, vp]),
    "borb_frames_compute_bow": (C.c_int, [vp, vp, vp, C.c_int, C.c_int, vp, vp, vp, vp, vp, vp, vp]),
    "borb_search_for_triangulation": (C.c_int, [vp, vp, vp, vp, C.c_float, C.c_float, C.c_int, C.c_int, vp, C.c_int, i32p]),
    "borb_search_for_triangulation_batch": (C.c_int, [vp, vp, C.c_int, C.c_int]),
    "borb_fuse_batch": (C.c_int, [vp, vp, C.c_int, vp]),
    "borb_voc_create": (C.c_int, [vp, vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(vp)]),
    "borb_voc_load_text": (C.c_int, [C.c_char_p, C.c_int, C.POINTER(vp)]),
    "borb_voc_destroy": (C.c_int, [vp]),
    "borb_voc_blob": (C.c_int, [vp, C.POINTER(vp), C.POINTER(C.c_size_t)]),
    "borb_voc_from_blob": (C.c_int, [vp, C.c_size_t, C.c_int, C.POINTER(vp)]),
    "borb_bow_transform": (C.c_int, [vp, vp, C.c_int, C.c_int, vp, vp, vp]),
    "borb_debug_candidates": (C.c_int, [vp, C.c_int, C.c_int, vp, C.c_int, i32p]),
    "borb_debug_selected": (C.c_int, [vp, C.c_int, C.c_int, vp, C.c_int, i32p]),
    "borb_debug_blurred": (C.c_int, [vp, C.c_int, C.c_int, vp, i32p, i32p]),
    "borb_nccl_unique_id": (C.c_int, [vp]),
    "borb_nccl_comm_create": (C.c_int, [vp, C.c_int, C.c_int, C.c_int, C.POINTER(vp)]),
    "borb_nccl_comm_destroy": (C.c_int, [vp]),
    "borb_voc_broadcast": (C.c_int, [vp, vp, C.c_int, C.c_int, C.c_int, C.POINTER(vp)]),
    "borb_compute_bow": (C.c_int, [vp, vp, C.c_int, C.c_int, vp, vp, i32p, vp, vp, vp, i32p]),
    "borb_matcher_set_timing": (C.c_int, [vp, C.c_int]),
    "borb_matcher_last_kernel_ms": (C.c_int, [vp, f32p]),
    "borb_matcher_launch_count": (C.c_int, [vp, C.POINTER(C.c_uint64)]),
    "borb_debug_set_poison": (C.c_int, [C.c_int]),
    "borb_debug_set_fast_mode": (C.c_int, [vp, C.c_int]),
    "borb_debug_brief_slots": (C.c_int, [vp, C.c_int, i32p]),
    "borb_debug_eval_math": (C.c_int, [C.c_int, vp, vp, C.c_int, C.c_float, C.c_int, vp]),
    "borb_launch_count": (C.c_int, [vp, C.POINTER(C.c_uint64)]),
    "borb_stage_times": (C.c_int, [vp, f32p]),
    "borb_set_timing": (C.c_int, [vp, C.c_int]),
}

_lib = None


def exported_names():
    return sorted(_SIGNATURES)


def load() -> C.CDLL:
    """Loads libborb.so; raises (never falls back) when it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                          "(orb_slam2_b200 has no CPU fallback)")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in _SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if the .so does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(status: int, where: str) -> None:
    if status != BORB_OK:
        detail = load().borb_last_error()
        raise BorbError(status, where, detail.decode() if detail else "")


def device_count() -> int:
    n = C.c_int32(0)
    st = load().borb_device_count(C.byref(n))
    return n.value if st == BORB_OK else 0


def ptr(a: np.ndarray):
    return a.ctypes.data_as(vp) if a is not None else None
