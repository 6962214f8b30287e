"""ctypes binding of the C ABI in include/onepose_b200.h.

There is deliberately NO fallback: if the shared library is missing or does not
load, importing the matcher raises.  (The oracle under /oracle is test
infrastructure and is never imported from here.)
"""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libonepose_b200.so")

OPB_OK = 0
ERRORS = {-1: "OPB_E_INVALID", -2: "OPB_E_CUDA", -3: "OPB_E_STATE", -4: "OPB_E_RANGE", -5: "OPB_E_NOT_IMPLEMENTED"}


class OpbConfig(C.Structure):
    _fields_ = [
        ("descriptor_dim", C.c_int32), ("num_heads", C.c_int32), ("scale_factor", C.c_float),
        ("match_threshold", C.c_float), ("include_self", C.c_int32), ("additional", C.c_int32),
        ("with_linear_transform", C.c_int32), ("device", C.c_int32),
    ]


class OpbSpConfig(C.Structure):
    _fields_ = [
        ("descriptor_dim", C.c_int32), ("nms_radius", C.c_int32), ("keypoint_threshold", C.c_float), ("max_keypoints", C.c_int32),
        ("remove_borders", C.c_int32), ("align_corners", C.c_int32), ("device", C.c_int32),
    ]


# every symbol include/onepose_b200.h declares: (restype, argtypes)
_P = C.c_void_p
_I = C.c_int32
SYMBOLS = {
    "opb_create": (C.c_int, [C.POINTER(OpbConfig), C.POINTER(_P)]),
    "opb_destroy": (None, [_P]),
    "opb_last_error": (C.c_char_p, [_P]),
    "opb_load_weight": (C.c_int, [_P, C.c_char_p, _P, C.c_size_t]),
    "opb_finalize_weights": (C.c_int, [_P]),
    "opb_set_object": (C.c_int, [_P, _P, _P, _I, _I, _P]),
    "opb_reserve_workspace": (C.c_int, [_P, _I, _I]),
    "opb_forward": (C.c_int, [_P, _P, _P, _I, _I, _P, _P, _P, _P, _P, _P]),
    "opb_forward_host": (C.c_int, [_P, _P, _P, _I, _I, _P, _P, _P, _P, _P, _I, _P]),
    "opb_check_range": (C.c_int, [_P, _P]),
    "opb_poll_range": (C.c_int, [_P]),
    "opb_last_launch_count": (C.c_int, [_P]),
    "opb_set_chunk_frames": (C.c_int, [_P, _I]),
    "opb_set_hoist": (C.c_int, [_P, _I]),
    "opb_set_profiling": (C.c_int, [_P, _I]),
    "opb_get_profile_entry": (C.c_int, [_P, C.c_char_p, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(_I)]),
    "opb_get_profile": (C.c_int, [_P, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(_I), C.POINTER(C.c_double)]),
    "opb_segmented_mean_f64": (C.c_int, [_P, _P, _I, _I, _P, _P]),
    "opb_segmented_mean_scores_f64": (C.c_int, [_P, _P, _I, _P, _P]),
    "opb_gather_features3d": (C.c_int, [_P, _P, _I, C.c_int64, _P, C.c_int64, _P, _P, C.c_int64, _P]),
    "opb_ransac_pnp": (C.c_int, [_P, _P, _P, _P, _I, _I, C.c_double, C.c_uint64, _P, _P, _P, _P, _P]),
    "opb_gather_matches": (C.c_int, [_P, _P, _P, _P, _I, _I, _I, _P, _P, _P, _P, _P, _P]),
    "opb_debug_set_pdl": (C.c_int, [_I]),
    "opb_debug_set_ws_fill": (C.c_int, [_I]),
    "opb_debug_set_kv_passes": (C.c_int, [_P, _I]),
    "opb_debug_set_identity_diag": (C.c_int, [_P, _I]),
    "opb_debug_gemm": (C.c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _P]),
    "opb_debug_gemm_timeline": (C.c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _P, _P]),
    "opb_debug_kv_state_h": (C.c_int, [_P, _I, _I, _I, _I, _P, C.POINTER(_I), _P]),
    "opb_debug_gemm_aconv": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I, _P, _P]),
    "opb_debug_split": (C.c_int, [_P, _P, _P, C.c_size_t, _P]),
    "opb_debug_read": (C.c_int, [_P, _I, _P, C.c_size_t, C.POINTER(C.c_int64), _P]),
    # SuperPoint extractor
    "opb_sp_create": (C.c_int, [C.POINTER(OpbSpConfig), C.POINTER(_P)]),
    "opb_sp_destroy": (None, [_P]),
    "opb_sp_last_error": (C.c_char_p, [_P]),
    "opb_sp_load_weight": (C.c_int, [_P, C.c_char_p, _P, C.c_size_t]),
    "opb_sp_finalize_weights": (C.c_int, [_P]),
    "opb_sp_detect": (C.c_int, [_P, _P, _I, _I, _I, _P, _P]),
    "opb_sp_describe": (C.c_int, [_P, _P, _P, _P, _P, _I, _P]),
    "opb_sp_forward": (C.c_int, [_P, _P, _I, _I, _I, _P, _P, _P, _P, _I, _P]),
    "opb_sp_last_launch_count": (C.c_int, [_P]),
    "opb_sp_set_profiling": (C.c_int, [_P, _I]),
    "opb_sp_get_profile": (C.c_int, [_P, _I, C.c_char_p, C.c_size_t, C.POINTER(C.c_double), C.POINTER(C.c_double)]),
    "opb_sp_debug_set_stop": (C.c_int, [_P, _I]),
    "opb_debug_set_conv_halo": (C.c_int, [_I]),
    "opb_sp_debug_read": (C.c_int, [_P, _I, _P, C.c_size_t, C.POINTER(C.c_int64), _P]),
}

_lib = None


def load() -> C.CDLL:
    """Load the in-tree CUDA library; raise loudly if it is not there."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: build it with `python -m onepose_b200.build` "
            "(there is no CPU or PyTorch fallback for this path)")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)  # AttributeError if the .so does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


class OpbError(RuntimeError):
    pass


def check_sp(rc: int, handle=None, lib=None):
    """Status check for the opb_sp_* (extractor) entry points."""
    if rc == OPB_OK:
        return
    msg = (lib or load()).opb_sp_last_error(handle)
    raise OpbError(f"{ERRORS.get(rc, rc)}: {msg.decode() if msg else ''}")


def check(rc: int, handle=None):
    if rc == OPB_OK:
        return
    msg = load().opb_last_error(handle)
    raise OpbError(f"{ERRORS.get(rc, rc)}: {msg.decode() if msg else ''}")
