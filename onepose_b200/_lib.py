"""ctypes binding of the C ABI in include/onepose_b200.h.

There is deliberately NO fallback: if the shared library is missing or does not
load, importing the matcher raises.  (The oracle under /oracle is test
infrastructure and is never imported from here.)
"""
from __future__ import annotations

import ctypes as C
import os

import torch

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


_P = C.c_void_p
_I = C.c_int32


class OpbDebugGemmDesc(C.Structure):
    """opb_debug_gemm_desc: one problem of the GEMM core (see the header).  Pointer fields take device addresses (ints)."""
    _fields_ = [
        ("epi", _I), ("bn", _I), ("rows", _I), ("n_out", _I), ("K1", _I), ("K2", _I), ("batch", _I),
        ("a_batch_rows", C.c_int64), ("b_batch_rows", C.c_int64),
        ("a1_hi", _P), ("a1_lo", _P), ("a1_ld", _I), ("a2_hi", _P), ("a2_lo", _P), ("a2_ld", _I),
        ("b1_hi", _P), ("b1_lo", _P), ("b1_ld", _I), ("b2_hi", _P), ("b2_lo", _P), ("b2_ld", _I),
        ("b2_mode", _I), ("a_hi_only", _I),
        ("a_raw", _P), ("a_raw_ld", _I), ("mu", _P), ("rstd", _P),
        ("B", _I), ("N", _I), ("M", _I), ("n_pad", _I), ("m_pad", _I), ("nlen", _P), ("mlen", _P),
        ("bias", _P), ("c", _P), ("ldc", _I), ("out_hi", _P), ("out_lo", _P), ("out_ld", _I),
        ("kmean", _P), ("cross", _I), ("statpart", _P),
        ("inv_scale", C.c_float), ("rowsum_part", _P), ("colsum_part", _P), ("inv_rowsum", _P), ("inv_colsum", _P),
        ("conf", _P), ("conf_ld", _I), ("rowbest", _P), ("colbest", _P),
        ("taps", _I), ("kb_per_tap", _I), ("tap_off", _I * 9), ("cv_w2", _I), ("cv_h", _I), ("cv_w", _I), ("cv_ppad", _I),
        ("relu", _I), ("range_flag", _P),
        ("max_ctas", _I), ("backend", _I),
    ]


# GemmEpilogue values of opb_debug_gemm_desc.epi
EPI_F32, EPI_F32_STATS, EPI_QSCALE, EPI_L2NORM, EPI_SCORE_SUMS, EPI_SCORE_CONF, EPI_QKV, EPI_BIAS_PLANES, EPI_CONV = 0, 1, 2, 5, 6, 7, 9, 10, 11


def gemm_desc(**fields) -> OpbDebugGemmDesc:
    """An opb_debug_gemm_desc with the given fields set and every other field zero (torch tensors stand for their data_ptr)."""
    d = OpbDebugGemmDesc()
    for k, v in fields.items():
        if k == "tap_off":
            d.tap_off[:] = list(v) + [0] * (9 - len(v))
        else:
            setattr(d, k, v.data_ptr() if hasattr(v, "data_ptr") else v)
    return d


# every symbol include/onepose_b200.h declares: (restype, argtypes)
SYMBOLS = {
    "opb_create": (C.c_int, [C.POINTER(OpbConfig), C.POINTER(_P)]),
    "opb_destroy": (None, [_P]),
    "opb_last_error": (C.c_char_p, [_P]),
    "opb_load_weight": (C.c_int, [_P, C.c_char_p, _P, C.c_size_t]),
    "opb_finalize_weights": (C.c_int, [_P]),
    "opb_set_object": (C.c_int, [_P, _P, _P, _I, _I, _P]),
    "opb_reserve_workspace": (C.c_int, [_P, _I, _I]),
    "opb_forward": (C.c_int, [_P, _P, _P, _I, _I, _P, _P, _P, _P, _P, _P]),
    "opb_add_object": (C.c_int, [_P, _P, _P, _I, _I, _P, C.POINTER(_I)]),
    "opb_remove_object": (C.c_int, [_P, _I]),
    "opb_forward_objects": (C.c_int, [_P, _P, _P, _P, _I, _I, _I, _P, _P, _P, _P, _P, _P]),
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
    "opb_segmented_mean_channels_f64": (C.c_int, [_P, _P, _I, _I, _P, _P]),
    "opb_segmented_mean_scores_f64": (C.c_int, [_P, _P, _I, _P, _P]),
    "opb_gather_features3d": (C.c_int, [_P, _P, _I, C.c_int64, _P, C.c_int64, _P, _P, C.c_int64, _P]),
    "opb_ransac_pnp": (C.c_int, [_P, _P, _P, _P, _I, _I, C.c_double, C.c_uint64, _P, _P, _P, _P, _P]),
    "opb_epnp": (C.c_int, [_P, _P, _P, _P, _I, _P, _P, _P]),
    "opb_ransac_epnp": (C.c_int, [_P, _P, _P, _P, _I, _I, C.c_double, C.c_uint64, _P, _P, _P, _P, _P]),
    "opb_ransac_epnp_cv": (C.c_int, [_P, _P, _P, _P, _I, _I, C.c_double, C.c_double, _P, _P, _P, _P, _P, _P]),
    "opb_debug_set_cv_wave": (C.c_int, [_I]),
    "opb_debug_set_cv_trace": (C.c_int, [_P, _P, _P, _I]),
    "opb_debug_cv_subsets": (C.c_int, [_I, _I, _I, _P, _P]),
    "opb_gather_matches": (C.c_int, [_P, _P, _P, _P, _I, _I, _I, _P, _P, _P, _P, _P, _P]),
    "opb_gather_matches_objects": (C.c_int, [_P, _P, _P, _P, _P, _P, _I, _I, _P, _P, _P, _P, _P, _P]),
    "opb_grey_frames": (C.c_int, [_P, C.c_int64, C.c_int64, _I, _I, _I, _I, _P, C.c_int64, C.c_int64, _P, _P]),
    "opb_boxes_from_poses": (C.c_int, [_P, _P, _P, _I, _I, _P, _P, _P]),
    "opb_crop_resize": (C.c_int, [_P, C.c_int64, C.c_int64, _I, _I, _I, _P, _P, _I, _P, _P, _P, _P, _P]),
    "opb_crop_resize_indexed": (C.c_int, [_P, C.c_int64, C.c_int64, _I, _I, _I, _P, _I, _P, _P, _I, _P, _P, _P, _P, _P]),
    "opb_warp_crop_u8": (C.c_int, [_P, C.c_int64, C.c_int64, _I, _I, _I, _P, _P, _I, _I, _P, _P, _P, _P]),
    "opb_crop_resize_colour": (C.c_int, [_P, C.c_int64, C.c_int64, _I, _I, _I, _I, _P, _I, _P, _P, _I, _P, _P, _P, _P, _P]),
    "opb_scan_poses": (C.c_int, [_P, _P, _I, _P, _P, _I, _I, _P, _P, _P, _P, _P, _P, _P]),
    "opb_scan_crop_geometry": (C.c_int, [_P, _P, _P, _P, _I, _P, _I, _P, _P, _P]),
    "opb_estimate_affine_partial": (C.c_int, [_P, _P, _P, _I, C.c_double, _I, C.c_double, _I, _P, _P, _P, _P, _P]),
    "opb_boxes_from_matches": (C.c_int, [_P, _P, _P, _I, _I, _P, _P, _I, _P, _I, _I, _I, _I, _P, _P, _P, _P, _P, _P]),
    "opb_boxes_from_matches_objects": (C.c_int, [_P, _P, _P, _I, _I, _P, _P, _I, _P, _P, _I, _I, _P, _P, _I, _I, _I, _I, _P, _P, _P, _P, _P,
                                                 _P]),
    "opb_debug_set_affine_trace": (C.c_int, [_P, _P, _P, _I]),
    "opb_optical_flow_workspace_bytes": (C.c_int, [_I, _I, _I, _I, C.POINTER(C.c_int64)]),
    "opb_calc_optical_flow_pyr_lk": (C.c_int, [_P, C.c_int64, C.c_int64, _P, C.c_int64, C.c_int64, _I, _I, _I, _P, _P, _P, _I, _I, _I, _I, _I, _I,
                                               C.c_double, C.c_double, _I, _P, C.c_int64, _P, _P, _P, _P]),
    "opb_flow_compact": (C.c_int, [_P, _P, _P, _P, _I, _I, _P, _P, _P, _P, _P, _P, _P]),
    "opb_flow_reprojection": (C.c_int, [_P, _P, _P, _P, _P, _I, _P, _P]),
    "opb_track_gate": (C.c_int, [_P, _I, _P, _P, _P, _P, _P]),
    "opb_track_select": (C.c_int, [_P, _P, _P, _I, _P, _P, _P, _P, _P, _P, _P, _P]),
    "opb_sfm_filter_workspace_bytes": (C.c_int, [_I, C.POINTER(C.c_int64)]),
    "opb_sfm_filter_points": (C.c_int, [_P, _P, _P, _I, _I, _P, _P, C.c_int64, _P, _P, _P, _P, _P]),
    "opb_sfm_merge_workspace_bytes": (C.c_int, [_I, C.POINTER(C.c_int64)]),
    "opb_sfm_merge_points": (C.c_int, [_P, _P, _P, _I, C.c_double, _P, C.c_int64, _P, _P, _P, _P, _P, _P, _P, _P]),
    "opb_sfm_gather_workspace_bytes": (C.c_int, [_I, _I, _I, C.POINTER(C.c_int64)]),
    "opb_sfm_gather_observations": (C.c_int, [_P, _P, _I, _I, _P, _P, _I, _P, _P, _P, _P, C.c_int64, _P, _P, _P, _P, _P]),
    "opb_sfm_gather_features": (C.c_int, [_P, C.c_int64, _I, _I, _I, _P, _P, _P, _P, _P]),
    "opb_sfm_assign_workspace_bytes": (C.c_int, [_I, _I, C.POINTER(C.c_int64)]),
    "opb_sfm_assign_pairs": (C.c_int, [_P, _P, _I, _I, _P, _P, _I, _P, C.c_int64, _P, _P, _P, _P]),
    "opb_json_float_repr": (C.c_int, [_P, C.c_int64, _P, _P, _P]),
    "opb_json_float_repr_host": (C.c_int, [_P, C.c_int64, _P, _P]),
    "opb_anno2d_text_workspace_bytes": (C.c_int, [_I, C.c_int64, C.POINTER(C.c_int64)]),
    "opb_anno2d_text_lengths": (C.c_int, [_P, _P, _I, C.c_int64, C.c_int64, _I, _I, _P, _P, _P, _P, C.c_int64, _P, C.c_int64, _P, _P]),
    "opb_anno2d_text_write": (C.c_int, [_P, _P, _I, C.c_int64, _I, _I, _P, _P, _P, _P, C.c_int64, _P, _P, _P, _P]),
    "opb_png_workspace_bytes": (C.c_int, [_I, _I, _I, _I, C.POINTER(C.c_int64)]),
    "opb_png_frame_bytes": (C.c_int, [_I, _I, _I, C.POINTER(C.c_int64)]),
    "opb_png_encode": (C.c_int, [_P, C.c_int64, C.c_int64, _I, _I, _I, _I, _P, C.c_int64, _P, C.c_int64, _P, _P]),
    "opb_png_decode_workspace_bytes": (C.c_int, [_I, _I, _I, C.c_int64, C.POINTER(C.c_int64)]),
    "opb_png_decode": (C.c_int, [_P, _P, _I, _I, _I, _I, _P, C.c_int64, _P, C.c_int64, C.c_int64, _P, _P, _P]),
    "opb_debug_set_pdl": (C.c_int, [_I]),
    "opb_debug_set_ws_fill": (C.c_int, [_I]),
    "opb_debug_set_kv_passes": (C.c_int, [_P, _I]),
    "opb_debug_gemm": (C.c_int, [C.POINTER(OpbDebugGemmDesc), _P]),
    "opb_debug_kv_state_h": (C.c_int, [_P, _I, _I, _I, _I, _P, C.POINTER(_I), _P]),
    "opb_debug_split": (C.c_int, [_P, _P, _P, C.c_size_t, _P]),
    "opb_debug_block": (C.c_int, [_I, _I, _I, _I, _I, _P, _P, _P, _P]),
    "opb_debug_set_stop": (C.c_int, [_P, _I, _I]),
    "opb_debug_set_stop_pass": (C.c_int, [_P, _I, _I]),
    "opb_debug_invalidate_prologues": (C.c_int, [_P]),
    "opb_debug_stopped_layout": (C.c_int, [_P, C.POINTER(_I)]),
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
    "opb_sp_check_range": (C.c_int, [_P, _P]),
    "opb_sp_poll_range": (C.c_int, [_P]),
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


def check(rc: int, handle=None, kind: str = "matcher"):
    """Raise OpbError with the library's message unless ``rc`` is OPB_OK.  ``handle`` is the handle the call took -- a
    matcher's, or an extractor's with ``kind="extractor"`` -- or None for a call without one."""
    if rc == OPB_OK:
        return
    lib = load()
    msg = (lib.opb_sp_last_error if kind == "extractor" else lib.opb_last_error)(handle)
    raise OpbError(f"{ERRORS.get(rc, rc)}: {msg.decode() if msg else ''}")


def cuda_device(t: torch.Tensor) -> torch.device:
    if t.device.type != "cuda":
        raise RuntimeError("onepose_b200 has no CPU path: tensors must be on a CUDA device")
    return t.device


def call(dev: torch.device, name: str, *args):
    """Run the handle-free entry point ``name`` on device ``dev`` and its current stream, which is appended to ``args``.
    Tensors pass as their data_ptr() and None as NULL; a failure raises OpbError with the library's message."""
    fn = getattr(load(), name)
    args = [a.data_ptr() if isinstance(a, torch.Tensor) else a for a in args]
    with torch.cuda.device(dev):
        check(fn(*args, torch.cuda.current_stream(dev).cuda_stream))
