"""Errors of the calls without a handle: a refused argument returns OPB_E_INVALID and leaves a message that names the entry
point and the refused condition, in the per-thread string that opb_last_error(NULL) and opb_sp_last_error(NULL) both return.

The argument checks run before any CUDA call, so these tests need no GPU.  Every call below is refused, so no kernel is
launched and the non-null addresses passed are never dereferenced.  Four handle-free entry points have nothing to refuse:
opb_debug_set_pdl, opb_debug_set_ws_fill, opb_debug_split and opb_debug_kv_state_h take every argument."""
import ctypes as C
import math

import pytest
import torch

from onepose_b200 import _lib, pnp

OPB_E_INVALID = -1
P = 64                      # a non-null address; never dereferenced (the call is refused first)
MAX_HYPOTHESES = 65535 * 128
LK_WS = 1 << 30             # a workspace size every refused LK call below would accept


def _lk(**kw):
    """The arguments of opb_calc_optical_flow_pyr_lk without the stream: one 64 x 64 pair, 4 points, the tracker's parameters,
    with the given ones replaced."""
    a = dict(prev=P, prev_frame_pitch=4096, prev_row_pitch=64, next=P, next_frame_pitch=4096, next_row_pitch=64, B=1, H=64, W=64,
             sizes=None, pts=P, offsets=P, total=4, win_w=15, win_h=15, max_level=2, criteria_type=3, max_count=10, epsilon=0.03,
             min_eig_threshold=1e-4, flags=0, workspace=P, workspace_bytes=LK_WS, next_pts=P, status=P, err=P)
    a.update(kw)
    return tuple(a.values())


def _desc(**fields):
    return C.byref(_lib.gemm_desc(**fields))


# (entry point, arguments of a refused call without the stream, text of the refused condition)
CASES = [
    # null pointers
    ("opb_segmented_mean_f64", (None, P, 4, 8, P), "desc && seg_len && out"),
    ("opb_segmented_mean_channels_f64", (P, None, 4, 8, P), "desc && seg_len && out"),
    ("opb_gather_matches", (None, None, P, P, 2, 4, 10, P, P, None, None, P), "N == 0 || (matches0 && keypoints2d && pts2d && pts3d)"),
    ("opb_gather_matches", (P, None, P, P, 2, 4, 10, P, P, P, None, P), "!mconf || mscores0"),
    ("opb_gather_matches_objects", (P, None, P, P, None, P, 2, 4, P, P, None, None, P), "kp3_first && kp3_count"),
    ("opb_ransac_epnp", (P, P, None, P, 1, 100, 5.0, 0, P, P, P, P), "K && pts2d && pts3d && offsets && workspace"),
    ("opb_ransac_epnp_cv", (P, P, P, P, 1, 100, 5.0, 0.99, P, P, P, P, None), "iterations && confidence >= 0.0"),
    ("opb_crop_resize", (None, 100, 10, 1, 10, 10, P, P, 16, P, P, P, P), "frames && box && K && image"),
    ("opb_warp_crop_u8", (P, 100, 10, 1, 10, 10, P, None, 8, 8, None, P, None), "(frames != nullptr) == (out != nullptr)"),
    ("opb_warp_crop_u8", (None, 0, 0, 1, 0, 0, P, P, 8, 8, None, P, None), "(K != nullptr) == (K_crop != nullptr)"),
    ("opb_debug_gemm", (None,), "d && d->backend >= 0"),
    ("opb_calc_optical_flow_pyr_lk", _lk(workspace=None), "prev && next && offsets && workspace"),
    ("opb_calc_optical_flow_pyr_lk", _lk(err=None), "total == 0 || (pts && next_pts && status && err)"),
    ("opb_flow_compact", (P, P, P, None, 1, 10, P, P, P, P, P, P), "counts && offsets && n_tracked"),
    ("opb_flow_compact", (P, None, P, P, 1, 10, P, P, P, P, P, P), "cap == 0 || (status && pts2d && pts3d"),
    ("opb_flow_reprojection", (P, None, P, P, P, 1, P), "K && pose && offsets && dist"),
    # a workspace that does not start at a multiple of 16 bytes: the derivative planes are read and written as short2
    ("opb_calc_optical_flow_pyr_lk", _lk(workspace=P + 1), "((uintptr_t)workspace & 15) == 0"),
    # counts <= 0
    ("opb_segmented_mean_f64", (P, P, 4, 0, P), "D > 0"),
    ("opb_segmented_mean_channels_f64", (P, P, 4, 0, P), "D > 0"),
    ("opb_segmented_mean_scores_f64", (P, P, -1, P), "M > 0"),
    ("opb_gather_features3d", (P, None, 0, 10, None, 10, P, None, 10), "dim > 0"),
    ("opb_gather_matches", (P, None, P, P, 2, -1, 10, P, P, None, None, P), "N >= 0"),
    ("opb_epnp", (P, P, P, P, 0, P, P), "B > 0"),
    ("opb_boxes_from_poses", (P, P, P, 1, 0, None, P), "n_corners > 0"),
    ("opb_estimate_affine_partial", (P, P, P, 0, 3.0, 2000, 0.99, 10, P, None, P, P), "B > 0"),
    ("opb_boxes_from_matches", (P, P, P, 1, 16, P, P, 0, P, 1, 1, 480, 640, P, P, P, P, P), "cap_query > 0"),
    ("opb_debug_cv_subsets", (4, 1, 1, P), "n >= 5"),
    ("opb_calc_optical_flow_pyr_lk", _lk(B=0), "B > 0"),
    ("opb_flow_compact", (P, P, P, P, 0, 10, P, P, P, P, P, P), "B > 0"),
    ("opb_flow_compact", (P, P, P, P, 1, -1, P, P, P, P, P, P), "cap >= 0"),
    ("opb_flow_reprojection", (P, P, P, P, P, 0, P), "B > 0"),
    # other bounds
    ("opb_gather_features3d", (P, None, 8, 10, None, 11, P, None, 10), "n_idx <= n_out"),
    ("opb_gather_features3d", (P, None, 65536, 10, None, 10, P, None, 10), "dim <= 65535"),
    ("opb_gather_matches", (P, None, P, P, 65536, 65536, 10, P, P, None, None, P), "(int64_t)B * N <= (int64_t)INT32_MAX"),
    ("opb_crop_resize", (P, 100, 10, 65536, 10, 10, P, P, 16, P, P, P, P), "B <= 65535"),
    ("opb_warp_crop_u8", (P, 100, 10, 65536, 10, 10, P, None, 8, 8, P, P, None), "B <= 65535"),
    ("opb_warp_crop_u8", (P, 100, 5, 1, 10, 10, P, None, 8, 8, P, P, None), "row_pitch >= W"),
    ("opb_boxes_from_matches", (P, P, P, 257, 16, P, P, 16, P, 1, 1, 480, 640, P, P, P, P, P), "V <= opb::kMaxViews"),
    ("opb_boxes_from_matches", (P, P, P, 1, 8193, P, P, 16, P, 1, 1, 480, 640, P, P, P, P, P), "cap_ref <= opb::kMaxRefPoints"),
    ("opb_ransac_pnp", (P, P, P, P, 1, MAX_HYPOTHESES + 1, 5.0, 0, P, P, P, P), "hypotheses <= opb::kMaxHypotheses"),
    ("opb_ransac_epnp", (P, P, P, P, 1, 100, 0.0, 0, P, P, P, P), "reproj_error > 0.0"),
    ("opb_crop_resize", (P, 100, 10, 1, 10, 10, P, P, 12, P, P, P, P), "crop_size % 8 == 0"),
    ("opb_boxes_from_matches", (P, P, P, 1, 16, P, P, 16, P, 2, 1, 480, 640, P, P, P, P, P), "(matches_int64 == 0 || matches_int64 == 1)"),
    ("opb_calc_optical_flow_pyr_lk", _lk(B=65536), "B <= 65535"),
    ("opb_calc_optical_flow_pyr_lk", _lk(W=32768, prev_row_pitch=32768, next_row_pitch=32768), "W <= kMaxSideLk"),
    ("opb_calc_optical_flow_pyr_lk", _lk(next_row_pitch=63), "next_row_pitch >= W"),
    ("opb_calc_optical_flow_pyr_lk", _lk(prev_frame_pitch=-1), "prev_frame_pitch >= 0"),
    ("opb_calc_optical_flow_pyr_lk", _lk(win_h=14), "win_h % 2 == 1"),
    ("opb_calc_optical_flow_pyr_lk", _lk(win_w=33), "win_w <= kMaxWin"),
    ("opb_calc_optical_flow_pyr_lk", _lk(max_level=5), "max_level <= kMaxLevel"),
    ("opb_calc_optical_flow_pyr_lk", _lk(criteria_type=4), "(criteria_type & ~3) == 0"),
    ("opb_calc_optical_flow_pyr_lk", _lk(max_count=101), "max_count <= 100"),
    ("opb_calc_optical_flow_pyr_lk", _lk(epsilon=math.nan), "epsilon >= 0.0"),
    ("opb_calc_optical_flow_pyr_lk", _lk(min_eig_threshold=-1e-9), "min_eig_threshold >= 0.0"),
    ("opb_calc_optical_flow_pyr_lk", _lk(flags=4), "flags == 0"),
    ("opb_calc_optical_flow_pyr_lk", _lk(workspace_bytes=1000), "workspace_bytes >= (int64_t)B * (int64_t)L.pair_bytes"),
    ("opb_flow_compact", (P, P, P, P, 65536, 32768, P, P, P, P, P, P), "(int64_t)B * cap <= (int64_t)INT32_MAX"),
    ("opb_debug_gemm", (_desc(backend=2),), "d->backend <= 1"),
    ("opb_debug_gemm", (_desc(b2_mode=3),), "d->b2_mode <= 2"),
    ("opb_debug_gemm", (_desc(backend=1, epi=_lib.EPI_QSCALE),), "p.epi == EPI_F32"),
    # confidence
    ("opb_ransac_epnp_cv", (P, P, P, P, 1, 100, 5.0, 1.5, P, P, P, P, P), "confidence <= 1.0"),
    ("opb_ransac_epnp_cv", (P, P, P, P, 1, 100, 5.0, math.nan, P, P, P, P, P), "confidence >= 0.0"),
    ("opb_estimate_affine_partial", (P, P, P, 1, 3.0, 2000, 1.0, 10, P, None, P, P), "confidence < 1.0"),
    ("opb_estimate_affine_partial", (P, P, P, 1, math.inf, 2000, 0.99, 10, P, None, P, P), "isfinite(threshold)"),
]

# the test hooks take no stream; (entry point, arguments, text of the refused condition)
HOOK_CASES = [
    ("opb_debug_set_conv_halo", (2,), "mode >= 0 && mode <= 1"),
    ("opb_debug_set_cv_wave", (-1,), "wave >= 0"),
    ("opb_debug_set_cv_trace", (P, None, None, 0), "capacity > 0 || (capacity == 0 && !samples && !counts)"),
    ("opb_debug_set_cv_trace", (None, None, None, -1), "capacity > 0 || (capacity == 0 && !samples && !counts)"),
    ("opb_debug_set_affine_trace", (None, None, P, 0), "capacity > 0 || (capacity == 0 && !samples && !counts && !models)"),
]

# calls that take no stream; (entry point, arguments, text of the refused condition)
NO_STREAM_CASES = [
    ("opb_optical_flow_workspace_bytes", (1, 64, 64, 2, None), "bytes && B > 0"),
    ("opb_optical_flow_workspace_bytes", (1, 64, 32768, 2, C.byref(C.c_int64())), "W <= opb::kMaxSideLk"),
    ("opb_optical_flow_workspace_bytes", (1, 64, 64, 5, C.byref(C.c_int64())), "max_level <= opb::kMaxLevel"),
]

NO_REFUSAL = {"opb_debug_set_pdl", "opb_debug_set_ws_fill", "opb_debug_split", "opb_debug_kv_state_h"}


def _messages(lib):
    return lib.opb_last_error(None), lib.opb_sp_last_error(None)


def _refused(name, args, cond):
    lib = _lib.load()
    rc = getattr(lib, name)(*args)
    assert rc == OPB_E_INVALID, (name, rc)
    for msg in _messages(lib):
        assert msg.startswith(name.encode() + b": "), (name, msg)
        assert cond.encode() in msg, (name, cond, msg)


@pytest.mark.parametrize("name,args,cond", CASES, ids=[f"{c[0]}:{c[2]}" for c in CASES])
def test_a_refused_call_names_its_entry_point_and_condition(name, args, cond):
    _refused(name, (*args, None), cond)


@pytest.mark.parametrize("name,args,cond", HOOK_CASES, ids=[f"{c[0]}:{c[2]}" for c in HOOK_CASES])
def test_a_refused_test_hook_names_itself_and_its_condition(name, args, cond):
    _refused(name, args, cond)


@pytest.mark.parametrize("name,args,cond", NO_STREAM_CASES, ids=[f"{c[0]}:{c[2]}" for c in NO_STREAM_CASES])
def test_a_refused_call_without_a_stream_names_its_entry_point_and_condition(name, args, cond):
    _refused(name, args, cond)


def test_every_handle_free_entry_point_that_can_refuse_is_covered():
    covered = {c[0] for c in CASES + HOOK_CASES + NO_STREAM_CASES}
    assert covered == {
        "opb_segmented_mean_f64", "opb_segmented_mean_channels_f64", "opb_segmented_mean_scores_f64", "opb_gather_features3d",
        "opb_debug_gemm", "opb_debug_set_conv_halo",
        "opb_gather_matches", "opb_gather_matches_objects", "opb_ransac_pnp", "opb_epnp", "opb_ransac_epnp", "opb_ransac_epnp_cv",
        "opb_debug_set_cv_wave", "opb_debug_set_cv_trace", "opb_debug_cv_subsets", "opb_boxes_from_poses", "opb_crop_resize",
        "opb_warp_crop_u8", "opb_estimate_affine_partial", "opb_boxes_from_matches", "opb_debug_set_affine_trace",
        "opb_optical_flow_workspace_bytes", "opb_calc_optical_flow_pyr_lk", "opb_flow_compact", "opb_flow_reprojection",
    }
    assert len(covered | NO_REFUSAL) == 29 and covered | NO_REFUSAL <= set(_lib.SYMBOLS)


def test_a_later_refusal_replaces_the_message():
    lib = _lib.load()
    _refused("opb_crop_resize", (P, 100, 10, 1, 10, 10, P, P, 12, P, P, P, P, None), "crop_size % 8 == 0")
    _refused("opb_boxes_from_matches", (P, P, P, 0, 16, P, P, 16, P, 1, 1, 480, 640, P, P, P, P, P, None), "V > 0")
    assert all(b"crop_size" not in m for m in _messages(lib))


def test_a_failed_create_still_leaves_its_own_message():
    lib = _lib.load()
    _refused("opb_epnp", (P, P, P, P, 0, P, P, None), "B > 0")
    h = C.c_void_p()
    assert lib.opb_create(C.byref(_lib.OpbConfig(256, 4, 0.0, 0.2, 1, 1, 0, 0)), C.byref(h)) == OPB_E_INVALID
    assert all(b"scale_factor" in m for m in _messages(lib))
    assert lib.opb_sp_create(C.byref(_lib.OpbSpConfig(128, 4, 0.005, -1, 4, 1, 0)), C.byref(h)) == OPB_E_INVALID
    assert all(b"descriptor_dim" in m for m in _messages(lib))


def test_check_raises_the_message_of_a_call_without_a_handle():
    lib = _lib.load()
    with pytest.raises(_lib.OpbError, match=r"OPB_E_INVALID: opb_debug_set_cv_wave: wave >= 0"):
        _lib.check(lib.opb_debug_set_cv_wave(-1))


@pytest.mark.gpu
def test_a_refusal_only_the_library_makes_reaches_python_with_its_message():
    dev = torch.device("cuda")
    K = torch.eye(3, dtype=torch.float64, device=dev)[None]
    pts2d = torch.zeros(4, 2, dtype=torch.float64, device=dev)
    pts3d = torch.zeros(4, 3, dtype=torch.float64, device=dev)
    offsets = torch.tensor([0, 4], dtype=torch.int32, device=dev)
    with pytest.raises(_lib.OpbError, match=r"opb_ransac_pnp: .*hypotheses <= opb::kMaxHypotheses"):
        pnp.ransac_pnp_batch(K, pts2d, pts3d, offsets, hypotheses=MAX_HYPOTHESES + 1)
