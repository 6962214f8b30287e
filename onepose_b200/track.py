"""The reference tracker's flow-only tracking on the GPU: its keyframe gate, motion prediction and choice of the reported pose.

With ``use_tracking`` the reference's live demo (``inference_demo.py:253-299``, ``track_interval = 5``) runs, per frame of a
track: ``update_kf`` every 5th frame (the frame's inlier pairs become the keyframe unless the matcher pose is more than
10 cm / 10 deg from the last reported pose), ``add_kf`` at the first frame, and ``track()`` on every other frame, which runs
``flow_track`` and reports the flow pose, a motion-predicted pose or the matcher pose (``src/tracker/ba_tracker.py:105-293,
:727-802``; bundle adjustment is not part of this path).  ``step`` does that for B tracks in one call on the device, with
no host synchronisation:

    state = track.init_state(B, cap, crop_size, device)
    for each frame:                                       # res: the frame's poses_from_matches[_objects] result on crops
        out = track.step(state, res, crops, K_crop)
        pose = out["pose"]                               # the demo's pose_opt

The state is a dict of device tensors the caller owns; ``reset(state, mask)`` starts the masked tracks over.  The state
machine runs in ``csrc/track.cu`` (``opb_track_gate`` / ``opb_track_select``); the keyframes and the flow pose are
``flow.keyframes_from_poses`` and ``flow.flow_track``.
"""
from __future__ import annotations

import torch

from . import _lib, flow

TRACK_INTERVAL = 5             # inference_demo.py:144
INIT_COUNT = 3                 # BATracker.__init__'s init_cnt
HISTORY = 3                    # motion_prediction reads pose_list[-3:]
# gate outcomes (opb_track_gate)
GATE_NONE, GATE_ADD, GATE_ACCEPT, GATE_REJECT = 0, 1, 2, 3
# branch codes of the reported pose (opb_track_select)
FLOW, MOTION, PRED, INIT, KEYFRAME = 0, 1, 2, 3, 4


def init_state(B: int, cap: int, crop_size: int, device) -> dict:
    """The state of B new tracks on ``device``: every track at its first frame, keyframes of ``cap`` rows and
    ``crop_size``-square crops (all zero, no points).  ``cap`` must be the pairs per frame of the results ``step`` gets."""
    B, cap, S = int(B), int(cap), int(crop_size)
    if B < 1 or cap < 1 or S < 1:
        raise ValueError(f"B, cap and crop_size must be >= 1, got {B}, {cap}, {S}")
    dev = torch.device(device)
    _lib.cuda_device(torch.empty(0, device=dev))
    i32 = dict(dtype=torch.int32, device=dev)
    return {"frame": torch.zeros(B, dtype=torch.int64, device=dev), "hist": torch.zeros(B, HISTORY, 4, 4, dtype=torch.float64, device=dev),
            "hist_len": torch.zeros(B, **i32), "init_cnt": torch.full((B,), INIT_COUNT, **i32), "use_motion_cnt": torch.zeros(B, **i32),
            "kf": {"image": torch.zeros(B, S, S, dtype=torch.uint8, device=dev), "pts2d": torch.zeros(B, cap, 2, dtype=torch.float32, device=dev),
                   "pts3d": torch.zeros(B, cap, 3, dtype=torch.float32, device=dev), "counts": torch.zeros(B, **i32)}}


def reset(state: dict, mask: torch.Tensor) -> None:
    """``BATracker.reset`` for the tracks where ``mask`` (bool [B]) is set, restricted to this path's fields: an empty history,
    init_cnt 3, use_motion_cnt 0 and the frame counter 0 (the next ``step`` adds their keyframe).  In place, no host
    synchronisation."""
    B = int(state["frame"].shape[0])
    if mask.dtype != torch.bool or tuple(mask.shape) != (B,):
        raise ValueError(f"mask must be bool [{B}], got {mask.dtype} {list(mask.shape)}")
    m = mask.to(state["frame"].device)
    state["frame"].masked_fill_(m, 0)
    state["hist_len"].masked_fill_(m, 0)
    state["init_cnt"].masked_fill_(m, INIT_COUNT)
    state["use_motion_cnt"].masked_fill_(m, 0)


def _check_state(state: dict):
    for k in ("frame", "hist", "hist_len", "init_cnt", "use_motion_cnt", "kf"):
        if k not in state:
            raise ValueError(f"track state lacks {k!r}: make it with track.init_state")
    dev, B, cap = flow._check_kf(state["kf"])
    want = {"frame": (torch.int64, (B,)), "hist": (torch.float64, (B, HISTORY, 4, 4)), "hist_len": (torch.int32, (B,)),
            "init_cnt": (torch.int32, (B,)), "use_motion_cnt": (torch.int32, (B,))}
    for k, (dt, shape) in want.items():
        t = state[k]
        if t.dtype != dt or tuple(t.shape) != shape or t.device != dev or not t.is_contiguous():
            raise ValueError(f"state[{k!r}] must be a contiguous {dt} {list(shape)} tensor on {dev}, got {t.dtype} {list(t.shape)} on {t.device}")
    return dev, B, cap


def step(state: dict, res: dict, crops: torch.Tensor, K_crop: torch.Tensor) -> dict:
    """One frame of the demo's tracking branch (``inference_demo.py:253-299``) for B tracks, on the device.

    state    ``init_state``'s dict, updated in place (the keyframe in ``state["kf"]`` is replaced by a new dict)
    res      the frame's ``pnp.poses_from_matches`` / ``poses_from_matches_objects`` result for the B tracks, on the crops
    crops    the B crops the result was solved on, uint8 [B,S,S] or ``crop.crop_frames``' fp32 [B,1,S,S]
    K_crop   [B,3,3] or [3,3], the crops' intrinsics

    Per track: (1) the gate -- add_kf at the first frame, update_kf every 5th; (2) the keyframe becomes the frame's inlier pairs
    (``flow.keyframes_from_poses``) where add_kf or an accepted update_kf says so; (3) ``flow.flow_track`` from the keyframe
    into the crop, scored against the matcher pose; (4) track()'s choice of the pose; (5) flow_track's accepted keyframes,
    except for tracks at their first frame, where the demo does not call track().

    Returns a dict of device tensors: pose f64 [B,4,4] (the demo's pose_opt: the matcher pose at the first frame, track()'s
    pose after), branch int32 [B] (FLOW, MOTION, PRED, INIT or KEYFRAME), gate int32 [B] (GATE_NONE, GATE_ADD, GATE_ACCEPT or
    GATE_REJECT) and flow_track's outputs under ``flow`` (its ``kf`` is the one before the first-frame rows are restored)."""
    dev, B, cap = _check_state(state)
    pose_pred = res["pose_homo"]
    if pose_pred.dtype != torch.float64 or tuple(pose_pred.shape) != (B, 4, 4) or pose_pred.device != dev:
        raise ValueError(f"res['pose_homo'] must be f64 [{B}, 4, 4] on {dev}, got {pose_pred.dtype} {list(pose_pred.shape)} on {pose_pred.device}")
    n_pairs = res["inlier_mask"].numel()
    if n_pairs != B * cap:
        raise ValueError(f"the result has {n_pairs} pairs, the state's keyframes {B} x {cap}: every result must have {cap} pairs per frame")
    S = int(state["kf"]["image"].shape[-1])
    if crops.shape[0] != B or crops.shape[-1] != S or crops.shape[-2] != S:
        raise ValueError(f"crops must be {B} crops of {S} x {S}, got {list(crops.shape)}")
    pose_pred = pose_pred.contiguous()
    gate = torch.empty(B, dtype=torch.int32, device=dev)
    _lib.call(dev, "opb_track_gate", pose_pred, B, state["frame"], state["hist"], state["hist_len"], gate)
    new = flow.keyframes_from_poses(res, crops)
    take = (gate == GATE_ADD) | (gate == GATE_ACCEPT)
    kf = state["kf"]
    kf = {k: torch.where(take.view(-1, *([1] * (v.dim() - 1))), new[k], v) for k, v in kf.items()}
    first = gate == GATE_ADD
    ft = flow.flow_track(kf, crops, K_crop, pose_pred)
    pose = torch.empty(B, 4, 4, dtype=torch.float64, device=dev)
    branch = torch.empty(B, dtype=torch.int32, device=dev)
    _lib.call(dev, "opb_track_select", pose_pred, ft["pose_init_homo"].contiguous(), ft["kpt_dist"].contiguous(), B, state["frame"], state["hist"],
              state["hist_len"], state["init_cnt"], state["use_motion_cnt"], pose, branch)
    state["kf"] = {k: torch.where(first.view(-1, *([1] * (v.dim() - 1))), kf[k], v) for k, v in ft["kf"].items()}
    return {"pose": pose, "branch": branch, "gate": gate, "flow": ft}
