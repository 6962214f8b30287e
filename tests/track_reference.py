"""numpy model of the tracker's flow-only state machine (csrc/track.cu, onepose_b200/track.py) on the same state layout.

It restates, from ``src/tracker/ba_tracker.py``: ``cm_degree_5_metric`` (:105-111) in ``pnp.pose_errors``' arithmetic (index
order, every operation rounded on its own), ``update_kf``'s gate (:128-145), ``add_kf``'s push of the first pose (:149),
``motion_prediction`` (:275-293, with its slip: rot_t is mat2euler of pose_list[-2]) and ``track()``'s choice with
``flow_track_only=True`` (:727-802).  ``mat2euler`` / ``euler2mat`` are ``transforms3d.euler``'s with the default axes 'sxyz',
restated from their formulas (the package is not a dependency).  Scalars go through Python floats and the ``math`` module, so
that nothing is fused.

State (numpy, one row per track): frame int64 [B], hist f64 [B,3,4,4] (oldest first), hist_len int32 [B], init_cnt int32 [B],
use_motion_cnt int32 [B].
"""
from __future__ import annotations

import math

import numpy as np

TRACK_INTERVAL = 5
UPDATE_CM = UPDATE_DEG = 10.0
MOTION_CM = MOTION_DEG = MOTION_PX = 10.0
MOTION_COUNT = 3
FLOW_CM = FLOW_DEG = 20.0
HISTORY = 3
EPS4 = 4.0 * np.finfo(np.float64).eps
GATE_NONE, GATE_ADD, GATE_ACCEPT, GATE_REJECT = 0, 1, 2, 3
FLOW, MOTION, PRED, INIT, KEYFRAME = 0, 1, 2, 3, 4


def cm_degree(a, b):
    """cm_degree_5_metric(a, b) -> (trans cm, rot deg) of two [3,4] / [4,4] poses, in pnp.pose_errors' order."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    s = 0.0
    for r in range(3):
        d = float(a[r, 3]) - float(b[r, 3])
        s = d * d if r == 0 else s + d * d
    cm = math.sqrt(s) * 100.0
    tr = 0.0
    for r in range(3):
        d = float(a[r, 0]) * float(b[r, 0]) + float(a[r, 1]) * float(b[r, 1]) + float(a[r, 2]) * float(b[r, 2])
        tr = d if r == 0 else tr + d
    tr = tr if tr <= 3.0 else 3.0
    x = (tr - 1.0) / 2.0
    deg = math.acos(x) * (180.0 / math.pi) if -1.0 <= x <= 1.0 else float("nan")
    return cm, deg


def mat2euler(M, axes="sxyz"):
    """transforms3d.euler.mat2euler for axes 'sxyz': (ai, aj, ak) of a rotation matrix (its top-left 3x3)."""
    if axes != "sxyz":
        raise NotImplementedError(axes)
    M = np.asarray(M, np.float64)
    m = [[float(M[i, j]) for j in range(3)] for i in range(3)]
    cy = math.sqrt(m[0][0] * m[0][0] + m[1][0] * m[1][0])
    if cy > EPS4:
        return math.atan2(m[2][1], m[2][2]), math.atan2(-m[2][0], cy), math.atan2(m[1][0], m[0][0])
    return math.atan2(-m[1][2], m[1][1]), math.atan2(-m[2][0], cy), 0.0


def euler2mat(ai, aj, ak, axes="sxyz"):
    """transforms3d.euler.euler2mat for axes 'sxyz': the 3x3 rotation of static x, then y, then z."""
    if axes != "sxyz":
        raise NotImplementedError(axes)
    ai, aj, ak = float(ai), float(aj), float(ak)
    si, sj, sk = math.sin(ai), math.sin(aj), math.sin(ak)
    ci, cj, ck = math.cos(ai), math.cos(aj), math.cos(ak)
    cc, cs, sc, ss = ci * ck, ci * sk, si * ck, si * sk
    return np.array([[cj * ck, sj * sc - cs, sj * cc + ss],
                     [cj * sk, sj * ss + cc, sj * cs - sc],
                     [-sj, cj * si, cj * ci]])


def motion_prediction(pose0, pose1, pose_t):
    """BATracker.motion_prediction on pose_list[-3:], slip included."""
    rot0, rot1, rot_t = mat2euler(pose0), mat2euler(pose1), mat2euler(pose1)
    a = [rot1[i] + ((rot1[i] - rot0[i]) + (rot_t[i] - rot1[i])) / 2.0 for i in range(3)]
    out = np.eye(4)
    out[:3, :3] = euler2mat(*a)
    for r in range(3):
        out[r, 3] = float(pose_t[r, 3]) + ((float(pose1[r, 3]) - float(pose0[r, 3])) + (float(pose_t[r, 3]) - float(pose1[r, 3]))) / 2.0
    return out


def init_state(B: int) -> dict:
    return {"frame": np.zeros(B, np.int64), "hist": np.zeros((B, HISTORY, 4, 4)), "hist_len": np.zeros(B, np.int32),
            "init_cnt": np.full(B, 3, np.int32), "use_motion_cnt": np.zeros(B, np.int32)}


def _first(state, b) -> bool:
    return state["frame"][b] <= 0 or state["hist_len"][b] <= 0


def _push(state, b, pose):
    n = int(min(max(state["hist_len"][b], 0), HISTORY))
    if n == HISTORY:
        state["hist"][b, :-1] = state["hist"][b, 1:].copy()
        n -= 1
    state["hist"][b, n] = pose
    state["hist_len"][b] = n + 1


def gate(state: dict, pose_pred) -> np.ndarray:
    """The gate outcome per track; pushes pose_pred at a track's first frame (add_kf).  In place."""
    B = len(state["frame"])
    out = np.zeros(B, np.int32)
    for b in range(B):
        if _first(state, b):
            state["hist_len"][b] = 0
            _push(state, b, pose_pred[b])
            out[b] = GATE_ADD
        elif state["frame"][b] % TRACK_INTERVAL == 0:
            cm, deg = cm_degree(pose_pred[b], state["hist"][b, min(state["hist_len"][b], HISTORY) - 1])
            out[b] = GATE_REJECT if (cm > UPDATE_CM or deg > UPDATE_DEG) else GATE_ACCEPT
        else:
            out[b] = GATE_NONE
    return out


def select(state: dict, pose_pred, pose_flow, kpt_dist):
    """track()'s steps 2-6 per track: (pose [B,4,4], branch [B]).  In place."""
    B = len(state["frame"])
    pose, branch = np.zeros((B, 4, 4)), np.zeros(B, np.int32)
    for b in range(B):
        n = int(min(state["hist_len"][b], HISTORY))
        first = _first(state, b)
        state["frame"][b] += 1
        if first:
            pose[b], branch[b] = pose_pred[b], KEYFRAME
            continue
        h = state["hist"][b]
        cm, deg = cm_degree(h[n - 1], pose_flow[b])
        umc = int(state["use_motion_cnt"][b])
        if ((cm > MOTION_CM or deg > MOTION_DEG) and umc < MOTION_COUNT) or kpt_dist[b] > MOTION_PX:
            flow = False
        else:
            flow = cm < FLOW_CM and deg < FLOW_DEG
        if flow:
            umc, p, code = 0, pose_flow[b], FLOW
        else:
            umc += 1
            p, code = (pose_pred[b], PRED) if n < HISTORY else (motion_prediction(h[0], h[1], h[2]), MOTION)
        state["use_motion_cnt"][b] = umc
        if state["init_cnt"][b] > 0:
            state["init_cnt"][b] -= 1
            p, code = pose_pred[b], INIT
        pose[b], branch[b] = p, code
        _push(state, b, p)
    return pose, branch
