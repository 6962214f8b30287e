"""Golden sequences of the tracker's flow-only tracking: the reference's unmodified ``BATracker`` driven through the live demo's
tracking branch (``inference_demo.py:253-299``, track_interval 5, ``track(frame_dict, auto_mode=False)`` with
``flow_track_only=True``) on rendered crops of non-planar blob objects (tests/track_scenes.py).  The crops are not stored: each frame keeps its
planted pose, the object's seed and the CRC-32 of its crop, and the tests render the crops again and check the CRCs.

    python tests/golden/make_track.py     # writes tests/golden/pnp_track_cases.npz (needs the reference tree and cv2 4.13)

What is stubbed, and why:
- the tracker's module imports DeepLM's solver, which is not part of the reference: the import is a mock, as make_flow.py does;
- ``__init__`` is the real one, with ``load_extractor_model`` (a SuperPoint checkpoint) and ``MovieWriter`` (video output)
  patched out;
- ``motion_prediction`` imports ``transforms3d.euler``, which is not installed: it is given ``mat2euler`` / ``euler2mat`` of
  ``tests/track_reference.py``.  So this golden pins the reference's logic -- its gate, counters, slip and choice of pose --
  not the Euler-angle code, which tests/test_track_reference_cpu.py pins to scipy.
- ``flow_track`` and ``motion_prediction`` are wrapped on the instance to record what they return (the branch a frame took);
  the wrappers call the class's own methods unchanged.

Every frame's matcher result is ``ransac_PnP(K_crop, mkpts2d, mkpts3d, scale=1000)`` (eval_utils.py:18-42, as the demo) on
planted matches: each visible 3D point projected with the frame's matcher pose plus 0.2 px of noise.  The generator asserts
that every decision (update_kf's gate, track()'s choice, flow_track's accept) stays the same when each distance it reads
moves by up to 0.5 cm / 0.5 deg / 0.5 px, so that the gap between cv2's EPnP and the device's cannot flip it.
"""
from __future__ import annotations

import itertools
import os
import sys
import types
from unittest import mock

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, "/root/reference")
sys.path.insert(0, ROOT)
for _m in ("DeepLM", "DeepLM.TorchLM", "DeepLM.TorchLM.solver"):
    sys.modules[_m] = mock.MagicMock()

from tests import track_reference as TR  # noqa: E402
from tests.flow_scenes import blob_object, pose_at, project  # noqa: E402
from tests.track_scenes import K, N, SCENES, crc, crop, truth as planted  # noqa: E402

_t3d = types.ModuleType("transforms3d")
_t3d.euler = types.ModuleType("transforms3d.euler")
_t3d.euler.mat2euler, _t3d.euler.euler2mat = TR.mat2euler, TR.euler2mat
sys.modules["transforms3d"], sys.modules["transforms3d.euler"] = _t3d, _t3d.euler

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "pnp_track_cases.npz")
MARGIN = 0.5


def _robust(decide, values, what):
    """decide(*values) is unchanged when each value moves by up to MARGIN (every combination of -MARGIN, 0, +MARGIN)."""
    want = decide(*values)
    for d in itertools.product((-MARGIN, 0.0, MARGIN), repeat=len(values)):
        assert decide(*(v + e for v, e in zip(values, d))) == want, f"{what}: {values} is within {MARGIN} of a threshold"


def run_scene(name, frames, seed, offsets, hidden, sparse):
    from src.tracker import ba_tracker
    from src.tracker.ba_tracker import BATracker
    from src.utils.eval_utils import ransac_PnP

    X = blob_object(seed, N)[0]
    rs = np.random.RandomState(seed + 100)
    with mock.patch.object(BATracker, "load_extractor_model", return_value=None), mock.patch.object(ba_tracker, "MovieWriter"):
        tracker = BATracker(mock.MagicMock())
    rec = {}

    def flow_track(frame_dict, kf_info):
        rec["flow"] = BATracker.flow_track(tracker, frame_dict, kf_info)
        rec["accept"] = tracker.last_kf_info is frame_dict
        rec["flow_dist"] = tracker.cm_degree_5_metric(rec["flow"][0], frame_dict["pose_gt"])
        return rec["flow"]

    def motion_prediction():
        rec["motion"] = BATracker.motion_prediction(tracker)
        return rec["motion"]

    tracker.flow_track, tracker.motion_prediction = flow_track, motion_prediction
    out = {k: [] for k in ("crc", "turned", "m2d", "m3d", "n", "mask", "pose_pred", "truth", "gate", "branch", "pose", "umc", "init_cnt", "accept",
                           "flow_pose", "kpt_dist", "motion")}
    for i in range(frames):
        truth = planted(seed, i)
        dw, dt = offsets.get(i, ([0.0] * 3, [0.0] * 3))
        seen = pose_at(truth, dw, dt)
        image = crop(seed, truth, i in hidden)
        n = 3 if i in sparse else N
        mk2 = (project(K, seen, X[:n]) + 0.2 * rs.randn(n, 2)).astype(np.float32)
        mk3 = X[:n].astype(np.float32)
        _, pose_pred_homo, inliers = ransac_PnP(K, mk2, mk3, scale=1000)
        inl = np.asarray(inliers, np.int64).reshape(-1)
        assert np.all(np.diff(inl) > 0), "cv2 returns the inliers in pair order"
        frame_dict = {"im_path": image, "pose_pred": pose_pred_homo, "pose_gt": pose_pred_homo, "K": K, "K_crop": K}
        gate = TR.GATE_NONE
        if i % 5 == 0:                                    # inference_demo.py:264-292
            kf_dict = {"im_path": image, "mkpts2d": mk2[inliers.flatten()], "mkpts3d": mk3[inliers.flatten()], "pose_pred": pose_pred_homo,
                       "pose_gt": pose_pred_homo, "K": K}
            if tracker.last_kf_info is not None:
                _robust(lambda t, r: t > TR.UPDATE_CM or r > TR.UPDATE_DEG, tracker.cm_degree_5_metric(pose_pred_homo, tracker.pose_list[-1]),
                        f"{name}[{i}] update_kf")
            accepted = tracker.update_kf(kf_dict)
            gate = TR.GATE_ADD if i == 0 else (TR.GATE_ACCEPT if accepted else TR.GATE_REJECT)
        rec.clear()
        if i == 0:
            tracker.add_kf({**kf_dict, "kpt_pred": {"keypoints": mk2, "descriptors": np.zeros((4, n), np.float32)},
                            "valid_query_id": np.arange(len(inl)), "kpt3d_ids": inl})
            pose_opt, branch, init_before = pose_pred_homo, TR.KEYFRAME, tracker.init_cnt
        else:
            last = tracker.pose_list[-1]
            init_before, umc_before = tracker.init_cnt, tracker.use_motion_cnt
            _, pose_opt, _ = tracker.track(frame_dict, auto_mode=False, flow_track_only=True)
            pose_ftk, kpt_dist = rec["flow"]
            tf, rf = tracker.cm_degree_5_metric(last, pose_ftk)
            _robust(lambda t, r, k: (((t > TR.MOTION_CM or r > TR.MOTION_DEG) and umc_before < TR.MOTION_COUNT) or k > TR.MOTION_PX,
                                     t < TR.FLOW_CM and r < TR.FLOW_DEG), (tf, rf, kpt_dist), f"{name}[{i}] track")
            _robust(lambda t, r, k: t <= 7 and r <= 7 and k < 10, (*rec["flow_dist"], kpt_dist), f"{name}[{i}] flow_track accept")
            if tracker.init_cnt < init_before:
                branch = TR.INIT
            elif pose_opt is pose_ftk:
                branch = TR.FLOW
            elif "motion" in rec and pose_opt is rec["motion"]:
                branch = TR.MOTION
            else:
                assert pose_opt is pose_pred_homo
                branch = TR.PRED
            out["flow_pose"].append(pose_ftk)
            out["kpt_dist"].append(kpt_dist)
        if i == 0:
            out["flow_pose"].append(np.eye(4))
            out["kpt_dist"].append(np.nan)
        m2, m3, mask = np.zeros((N, 2), np.float32), np.zeros((N, 3), np.float32), np.zeros(N, bool)
        m2[:n], m3[:n] = mk2, mk3
        mask[inl] = True
        for k, v in (("crc", crc(image)), ("turned", i in hidden), ("m2d", m2), ("m3d", m3), ("n", n), ("mask", mask), ("pose_pred", pose_pred_homo),
                     ("truth", np.concatenate([truth, [[0, 0, 0, 1.0]]])), ("gate", gate), ("branch", branch), ("pose", pose_opt),
                     ("umc", tracker.use_motion_cnt), ("init_cnt", tracker.init_cnt), ("accept", bool(rec.get("accept", False))),
                     ("motion", rec.get("motion", np.full((4, 4), np.nan)))):
            out[k].append(v)
    return {k: np.array(v) for k, v in out.items()}


def main():
    out, names = {}, []
    for s, (name, frames, seed, offsets, hidden, sparse) in enumerate(SCENES):
        r = run_scene(name, frames, seed, offsets, hidden, sparse)
        out.update({f"s{s}_{k}": v for k, v in r.items()})
        out[f"s{s}_seed"] = np.array(seed)
        names.append(name)
        print(name, "branch", "".join("FMPIK"[c] for c in r["branch"]), "gate", "".join(".KAR"[g] for g in r["gate"]),
              "umc", "".join(str(u) for u in r["umc"]), "accept", "".join("a" if a else "." for a in r["accept"]))
    out.update({"names": np.array(names), "K": K, "cap": np.array(N)})
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
