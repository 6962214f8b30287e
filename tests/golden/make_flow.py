"""Golden cases of the tracker's flow step: cv2.calcOpticalFlowPyrLK on seeded scenes and the reference's unmodified
``BATracker.flow_track`` / ``kpt_flow_track`` (src/tracker/ba_tracker.py) on seeded crops of a non-planar object of Gaussian blobs (tests/flow_scenes.py).

    python tests/golden/make_flow.py      # writes tests/golden/pnp_flow_cases.npz (needs the reference tree and cv2 4.13)

The tracker's module imports DeepLM's solver (not part of the reference) and builds a SuperPoint in __init__: the import is
stubbed and the instance made with ``__new__``; its MovieWriter is replaced by one that drops the frames.
"""
from __future__ import annotations

import os
import sys
from unittest import mock

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, "/root/reference")
sys.path.insert(0, ROOT)
for _m in ("DeepLM", "DeepLM.TorchLM", "DeepLM.TorchLM.solver"):
    sys.modules[_m] = mock.MagicMock()

import cv2  # noqa: E402

from onepose_b200 import synthetic  # noqa: E402

from tests.flow_scenes import blob_object, lk_scene, pose_at, project, render_blobs, rodrigues  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "pnp_flow_cases.npz")
S = 192                 # crop side of the flow_track cases

# ---- LK scenes: (seed, h, w, win, max_level, criteria, motion) ----
LK_SCENES = [
    (1, 96, 128, (15, 15), 2, (3, 10, 0.03), "affine"),
    (2, 120, 160, (21, 21), 3, (3, 30, 0.01), "perspective"),
    (3, 80, 100, (7, 7), 4, (1, 5, 0.0), "affine"),
    (4, 64, 64, (31, 31), 1, (2, 0, 0.1), "perspective"),
    (5, 100, 90, (3, 3), 0, (3, 20, 0.01), "affine"),
    (6, 96, 128, (9, 13), 2, (3, 10, 0.03), "large"),
]


def main():
    out = {}
    for i, (seed, h, w, win, lev, crit, motion) in enumerate(LK_SCENES):
        img, nxt, pts = lk_scene(seed, h, w, motion)
        p, st, err = cv2.calcOpticalFlowPyrLK(img, nxt, pts[:, None], None, winSize=win, maxLevel=lev, criteria=crit)
        n_lev, pyr_p = cv2.buildOpticalFlowPyramid(img, win, lev, withDerivatives=True)
        _, pyr_n = cv2.buildOpticalFlowPyramid(nxt, win, lev, withDerivatives=False)
        out.update({f"lk{i}_prev": img, f"lk{i}_next": nxt, f"lk{i}_pts": pts, f"lk{i}_params": np.array([win[0], win[1], lev, *crit], np.float64),
                    f"lk{i}_next_pts": p[:, 0], f"lk{i}_status": st[:, 0], f"lk{i}_err": err[:, 0], f"lk{i}_levels": np.array(n_lev)})
        for level in range(n_lev + 1):                    # level 0 of the images is the scene itself
            out[f"lk{i}_pyr_der{level}"] = pyr_p[2 * level + 1]
            if level:
                out[f"lk{i}_pyr_prev{level}"] = pyr_p[2 * level]
                out[f"lk{i}_pyr_next{level}"] = pyr_n[level]

    from src.tracker.ba_tracker import BATracker
    from src.tracker.tracking_utils import Timer
    from src.utils.eval_utils import ransac_PnP

    X, amp = blob_object(11, 80)             # a non-planar object: 80 blobs in a 12 cm cube
    K = np.array([[450.0, 0, S / 2], [0, 450.0, S / 2], [0, 0, 1]])
    pose_kf = np.concatenate([rodrigues([0.15, -0.1, 0.05]), [[0.0], [0.0], [0.45]]], 1)
    x_kf = project(K, pose_kf, X).astype(np.float32)
    im_kf = render_blobs(K, pose_kf, X, amp, S)

    cases = [  # (name, query pose, pose_ref, keyframe rows)
        ("small", pose_at(pose_kf, [0.01, -0.008, 0.006], [0.003, -0.002, 0.004]), None, slice(None)),
        ("small2", pose_at(pose_kf, [-0.012, 0.01, -0.004], [-0.004, 0.003, -0.006]), None, slice(0, 50)),
        ("wrong_ref", pose_at(pose_kf, [0.01, -0.008, 0.006], [0.003, -0.002, 0.004]), pose_at(pose_kf, [0.2, 0.0, 0.0], [0.1, 0.0, 0.0]),
         slice(None)),
        ("large", pose_at(pose_kf, [0.05, 0.25, 0.1], [0.05, -0.04, 0.02]), None, slice(None)),
        ("three", pose_at(pose_kf, [0.01, -0.008, 0.006], [0.003, -0.002, 0.004]), None, slice(0, 3)),
        ("none", pose_at(pose_kf, [0.01, -0.008, 0.006], [0.003, -0.002, 0.004]), None, "outside"),
    ]
    cap = 96
    names = []
    for c, (name, pose_q, pose_ref, rows) in enumerate(cases):
        pose_ref = pose_q if pose_ref is None else pose_ref
        pose_ref_h = np.concatenate([pose_ref, [[0, 0, 0, 1.0]]], 0)
        im_q = render_blobs(K, pose_q, X, amp, S)
        if isinstance(rows, str):
            kp2, kp3 = np.full((10, 2), -500.0, np.float32), X[:10]
        else:
            kp2, kp3 = x_kf[rows], X[rows]
        tr = BATracker.__new__(BATracker)
        tr.tm = Timer()
        tr.mw = mock.MagicMock()
        tr.out = ""
        tr.last_kf_info = None
        kf_info = {"im_path": im_kf, "mkpts2d": kp2, "mkpts3d": kp3}
        frame = {"im_path": im_q, "K_crop": K, "pose_gt": pose_ref_h}
        pose_h, kpt_dist = tr.flow_track(frame, kf_info)
        trans, rot = tr.cm_degree_5_metric(pose_h, pose_ref_h)
        tracked, valid = tr.kpt_flow_track(im_kf, im_q, kp2)                # the same call flow_track made
        _, _, inliers = ransac_PnP(K, tracked[valid], kp3[valid])           # and its PnP, for the inlier count
        accept = tr.last_kf_info is not None
        p2 = np.zeros((cap, 2), np.float32)
        p3 = np.zeros((cap, 3), np.float32)
        p2[:len(kp2)], p3[:len(kp3)] = kp2, kp3
        status = np.zeros(len(kp2), np.uint8)
        status[valid] = 1
        out.update({f"ft{c}_query": im_q, f"ft{c}_pts2d": p2, f"ft{c}_pts3d": p3, f"ft{c}_count": np.array(len(kp2)),
                    f"ft{c}_pose_ref": pose_ref_h, f"ft{c}_pose_truth": pose_q, f"ft{c}_pose": pose_h, f"ft{c}_kpt_dist": np.array(kpt_dist),
                    f"ft{c}_trans": np.array(trans), f"ft{c}_rot": np.array(rot), f"ft{c}_n_tracked": np.array(len(valid[0])),
                    f"ft{c}_tracked": tracked.astype(np.float32), f"ft{c}_status": status, f"ft{c}_n_inliers": np.array(len(inliers)),
                    f"ft{c}_accept": np.array(accept)})
        if accept:
            out[f"ft{c}_kf_pts2d"] = np.asarray(tr.last_kf_info["mkpts2d"], np.float32)
            out[f"ft{c}_kf_pts3d"] = np.asarray(tr.last_kf_info["mkpts3d"], np.float32)
        names.append(name)
        print(name, "tracked", len(valid[0]), "inliers", len(inliers), "kpt_dist", kpt_dist, "trans", trans, "rot", rot, "accept", accept)
    out.update({"ft_names": np.array(names), "ft_K": K, "ft_kf_image": im_kf, "ft_cap": np.array(cap)})
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
