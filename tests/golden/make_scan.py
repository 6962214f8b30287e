"""Generate the annotated-scan golden vectors with the reference model of parse_scanned_data.py (tests/scan_reference.py).

    python tests/golden/make_scan.py

Writes ``pnp_scan_cases.npz`` (the ``pnp_`` prefix keeps it out of the matcher's forward cases, which tests/golden_util.py
collects by file name): the text of a synthetic ``Frames.txt``, ``Box.txt`` and ``ARposes.txt`` -- comment lines, blank lines,
non-unit quaternions and rows past each of the four skip bounds included -- and what data_process_anno and parse_video make of
them.  The video frames are not stored: both sides make frame f with ``scan_reference.colour_frame(H, W, f)`` (integers only).

Every row's camera is planted: a seeded rotation, a target pixel for the object's centre and a depth, the position solved so
that the centre projects there.  A row is drawn again until every projected corner coordinate lies at least 1e-6 from an
integer and from the skip bounds, so that neither the truncation nor the skip rule depends on the last bits of an inverse that
LAPACK and the device compute differently.
"""
import os
import sys

import numpy as np
from scipy.spatial.transform import Rotation

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

from tests import scan_reference as sr  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "pnp_scan_cases.npz")
H, W, S = 480, 640, 512
MARGIN = 1e-6


def _safe(v):
    v = np.asarray(v).reshape(-1)
    near_int = np.abs(v - np.rint(v)) < MARGIN
    near_bound = (np.abs(v + 1000) < MARGIN) | (np.abs(v - 3000) < MARGIN)
    return bool(np.all(np.isfinite(v)) and not near_int.any() and not near_bound.any())


def main():
    rng = np.random.default_rng(20261018)
    # Frames.txt: timestamp, frame index, fx, fy, cx, cy per frame; the reference averages columns 2-5
    frames_lines = ["# Frames: timestamp, frame index, fx, fy, cx, cy\n"]
    for i in range(12):
        fx, fy = 512.3 + rng.uniform(-0.01, 0.01), 511.7 + rng.uniform(-0.01, 0.01)
        frames_lines.append(f"{0.033 * i!r},{i},{fx!r},{fy!r},{319.61 + rng.uniform(-0.01, 0.01)!r},{240.27 + rng.uniform(-0.01, 0.01)!r}\n")
    fx, fy, cx, cy = sr.intrinsics(frames_lines)
    K = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]])

    centre = rng.uniform(-0.5, 0.5, 3)
    extent = rng.uniform(0.08, 0.2, 3)
    q_box = Rotation.random(random_state=7).as_quat()                 # x, y, z, w
    box_lines = ["# position, extent, quaternion\n",
                 ",".join(repr(float(v)) for v in list(centre) + list(extent) + [q_box[3], *q_box[:3]]) + "\n"]
    bbox3d, bbox_homo = sr.get_bbox3d(box_lines)
    T_ow = sr.parse_box(box_lines)
    K_homo = np.concatenate([K, np.zeros((3, 1))], axis=1)

    # (target pixel of the centre, depth, quaternion scale): in-frame boxes, boxes crossing an edge, and rows past each bound
    kinds = ["in"] * 18 + ["edge"] * 6 + ["x0", "y0", "x1", "y1"] * 2
    rng.shuffle(kinds)
    kinds = ["in"] + list(kinds)
    arposes_lines = ["# timestamp, position, quaternion (w, x, y, z)\n"]
    for r, kind in enumerate(kinds):
        while True:
            z = rng.uniform(0.45, 1.2)
            if kind == "in":
                u, v = rng.uniform(200, 440), rng.uniform(150, 330)
            elif kind == "edge":
                u, v = rng.choice([rng.uniform(-40, 40), rng.uniform(600, 680)]), rng.uniform(-40, 520)
            else:
                far = rng.uniform(1300, 2500)
                u, v = {"x0": (-far, 240), "y0": (320, -far), "x1": (3000 + far, 240), "y1": (320, 3000 + far)}[kind]
                z = rng.uniform(0.9, 1.2)
            R_cv = Rotation.from_rotvec(rng.normal(0, 0.6, 3)).as_matrix()
            p = T_ow[:3, 3] - R_cv @ (z * np.linalg.solve(K, [u, v, 1.0]))
            q = Rotation.from_matrix(R_cv @ sr.FLIP).as_quat()
            q = np.array([q[3], *q[:3]]) * (rng.uniform(0.5, 2.0) if r % 3 == 1 else 1.0) * (-1 if r % 5 == 2 else 1)
            row = [0.0333 * r, *p, *q]
            T_cw = sr.compose(p, sr.quat2mat(q) @ sr.FLIP, np.ones(3))
            proj = sr.reproj(K_homo, np.linalg.inv(T_cw) @ T_ow, bbox_homo.T)
            if not _safe(proj) or sr.skipped(proj) != (kind in ("x0", "y0", "x1", "y1")):
                continue
            if kind != "in" and kind != "edge":          # past one bound only
                x0, y0 = proj.min(0)
                x1, y1 = proj.max(0)
                if [x0 < -1000, y0 < -1000, x1 > 3000, y1 > 3000] != [kind == k for k in ("x0", "y0", "x1", "y1")]:
                    continue
            else:
                b = proj.astype(int)
                if not (b.max(0) - b.min(0) > 1).all():
                    continue
            break
        arposes_lines.append(",".join(repr(float(v)) for v in row) + "\n")
        if r == 5:
            arposes_lines.append("\n")                    # a blank line: skipped
        if r == 11:
            arposes_lines.append("# a comment between rows\n")

    saved, keep = sr.process_poses(K, box_lines, arposes_lines)
    count = len(saved)
    F = count + 3                                         # frames past the kept count get nothing
    frames = [sr.colour_frame(H, W, f) for f in range(F)]
    res = sr.parse_video(frames, saved, K, bbox_homo, S)
    assert all(r is not None for r in res[:count]) and all(r is None for r in res[count:])
    out = {
        "frames_txt": np.array("".join(frames_lines)), "box_txt": np.array("".join(box_lines)), "arposes_txt": np.array("".join(arposes_lines)),
        "frame_hw": np.array([H, W]), "crop_size": np.array(S), "n_frames": np.array(F),
        "K": K, "bbox3d": bbox3d, "T_ow": T_ow, "keep": keep, "count": np.array(count),
        "pose": np.stack([saved[i][0] for i in range(count)]), "proj": np.stack([saved[i][1] for i in range(count)]),
        "row": np.array([saved[i][2] for i in range(count)], np.int32),
        "box": np.stack([r["box"] for r in res[:count]]).astype(np.int32),
        "K_crop": np.stack([r["K_crop"] for r in res[:count]]), "M": np.stack([r["M"] for r in res[:count]]),
        "box_crop": np.stack([r["box_crop"] for r in res[:count]]),
    }
    np.savez_compressed(OUT, **out)
    print(OUT, "rows", len(keep), "kept", count, "frames", F)


if __name__ == "__main__":
    main()
