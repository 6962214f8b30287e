"""Generate the crop golden vectors by running the UNMODIFIED reference functions with this machine's OpenCV.

Run in the build container only (needs /root/reference and cv2):

    python tests/golden/make_crop.py

Imports ``get_image_crop_resize`` / ``get_K_crop_resize`` (reference ``src/utils/data_utils.py:233-272``) and ``reproj``
(``src/utils/vis_utils.py:209-236``) and runs the bodies of ``crop_img_by_bbox`` / ``previous_pose_detect``
(``local_feature_2D_detector.py:160-186``, ``:232-259``) on them.  Writes ``pnp_crop_cases.npz`` (the ``pnp_`` prefix keeps it out
of the matcher's forward cases, which tests/golden_util.py collects by file name).  The frames are not stored: both sides make
them with ``tests.crop_reference.synthetic_frame`` (integers only).  Data only: no reference source is copied.
"""
import os
import sys

import cv2
import numpy as np

sys.path.insert(0, "/root/reference")
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

for _m in ("matplotlib", "matplotlib.cm", "matplotlib.pyplot", "natsort"):    # vis_utils' plotting imports; reproj uses none
    try:
        __import__(_m)
    except ImportError:
        from unittest import mock
        sys.modules[_m] = mock.MagicMock()

from src.utils.data_utils import get_image_crop_resize, get_K_crop_resize  # noqa: E402
from src.utils.vis_utils import reproj  # noqa: E402
from tests.crop_reference import synthetic_frame  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "pnp_crop_cases.npz")
FRAMES = [(480, 640, 0), (96, 128, 1), (1440, 1920, 2)]            # h, w, seed

# (frame, [x0, y0, x1, y1], crop_size)
CASES = [
    (0, [100, 80, 180, 150], 64), (0, [301, 33, 372, 120], 64), (0, [10, 10, 110, 90], 64),          # inside: even, odd, even
    (0, [-30, 100, 50, 170], 64), (0, [200, -25, 290, 40], 64), (0, [600, 200, 680, 260], 64),       # crossing left, top, right
    (0, [300, 440, 370, 510], 64), (0, [-20, -20, 45, 50], 64), (0, [590, 430, 655, 497], 64),       # bottom, two corners
    (0, [700, 100, 760, 150], 64), (0, [-200, -100, -120, -40], 64), (0, [100, 480, 160, 530], 64),  # wholly outside
    (0, [320, 100, 321, 180], 64), (0, [100, 240, 190, 241], 64), (0, [50, 50, 51, 51], 64),         # one pixel wide / tall / both
    (0, [50, 300, 200, 330], 64), (0, [500, 50, 520, 200], 64), (0, [0, 0, 300, 200], 64),           # non-square, reducing
    (0, [200, 150, 330, 290], 512), (0, [100, 100, 164, 164], 8), (0, [40, 60, 296, 316], 256),      # the reference's size, 8, 1:1
    (0, [333, 222, 400, 301], 128), (0, [639, 479, 700, 520], 64),
    (1, [-20, -15, 150, 110], 64), (1, [-5, -40, 133, 136], 64), (1, [20, 20, 60, 50], 64),           # larger than the frame
    (1, [0, 0, 128, 96], 128), (1, [127, 95, 140, 101], 64),
    (2, [800, 600, 1100, 860], 512), (2, [1800, 1300, 2000, 1500], 64), (2, [5, 7, 262, 300], 128),
]


def crop_img_by_bbox(img, bbox, K, crop_size):
    """The body of the reference method on an image in memory, keeping the first stage too."""
    x0, y0, x1, y1 = bbox
    resize_shape = np.array([y1 - y0, x1 - x0])
    K_crop, _ = get_K_crop_resize(bbox, K, resize_shape)
    stage1, trans1 = get_image_crop_resize(img, bbox, resize_shape)
    bbox_new = np.array([0, 0, x1 - x0, y1 - y0])
    resize_shape = np.array([crop_size, crop_size])
    K_crop, _ = get_K_crop_resize(bbox_new, K_crop, resize_shape)
    stage2, trans2 = get_image_crop_resize(stage1, bbox_new, resize_shape)
    return stage1, stage2, trans1[:2], trans2[:2], K_crop


def scenes(rng):
    """(K, pose [3,4], corners [8,3]) with the object in view, partly left of / above the image, and across the camera plane."""
    out = []
    for i in range(14):
        half = rng.uniform(0.03, 0.12, 3)
        corners = np.array([[sx, sy, sz] for sx in (-1, 1) for sy in (-1, 1) for sz in (-1, 1)], np.float64) * half + rng.uniform(-0.02, 0.02, 3)
        q = rng.normal(size=4)
        q /= np.linalg.norm(q)
        w, x, y, z = q
        R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                      [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                      [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
        t = np.array([rng.uniform(-0.1, 0.1), rng.uniform(-0.08, 0.08), rng.uniform(0.4, 0.9)])
        if i in (4, 5):
            t[:2] = [-0.45, -0.30]                                   # negative image coordinates: truncation is not floor
        if i in (6, 7):
            t[2] = 0.02 * (i - 6)                                    # some corners behind the camera
        f = rng.uniform(1200, 1700)
        K = np.array([[f, 0, 960 + rng.uniform(-20, 20)], [0, f * rng.uniform(0.98, 1.02), 720 + rng.uniform(-20, 20)], [0, 0, 1]])
        out.append((K, np.concatenate([R, t[:, None]], axis=1), corners))
    return out


def main():
    print("cv2", cv2.__version__)
    rng = np.random.default_rng(20240)
    frames = [synthetic_frame(*f) for f in FRAMES]
    sc = scenes(rng)
    g = {"frames": np.array(FRAMES, np.int32), "sc_K": np.stack([s[0] for s in sc]), "sc_pose": np.stack([s[1] for s in sc]),
         "sc_corners": np.stack([s[2] for s in sc])}
    proj, boxes = [], []
    for i, (K, pose, corners) in enumerate(sc):
        pose_in = pose if i % 2 == 0 else np.concatenate([pose, [[0, 0, 0, 1.0]]], axis=0)
        p = reproj(K, pose_in, corners)                              # previous_pose_detect :246-249
        x0, y0 = np.min(p, axis=0)
        x1, y1 = np.max(p, axis=0)
        ext = np.array([x0, y0, x1, y1])
        assert np.all(np.abs(ext - np.rint(ext)) > 1e-6) and np.all(np.abs(ext) < 2 ** 31), (i, ext)
        proj.append(p)
        boxes.append(ext.astype(np.int32))
    g["sc_proj"], g["sc_box"] = np.stack(proj), np.stack(boxes)
    assert (g["sc_box"] < 0).any() and (np.trunc(g["sc_proj"].min(1)) != np.floor(g["sc_proj"].min(1))).any()

    # crops: the listed boxes with a per-case K, then previous_pose_detect's own box of one scene on the camera frame
    cases = [(f, np.array(b, np.int32), s, np.array([[500.0 + 3 * i, 0, 320.5 - i], [0, 498.0 + 2 * i, 240.25 + i], [0, 0, 1]]))
             for i, (f, b, s) in enumerate(CASES)]
    for i in (2,):
        cases.append((2, g["sc_box"][i], 64, g["sc_K"][i]))
    for i, (f, box, S, K) in enumerate(cases):
        s1, s2, T1, T2, K_crop = crop_img_by_bbox(frames[f], box, K, S)
        assert s1.shape == (box[3] - box[1], box[2] - box[0]) and s2.shape == (S, S) and s2.dtype == np.uint8
        g[f"stage1_{i}"], g[f"stage2_{i}"] = s1, s2
        for k, v in (("T1", T1), ("T2", T2), ("K_crop", K_crop)):
            g.setdefault(k, []).append(v)
    g["case_frame"] = np.array([c[0] for c in cases], np.int32)
    g["box"] = np.stack([c[1] for c in cases]).astype(np.int32)
    g["crop_size"] = np.array([c[2] for c in cases], np.int32)
    g["K"] = np.stack([c[3] for c in cases])
    for k in ("T1", "T2", "K_crop"):
        g[k] = np.stack(g[k])
    g["cv2_version"] = np.array(cv2.__version__)
    np.savez_compressed(OUT, **g)
    print(OUT, len(cases), "crops,", len(sc), "scenes,", os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
