"""Generate the detection golden vectors by running the UNMODIFIED reference detector with this machine's OpenCV.

Run in the build container only (needs /root/reference, cv2 and torch; no GPU):

    python tests/golden/make_detect.py

Imports ``LocalFeatureObjectDetector`` (reference ``src/local_feature_2D_detector/local_feature_2D_detector.py``) and runs its
own ``match_worker`` / ``detect_by_matching`` (the per-view ``cv2.estimateAffinePartial2D``, the box and the choice) and
``crop_img_by_bbox`` on planted scenes.  The COLMAP model is replaced by setting ``db_dict`` directly, the matcher by a stub that
returns seeded ``matches0`` per view, and the module's ``pack_match_data`` (which moves tensors to a GPU) by one that hands the
view to the stub.  Writes ``pnp_detect_cases.npz`` (the ``pnp_`` prefix keeps it out of the matcher's forward cases, which
tests/golden_util.py collects by file name).  Frames are not stored: both sides make them with
``tests.crop_reference.synthetic_frame``.  Data only: no reference source is copied.
"""
import os
import sys
import tempfile

import cv2
import numpy as np
import torch

sys.path.insert(0, "/root/reference")
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

for _m in ("matplotlib", "matplotlib.cm", "matplotlib.pyplot", "natsort"):    # vis_utils' plotting imports; detection uses none
    try:
        __import__(_m)
    except ImportError:
        from unittest import mock
        sys.modules[_m] = mock.MagicMock()

import src.local_feature_2D_detector.local_feature_2D_detector as lfd  # noqa: E402
from tests.crop_reference import synthetic_frame  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "pnp_detect_cases.npz")


def _pack_match_data(db, query, db_size, query_size):
    return {"db": db}


class StubMatcher:
    """Returns the view's seeded matches0, as the reference reads it: match_pred['matches0'][0]."""

    def __call__(self, data):
        m = data["db"]["matches0_stub"]
        return {"matches0": torch.from_numpy(m)[None], "matching_scores0": torch.ones(1, len(m))}


def similarity(rng, view_hw, frame_hw):
    """A 2x3 similarity that puts the view's image well inside the frame."""
    h, w = view_hw
    H, W = frame_hw
    s = rng.uniform(0.25, 0.6) * min(H / h, W / w)
    a = rng.uniform(-0.6, 0.6)
    R = s * np.array([[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]])
    c = R @ np.array([w / 2, h / 2])
    t = np.array([W / 2, H / 2]) - c + rng.uniform(-0.15, 0.15, 2) * np.array([W, H])
    return np.concatenate([R, t[:, None]], axis=1)


def scene(rng, frame_hw, sizes, counts, queries):
    """Reference views (integer key points, as SuperPoint's are) and per query, per view, (matches, inlier fraction).  Inlier
    matches are the view's key point under the view's planted similarity plus 0.5 px noise; outliers land anywhere in the
    frame.  The query's key points are shuffled and padded with unmatched ones."""
    H, W = frame_hw
    views = [np.stack([rng.integers(0, w, n), rng.integers(0, h, n)], axis=1).astype(np.float32) for (h, w), n in zip(sizes, counts)]
    out = []
    for spec in queries:
        pts, m0 = [], []
        for v, (kp, (k, f)) in enumerate(zip(views, spec)):
            m = np.full(len(kp), -1, np.int64)
            idx = np.sort(rng.choice(len(kp), size=k, replace=False))
            S = similarity(rng, sizes[v], frame_hw)
            n_in = int(round(k * f))
            for j, i in enumerate(rng.permutation(idx)):
                if j < n_in:
                    p = S @ np.array([kp[i, 0], kp[i, 1], 1.0]) + rng.normal(0, 0.5, 2)
                else:
                    p = rng.uniform([0, 0], [W, H])
                m[i] = len(pts)
                pts.append(np.round(p))
            m0.append(m)
        n_extra = int(rng.integers(0, 60))
        pts += [np.round(rng.uniform([0, 0], [W, H])) for _ in range(n_extra)]
        perm = rng.permutation(len(pts)) if pts else np.zeros(0, np.int64)
        inv = np.empty_like(perm)
        inv[perm] = np.arange(len(perm))
        q = np.array(pts, np.float32).reshape(-1, 2)[perm]
        m0 = [np.where(m >= 0, inv[np.maximum(m, 0)] if len(inv) else -1, -1) for m in m0]
        out.append((q, m0))
    return views, out


def main():
    print("cv2", cv2.__version__)
    lfd.pack_match_data = _pack_match_data
    det = object.__new__(lfd.LocalFeatureObjectDetector)
    det.matcher = StubMatcher()
    det.output_results = False
    rng = np.random.default_rng(20261016)
    tmp = tempfile.mkdtemp()
    R15 = [(480, 640), (640, 480), (512, 512), (360, 640), (480, 360)] * 3
    scenes = [
        # frame (h, w, seed), view sizes, key points per view, queries: per view (matches, inlier fraction)
        ((480, 640, 0), R15, [int(v) for v in rng.integers(80, 700, 15)], [
            [(60, 0.7)] + [(int(rng.integers(0, 40)), 0.5) for _ in range(14)],                          # view 0 wins
            [(int(rng.integers(0, 40)), 0.5) for _ in range(9)] + [(300, 0.5)] + [(20, 0.3)] * 5,         # view 9 wins
            [(5, 1.0)] * 7 + [(4, 1.0)] * 8,                                                             # every view below 6
            [(3, 1.0)] * 4 + [(6, 1.0)] + [(5, 1.0)] * 10,                                               # exactly 6 matches
            [(10, 0.8), (40, 0.9), (25, 0.5), (40, 0.75)] + [(39, 0.2)] * 11,                             # a tie: view 1 over 3
            [(50, 0.75)] + [(0, 0.0)] * 13 + [(51, 0.1)],                                                 # the last view, 90 % out
        ]),
        ((640, 360, 1), [(480, 640), (300, 200), (640, 480), (128, 96)], [400, 150, 500, 60], [
            [(5, 1.0), (2, 1.0), (0, 0.0), (5, 1.0)],                                                     # portrait, [0, 0, H, W]
            [(30, 0.9), (120, 0.6), (200, 0.75), (6, 1.0)],
            [(0, 0.0), (0, 0.0), (0, 0.0), (60, 0.5)],
        ]),
        ((1440, 1920, 2), R15, [int(v) for v in rng.integers(1000, 1400, 15)], [
            [(int(rng.integers(20, 300)), 0.5) for _ in range(3)] + [(1000, 0.1)] + [(int(rng.integers(20, 300)), 0.4) for _ in range(11)],
            [(int(rng.integers(50, 400)), 0.3) for _ in range(14)] + [(999, 0.5)],
            [(600, 0.25)] * 15,                                                                           # all tie: view 0
        ]),
    ]
    g = {"cv2_version": np.array(cv2.__version__), "n_scenes": np.array(len(scenes))}
    for s, (frame, sizes, counts, queries) in enumerate(scenes):
        H, W, seed = frame
        img = synthetic_frame(H, W, seed)
        path = os.path.join(tmp, f"frame{s}.png")
        cv2.imwrite(path, img)
        assert np.array_equal(cv2.imread(path, cv2.IMREAD_GRAYSCALE), img)
        K = np.array([[900.0 + 10 * s, 0, W / 2 + 0.5], [0, 905.0, H / 2 - 0.25], [0, 0, 1]])
        views, qs = scene(rng, (H, W), sizes, counts, queries)
        cap = max(len(v) for v in views)
        g[f"s{s}_frame"] = np.array(frame, np.int32)
        g[f"s{s}_K"] = K
        g[f"s{s}_ref_sizes"] = np.array(sizes, np.int32)
        g[f"s{s}_ref_counts"] = np.array([len(v) for v in views], np.int32)
        g[f"s{s}_ref_keypoints"] = np.stack([np.pad(v, ((0, cap - len(v)), (0, 0))) for v in views])
        g[f"s{s}_n_queries"] = np.array(len(qs))
        for k, (q, m0) in enumerate(qs):
            det.db_dict = {}
            for v, kp in enumerate(views):
                det.db_dict[1 + 7 * v] = {"keypoints": kp, "scores": np.ones(len(kp), np.float32),
                                          "descriptors": np.zeros((256, len(kp)), np.float32), "size": np.array(sizes[v]),
                                          "matches0_stub": m0[v]}
            query = {"keypoints": q, "scores": np.ones(len(q), np.float32), "descriptors": np.zeros((256, len(q)), np.float32),
                     "size": np.array(img.shape[-2:])}
            per_view = det.match_worker(query)
            bbox = det.detect_by_matching(query)
            n_m = [int((m >= 0).sum()) for m in m0]
            key = [n if n >= 6 else 0 for n in n_m]
            win = int(np.argmax(key)) if max(key) > 0 else 0
            assert np.array_equal(per_view[1 + 7 * win]["bbox"], bbox)
            affine = np.zeros((2, 3))
            if max(key) > 0:
                valid = m0[win] > -1
                affine, _ = cv2.estimateAffinePartial2D(views[win][valid], q[m0[win][valid]], ransacReprojThreshold=6)
            crop_size = 512 if k == 0 else 128
            image_crop, K_crop = det.crop_img_by_bbox(path, bbox, K, crop_size=crop_size)
            p = f"s{s}_q{k}_"
            g[p + "keypoints"] = q
            g[p + "matches0"] = np.stack([np.pad(m, (0, cap - len(m)), constant_values=-1) for m in m0])
            g[p + "bbox"] = np.asarray(bbox).astype(np.int32)
            g[p + "view_bbox"] = np.stack([np.asarray(per_view[1 + 7 * v]["bbox"]).astype(np.int32) for v in range(len(views))])
            g[p + "view"] = np.array(win, np.int32)
            g[p + "n_matches"] = np.array(n_m[win], np.int32)
            g[p + "affine"] = affine
            g[p + "crop_size"] = np.array(crop_size, np.int32)
            g[p + "image_crop"] = image_crop
            g[p + "K_crop"] = K_crop
            print(f"scene {s} query {k}: view {win}, {n_m[win]} matches, bbox {np.asarray(bbox).tolist()}")
    np.savez_compressed(OUT, **g)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
