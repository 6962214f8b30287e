"""Generate the fixtures of the pose solvers' domain test (tests/test_pose_domain_gpu.py) on a machine with OpenCV:

    python tests/golden/make_pose_domain.py

Writes ``pnp_domain_cases.npz``: cv2.solvePnPRansac(..., flags=SOLVEPNP_EPNP) on noise-free scenes with outliers at every
threshold the confidence mode is tested at.  Per case ``c{i}_K``, ``c{i}_uv``, ``c{i}_P`` (millimetres), ``c{i}_thr``,
``c{i}_conf``, ``c{i}_iters``, cv2's ``c{i}_ok``, ``c{i}_cv`` (pose [3,4]; the identity when it fails) and ``c{i}_inliers``,
and the restatement's (tests/opencv_ransac_reference.py) ``c{i}_iterations``, ``c{i}_winner``, ``c{i}_counts`` and
``c{i}_samples``; ``c_tags`` names them.  The restatement's inlier list and pose equal cv2's on every case (asserted here).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))

from onepose_b200 import synthetic  # noqa: E402
from tests import opencv_ransac_reference as O  # noqa: E402

THRESHOLDS = (0.05, 0.7, 1.0, 3.0, 5.3, 5.7, 8.0, 1e6, float("inf"))
SCENES = ((1700, 60, 0.4), (1701, 200, 0.5), (1702, 30, 0.2))      # seed, n, outlier ratio; noise-free inliers
CONF, ITERS = 0.99, 2000


def main():
    import cv2
    res = {"cv2_version": np.array(cv2.__version__)}
    tags = []
    i = 0
    for thr in THRESHOLDS:
        for seed, n, frac in SCENES:
            K, uv, P, _ = synthetic.make_pnp_scene(seed, n, outlier_frac=frac, noise_px=0.0)
            P = P * 1000
            ok, rv, tv, inl = cv2.solvePnPRansac(P, uv, K, np.zeros((8, 1)), reprojectionError=thr, iterationsCount=ITERS,
                                                 confidence=CONF, flags=cv2.SOLVEPNP_EPNP)
            inl = np.zeros(0, np.int64) if inl is None else inl.reshape(-1).astype(np.int64)
            pose = np.concatenate([cv2.Rodrigues(rv)[0], tv], 1) if ok else np.eye(4)[:3]
            ok_r, rv_r, tv_r, inl_r, info = O.solve_pnp_ransac(P, uv, K, None, thr, ITERS, CONF)
            tag = f"thr{thr}_n{n}_out{frac}"
            assert ok_r == ok and inl_r.tolist() == inl.tolist(), tag
            assert not ok or (rv_r.tobytes() == rv.tobytes() and tv_r.tobytes() == tv.tobytes()), tag
            res.update({f"c{i}_K": K, f"c{i}_uv": uv, f"c{i}_P": P, f"c{i}_thr": np.float64(thr), f"c{i}_conf": np.float64(CONF),
                        f"c{i}_iters": np.int64(ITERS), f"c{i}_ok": np.bool_(ok), f"c{i}_cv": pose, f"c{i}_inliers": inl,
                        f"c{i}_iterations": np.int64(info["iterations"]), f"c{i}_winner": np.int64(info["winner"]),
                        f"c{i}_counts": np.asarray(info["counts"], np.int32), f"c{i}_samples": np.asarray(info["samples"], np.int32).reshape(-1, 5)})
            tags.append(tag)
            print(tag, "iterations", info["iterations"], "winner", info["winner"], "inliers", len(inl))
            i += 1
    res["c_tags"] = np.array(tags)
    np.savez_compressed(os.path.join(HERE, "pnp_domain_cases.npz"), **res)
    print(len(tags), "cases")


if __name__ == "__main__":
    main()
