"""Generate the fixtures of EPnP-RANSAC with OpenCV's loop (opb_ransac_epnp_cv) on a machine with OpenCV:

    python tests/golden/make_epnp_cv.py

Writes ``pnp_epnp_cv_cases.npz``: per case ``c{i}_K``, ``c{i}_uv``, ``c{i}_P`` (the 3D points as passed, millimetres as the
reference's ransac_PnP(scale=1000) passes them), ``c{i}_gt`` ([3,4], translation in millimetres), ``c{i}_conf``,
``c{i}_iters`` (iterationsCount), cv2.solvePnPRansac(..., flags=SOLVEPNP_EPNP)'s ``c{i}_ok``, ``c{i}_cv`` (pose [3,4]; the
identity when it fails) and ``c{i}_inliers``, and the restatement's (tests/opencv_ransac_reference.py) ``c{i}_iterations``,
``c{i}_winner``, ``c{i}_counts`` (per sample, -1 = no model) and ``c{i}_samples`` ([iterations, 5]); ``c_tags`` names them.
The restatement's inlier list and pose equal cv2's on every case (asserted here).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))

from onepose_b200 import synthetic  # noqa: E402
from tests import opencv_ransac_reference as O  # noqa: E402


def cases():
    out = []
    k = 0
    for n in (20, 100, 500):                                       # noise-free with outliers: every clean sample is exact
        for f, conf in ((0.3, 0.99), (0.5, 0.99), (0.7, 0.99), (0.5, 0.9), (0.5, 0.999)):
            out.append((f"clean_n{n}_out{f}_c{conf}", 600 + k, n, f, 0.0, conf, 10000))
            k += 1
    for n in (50, 200):                                            # 1 px noise
        for f in (0.25, 0.5):
            out.append((f"noisy_n{n}_out{f}", 700 + k, n, f, 1.0, 0.99, 10000))
            k += 1
    out.append(("noisy_n100_out0.8_iters300", 800, 100, 0.8, 1.0, 0.99, 300))
    g = np.load(os.path.join(HERE, "pnp_scenes.npz"))
    for s, n, fr in g["scenes"]:
        out.append((f"pnp_scene_{int(s)}", int(s), int(n), float(fr), 0.5, 0.99, 10000))
    out.append(("four", 901, 4, 0.0, 0.5, 0.99, 10000))
    out.append(("five", 902, 5, 0.0, 0.5, 0.99, 10000))
    out.append(("six", 903, 6, 0.0, 1.0, 0.99, 10000))
    return out


def main():
    import cv2
    res = {"cv2_version": np.array(cv2.__version__)}
    tags = []
    for i, (tag, seed, n, frac, noise, conf, iters) in enumerate(cases()):
        K, uv, P, gt = synthetic.make_pnp_scene(seed, n, outlier_frac=frac, noise_px=noise)
        P = P * 1000
        gt = np.concatenate([gt[:, :3], gt[:, 3:] * 1000], 1)
        if n < 4:                                                  # cv2 raises; the reference's except-branch
            ok, inl, pose = False, np.zeros(0, np.int64), np.eye(4)[:3]
            ok_r, inl_r, info = False, inl, {"iterations": 0, "winner": -1, "counts": [], "samples": []}
        else:
            ok, rv, tv, inl = cv2.solvePnPRansac(P, uv, K, np.zeros((8, 1)), reprojectionError=5, iterationsCount=iters,
                                                 confidence=conf, flags=cv2.SOLVEPNP_EPNP)
            inl = np.zeros(0, np.int64) if inl is None else inl.reshape(-1).astype(np.int64)
            pose = np.concatenate([cv2.Rodrigues(rv)[0], tv], 1) if ok else np.eye(4)[:3]
            ok_r, rv_r, tv_r, inl_r, info = O.solve_pnp_ransac(P, uv, K, None, 5.0, iters, conf)
        assert ok_r == ok and inl_r.tolist() == inl.tolist(), tag
        assert not ok or (rv_r.tobytes() == rv.tobytes() and tv_r.tobytes() == tv.tobytes()), tag
        res.update({f"c{i}_K": K, f"c{i}_uv": uv, f"c{i}_P": P, f"c{i}_gt": gt, f"c{i}_conf": np.float64(conf), f"c{i}_iters": np.int64(iters),
                    f"c{i}_ok": np.bool_(ok), f"c{i}_cv": pose, f"c{i}_inliers": inl, f"c{i}_iterations": np.int64(info["iterations"]),
                    f"c{i}_winner": np.int64(info["winner"]), f"c{i}_counts": np.asarray(info["counts"], np.int32),
                    f"c{i}_samples": np.asarray(info["samples"], np.int32).reshape(-1, 5)})
        tags.append(tag)
        print(tag, "n", n, "iterations", info["iterations"], "winner", info["winner"], "inliers", len(inl))
    res["c_tags"] = np.array(tags)
    np.savez_compressed(os.path.join(HERE, "pnp_epnp_cv_cases.npz"), **res)
    print(len(tags), "cases")


if __name__ == "__main__":
    main()
