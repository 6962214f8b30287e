"""Generate the EPnP golden vectors with OpenCV used as a black box:

    python tests/golden/make_epnp.py

Writes ``pnp_epnp_cases.npz`` (the ``pnp_`` prefix keeps it out of the matcher cases that ``tests/golden_util.py`` collects):
- ``cv2.solvePnP(flags=SOLVEPNP_EPNP)`` on fixed point sets: generic scenes of n = 4, 5, 6, 10, 50, 300 and 1000 pairs with
  0, 0.5 and 2 px of pixel noise, in metres and in millimetres; fp32-rounded copies of the 0.5 px sets in metres; planar sets.
  Keys ``p{i}_K``, ``p{i}_uv``, ``p{i}_P``, ``p{i}_gt`` (ground truth [3,4]), ``p{i}_cv`` ([3,4]) and ``p_tags``.
- ``cv2.solvePnPRansac(..., reprojectionError=5, iterationsCount=10000, flags=SOLVEPNP_EPNP)`` as the reference's
  ``ransac_PnP`` calls it (3D points x 1000, translation / 1000) on the ``pnp_scenes`` seeds, and on a scene whose last 20 of
  80 points are mirrored through the camera centre (behind the camera, at the same pixels), and on a 4-pair scene (a
  five-point model cannot be drawn from it: a pose with 4 inliers shows that OpenCV switches to a 4-point model there).  Keys ``r{i}_K``, ``r{i}_uv``,
  ``r{i}_P``, ``r{i}_gt``, ``r{i}_cv`` (pose [3,4], the identity when OpenCV fails), ``r{i}_inliers`` and ``r_tags``.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))

from onepose_b200 import synthetic  # noqa: E402


def _rodrigues(w):
    th = np.linalg.norm(w)
    W = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
    return np.eye(3) + np.sin(th) / th * W + (1 - np.cos(th)) / (th * th) * W @ W


def _project(K, P, R, t):
    X = P @ R.T + t
    return X[:, :2] / X[:, 2:3] * np.array([K[0, 0], K[1, 1]]) + K[:2, 2]


def planar_scene(seed, n):
    rs = np.random.RandomState(seed)
    K = np.array([[620.0, 0, 250], [0, 630.0, 262], [0, 0, 1]])
    P = np.concatenate([rs.uniform(-0.06, 0.06, size=(n, 2)), np.zeros((n, 1))], 1)
    R = _rodrigues(rs.uniform(-0.6, 0.6, 3))
    t = np.array([0.02, -0.01, 0.6])
    return K, _project(K, P, R, t), P, np.concatenate([R, t[:, None]], 1)


def behind_scene():
    """80 pairs: 60 ordinary ones with 0.5 px noise, then 20 whose world points are mirrored through the camera centre under
    the true pose (camera coordinates -X: behind the camera, projecting to the same pixels)."""
    K, uv, P, gt = synthetic.make_pnp_scene(900, 80, outlier_frac=0.0, noise_px=0.5)
    R, t = gt[:, :3], gt[:, 3]
    X = P[60:] @ R.T + t
    P = P.copy()
    P[60:] = (-X - t) @ R
    return K, uv, P, gt


def main():
    import cv2

    def solve(K, uv, P):
        ok, rv, tv = cv2.solvePnP(P, uv, K, np.zeros(4), flags=cv2.SOLVEPNP_EPNP)
        return np.concatenate([cv2.Rodrigues(rv)[0], tv], 1)

    out = {"cv2_version": np.array(cv2.__version__)}
    tags = []
    for n in (4, 5, 6, 10, 50, 300, 1000):
        for noise in (0.0, 0.5, 2.0):
            for unit, s in (("m", 1.0), ("mm", 1000.0)):
                K, uv, P, gt = synthetic.make_pnp_scene(7000 + n, n, outlier_frac=0.0, noise_px=noise)
                tags.append((f"generic_n{n}_noise{noise}_{unit}", K, uv, P * s, np.concatenate([gt[:, :3], gt[:, 3:] * s], 1)))
        K, uv, P, gt = synthetic.make_pnp_scene(7000 + n, n, outlier_frac=0.0, noise_px=0.5)
        f = lambda x: x.astype(np.float32).astype(np.float64)   # noqa: E731
        tags.append((f"generic_n{n}_noise0.5_m_fp32", K, f(uv), f(P), gt))
    for n in (6, 50, 500):
        tags.append((f"planar_n{n}", *planar_scene(8000 + n, n)))
    for i, (tag, K, uv, P, gt) in enumerate(tags):
        out.update({f"p{i}_K": K, f"p{i}_uv": uv, f"p{i}_P": P, f"p{i}_gt": gt, f"p{i}_cv": solve(K, uv, P)})
    out["p_tags"] = np.array([t[0] for t in tags])

    g = np.load(os.path.join(HERE, "pnp_scenes.npz"))
    scenes = [(f"pnp_scene_{int(s)}", *synthetic.make_pnp_scene(int(s), int(n), float(fr))) for s, n, fr in g["scenes"]]
    scenes.append(("behind", *behind_scene()))
    scenes.append(("four", *synthetic.make_pnp_scene(901, 4, outlier_frac=0.0, noise_px=0.5)))   # below EPnP's 5-point sample
    for i, (tag, K, uv, P, gt) in enumerate(scenes):
        try:
            _, rv, tv, inl = cv2.solvePnPRansac(P * 1000, uv, K, np.zeros((8, 1)), reprojectionError=5, iterationsCount=10000,
                                                flags=cv2.SOLVEPNP_EPNP)
            pose = np.concatenate([cv2.Rodrigues(rv)[0], tv / 1000], 1)
            inl = np.zeros(0, np.int64) if inl is None else inl.reshape(-1).astype(np.int64)
        except cv2.error:
            pose, inl = np.eye(4)[:3], np.zeros(0, np.int64)
        out.update({f"r{i}_K": K, f"r{i}_uv": uv, f"r{i}_P": P, f"r{i}_gt": gt, f"r{i}_cv": pose, f"r{i}_inliers": inl})
        print(tag, "n", len(uv), "inliers", len(inl))
    out["r_tags"] = np.array([s[0] for s in scenes])
    np.savez_compressed(os.path.join(HERE, "pnp_epnp_cases.npz"), **out)
    print(len(tags), "solvePnP cases,", len(scenes), "solvePnPRansac cases")


if __name__ == "__main__":
    main()
