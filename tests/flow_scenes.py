"""Seeded scenes of the flow step's tests and goldens, free of side effects on import (cv2 is imported only by ``lk_scene``).

``lk_scene``      a textured image, its affine / perspective / large motion, and points in a flat corner, on and past the borders.
``blob_object``   a non-planar object: M 3D points (metres, ~10 cm across) that each carry a Gaussian blob of their own grey level.
``render_blobs``  the object seen from a pose in an S x S crop: every point's blob at its projection (numpy, fp64, then uint8).
"""
from __future__ import annotations

import numpy as np

from onepose_b200 import synthetic


def texture(seed: int, h: int, w: int) -> np.ndarray:
    return np.round(synthetic.make_image(seed, h, w)[0] * 255).astype(np.uint8)


def lk_scene(seed, h, w, motion):
    import cv2
    rs = np.random.RandomState(seed)
    img = texture(seed, h, w)
    img[: h // 4, : w // 4] = 90                      # a flat corner: points there fail the eigenvalue test
    if motion == "perspective":
        src = np.float32([[0, 0], [w, 0], [w, h], [0, h]])
        M = cv2.getPerspectiveTransform(src, src + rs.uniform(-5, 5, (4, 2)).astype(np.float32))
        nxt = cv2.warpPerspective(img, M, (w, h), borderMode=cv2.BORDER_REFLECT)
    else:
        a = 0.02 if motion == "affine" else 0.1
        shift = 2.5 if motion == "affine" else 12.0
        M = np.array([[1 + a * rs.randn(), a * rs.randn(), shift * rs.randn()], [a * rs.randn(), 1 + a * rs.randn(), shift * rs.randn()]])
        nxt = cv2.warpAffine(img, M, (w, h), borderMode=cv2.BORDER_REFLECT)
    n = 400
    pts = np.stack([rs.uniform(-25, w + 25, n), rs.uniform(-25, h + 25, n)], 1)
    pts[:20] = np.stack([rs.uniform(0, w / 4, 20), rs.uniform(0, h / 4, 20)], 1)     # in the flat corner
    pts[20:40, 0] = rs.choice([-0.5, 0.0, w - 1.0, w - 0.5, w + 3.0], 20)          # on and past the borders
    return img, nxt, pts.astype(np.float32)


def rodrigues(w) -> np.ndarray:
    w = np.asarray(w, np.float64)
    th = np.linalg.norm(w)
    if th == 0:
        return np.eye(3)
    k = w / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx


def blob_object(seed: int, M: int):
    """(X fp32 [M,3], grey amplitudes [M]) of a seeded non-planar point cloud."""
    rs = np.random.RandomState(seed)
    X = (rs.uniform(-0.06, 0.06, (M, 3))).astype(np.float32)
    amp = rs.uniform(60, 200, M) * rs.choice([-1, 1], M)
    return X, amp


def project(K, pose, X):
    x = np.asarray(X, np.float64) @ pose[:3, :3].T + pose[:3, 3]
    x = x @ K.T
    return x[:, :2] / x[:, 2:]


def render_blobs(K, pose, X, amp, S: int, sigma: float = 1.8) -> np.ndarray:
    uv = project(K, pose, X)
    yy, xx = np.mgrid[0:S, 0:S].astype(np.float64)
    img = np.full((S, S), 128.0)
    for (u, v), a in zip(uv, amp):
        if -10 < u < S + 10 and -10 < v < S + 10:
            y0, y1, x0, x1 = max(int(v) - 8, 0), min(int(v) + 9, S), max(int(u) - 8, 0), min(int(u) + 9, S)
            if y0 < y1 and x0 < x1:
                img[y0:y1, x0:x1] += a * np.exp(-((yy[y0:y1, x0:x1] - v) ** 2 + (xx[y0:y1, x0:x1] - u) ** 2) / (2 * sigma * sigma))
    return np.clip(np.round(img), 0, 255).astype(np.uint8)


def pose_at(pose0, dw, dt) -> np.ndarray:
    """pose0 [3,4] moved by the rotation vector dw (about the camera) and the translation dt."""
    return np.concatenate([rodrigues(dw) @ pose0[:, :3], pose0[:, 3:] + np.reshape(dt, (3, 1))], 1)
