"""Seeded scenes of the flow step's tests and goldens, free of side effects on import (cv2 is imported only by ``lk_scene``).

``lk_scene``      a textured image, its affine / perspective / large motion, and points in a flat corner, on and past the borders.
``warp_scene``    the same without cv2 (the GPU tests use it): a textured image with a flat corner and its affine motion, warped in
                  numpy (fp64 bilinear, BORDER_REFLECT, rounded to uint8).
``scene_points``  seeded points over and past an image, a share of them in its flat corner.
``border_points`` points on the integer-corner edges of every pyramid level of a window, one fp32 ulp either side, and the
                  non-finite and huge coordinates.
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


def _reflect(i: np.ndarray, n: int) -> np.ndarray:
    """cv::borderInterpolate(i, n, BORDER_REFLECT): ... 1 0 | 0 1 ... n-1 | n-1 n-2 ..."""
    m = np.mod(i, 2 * n)
    return np.where(m >= n, 2 * n - 1 - m, m)


def warp_scene(seed: int, h: int, w: int, motion: str = "affine"):
    """(prev, next) uint8 [h, w]: the texture with a flat corner, and it under a seeded affine map -- sub-pixel ("affine": 2 %
    linear part, 2.5 px shift) or "large" (10 %, 12 px).  next(x, y) = prev(M [x, y, 1]) by fp64 bilinear interpolation with a
    BORDER_REFLECT border, rounded to the nearest grey level."""
    rs = np.random.RandomState(seed)
    img = np.ascontiguousarray(texture(seed, max(h, 32), max(w, 32))[:h, :w])     # tiny images: a corner of a larger texture
    if h >= 16 and w >= 16:
        img[: h // 4, : w // 4] = 90                    # a flat corner: points there fail the eigenvalue test
    a, shift = (0.02, 2.5) if motion == "affine" else (0.1, 12.0)
    M = np.array([[1 + a * rs.randn(), a * rs.randn(), shift * rs.randn()], [a * rs.randn(), 1 + a * rs.randn(), shift * rs.randn()]])
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    sx = M[0, 0] * xx + M[0, 1] * yy + M[0, 2]
    sy = M[1, 0] * xx + M[1, 1] * yy + M[1, 2]
    x0, y0 = np.floor(sx).astype(np.int64), np.floor(sy).astype(np.int64)
    fx, fy = sx - x0, sy - y0
    src = img.astype(np.float64)
    xa, xb, ya, yb = _reflect(x0, w), _reflect(x0 + 1, w), _reflect(y0, h), _reflect(y0 + 1, h)
    v = (src[ya, xa] * (1 - fx) + src[ya, xb] * fx) * (1 - fy) + (src[yb, xa] * (1 - fx) + src[yb, xb] * fx) * fy
    return img, np.clip(np.rint(v), 0, 255).astype(np.uint8)


def scene_points(seed: int, h: int, w: int, n: int, margin: float = 25.0) -> np.ndarray:
    """fp32 [n, 2] seeded points over [-margin, w + margin] x [-margin, h + margin], the first n // 20 in the flat corner."""
    rs = np.random.RandomState(seed + 1000)
    pts = np.stack([rs.uniform(-margin, w + margin, n), rs.uniform(-margin, h + margin, n)], 1)
    k = n // 20
    pts[:k] = np.stack([rs.uniform(0, w / 4, k), rs.uniform(0, h / 4, k)], 1)
    return pts.astype(np.float32)


SPECIAL = np.array([np.nan, np.inf, -np.inf, 9.99e8, -9.99e8, 1e9, -1e9], np.float32)


def border_points(h: int, w: int, win, levels: int) -> np.ndarray:
    """fp32 [n, 2]: for each level l <= levels of an h x w pyramid, the points p whose floor(p 2^-l - half) is exactly -win - 1,
    -win, side_l - 1 or side_l along x (y at the middle of the image) and along y (x at the middle), each at the exact value
    and one fp32 ulp either side; then SPECIAL along x and along y, and both coordinates NaN."""
    ww, wh = win
    out = []
    for axis, (n, half, other) in enumerate([(w, (ww - 1) / 2, h / 2), (h, (wh - 1) / 2, w / 2)]):
        side, win_side = n, (ww, wh)[axis]
        for lev in range(levels + 1):
            for k in (-win_side - 1, -win_side, side - 1, side):
                p = np.float32((k + half) * 2.0 ** lev)
                for q in (np.nextafter(p, np.float32(-np.inf)), p, np.nextafter(p, np.float32(np.inf))):
                    out.append((q, other) if axis == 0 else (other, q))
            side = (side + 1) // 2
        out += [(s, other) if axis == 0 else (other, s) for s in SPECIAL]
    out.append((np.nan, np.nan))
    return np.array(out, np.float32)


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
