"""numpy restatement of cv2.estimateAffinePartial2D(from, to, method=RANSAC) -- test infrastructure, not product code.

OpenCV's path (calib3d/src/ptsetreg.cpp: ``estimateAffinePartial2D``, ``RANSACPointSetRegistrator::run``,
``AffinePartial2DEstimatorCallback``, ``Affine2DEstimatorCallback::computeError``, ``AffinePartial2DRefineCallback``;
calib3d/src/levmarq.cpp: ``LMSolver``), stage by stage:
- the points are used as float32 (float64 input is converted first);
- ``n < 2``: no model; ``n == 2``: the one 2-point model, both pairs inliers, no refinement;
- the loop: ``cv::RNG((uint64)-1)``, two distinct indices per sample by ``getSubset`` (``draw_subset(k=2)``; the callback's
  ``checkSubset`` tests three or more points only, so every pair of distinct indices is accepted), the 2-point model, OpenCV's
  fp32 error against ``(float)(thr * thr)``, a win when the count is strictly above ``max(best, 1)``, then
  ``RANSACUpdateNumIters(confidence, outlier ratio, 2, budget)``; the loop exits at ``iter >= budget``;
- no winner: ``(None, zero mask)``;
- the refinement: the winner's inliers compressed in order, OpenCV's Levenberg-Marquardt on ``(a, b, tx, ty)`` for at most
  ``refineIters`` iterations (accepted steps), each step ``(J^T J) diag * (1 + 10^k)`` solved against ``J^T r``.
``minimal="cv2"`` takes each minimal model from ``cv2.estimateAffinePartial2D`` on exactly the two sampled pairs (OpenCV's own
``runKernel`` result); ``minimal="closed"`` evaluates ``run_kernel`` below, the closed form restated in numpy fp64.  The
generator and the 2-point scan need no cv2, so GPU tests use them without it.
"""
from __future__ import annotations

import numpy as np

from tests.opencv_ransac_reference import CvRNG, draw_subset, update_num_iters

MODEL_POINTS = 2
FLT_EPSILON = float(np.finfo(np.float32).eps)


def subsets(n: int, count: int):
    """The first ``count`` 2-point samples OpenCV draws for n pairs (a fresh generator)."""
    rng = CvRNG()
    return [draw_subset(rng, n, MODEL_POINTS) for _ in range(count)]


def scan(counts, n: int, confidence: float, max_iters: int):
    """The loop of ``run`` on per-sample inlier counts, for 2 model points.  Returns (winner or -1, best count, iterations)."""
    niters = max(max_iters, 1)
    best, winner, it = 0, -1, 0
    while it < niters:
        c = int(counts[it])
        if c > max(best, MODEL_POINTS - 1):
            best, winner = c, it
            niters = update_num_iters(confidence, (n - c) / n, MODEL_POINTS, niters)
        it += 1
    return winner, best, it


def run_kernel(f, t) -> np.ndarray:
    """``AffinePartial2DEstimatorCallback::runKernel`` on two fp32 pairs: the closed-form similarity in fp64, every operation
    rounded on its own (numpy never fuses a multiply-add).  Returns the 2x3 model."""
    x1, y1, x2, y2 = (float(v) for v in (f[0, 0], f[0, 1], f[1, 0], f[1, 1]))
    X1, Y1, X2, Y2 = (float(v) for v in (t[0, 0], t[0, 1], t[1, 0], t[1, 1]))
    with np.errstate(divide="ignore", invalid="ignore"):
        d = np.float64(1.0) / np.float64((x1 - x2) * (x1 - x2) + (y1 - y2) * (y1 - y2))
        S0 = d * ((X1 - X2) * (x1 - x2) + (Y1 - Y2) * (y1 - y2))
        S1 = d * ((Y1 - Y2) * (x1 - x2) - (X1 - X2) * (y1 - y2))
        S2 = d * ((Y1 - Y2) * (x1 * y2 - x2 * y1) - (X1 * y2 - X2 * y1) * (y1 - y2) - (X1 * x2 - X2 * x1) * (x1 - x2))
        S3 = d * (-(X1 - X2) * (x1 * y2 - x2 * y1) - (Y1 * x2 - Y2 * x1) * (x1 - x2) - (Y1 * y2 - Y2 * y1) * (y1 - y2))
    return np.array([[S0, -S1, S2], [S1, S0, S3]], np.float64)


def cv2_kernel(f, t) -> np.ndarray:
    """The 2-point model from OpenCV itself: estimateAffinePartial2D on exactly two pairs runs runKernel once."""
    import cv2
    H, _ = cv2.estimateAffinePartial2D(np.ascontiguousarray(f, np.float32), np.ascontiguousarray(t, np.float32))
    return H


def fp32_errors(H, f32, t32) -> np.ndarray:
    """``Affine2DEstimatorCallback::computeError``: the model rounded to fp32, ((F0 x + F1 y) + F2) - X in fp32, a^2 + b^2."""
    F = np.asarray(H, np.float64).reshape(6).astype(np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        a = F[0] * f32[:, 0] + F[1] * f32[:, 1] + F[2] - t32[:, 0]
        b = F[3] * f32[:, 0] + F[4] * f32[:, 1] + F[5] - t32[:, 1]
        return a * a + b * b


def _residuals(h, src, dst):
    Mx, My = src[:, 0].astype(np.float64), src[:, 1].astype(np.float64)
    r = np.empty(2 * len(src))
    r[0::2] = h[0] * Mx - h[1] * My + h[2] - dst[:, 0].astype(np.float64)
    r[1::2] = h[1] * Mx + h[0] * My + h[3] - dst[:, 1].astype(np.float64)
    return r


def _normal(h, src, dst):
    """(J^T J, J^T r, r) of AffinePartial2DRefineCallback: rows (x, -y, 1, 0) and (y, x, 0, 1) per pair."""
    Mx, My = src[:, 0].astype(np.float64), src[:, 1].astype(np.float64)
    J = np.zeros((2 * len(src), 4))
    J[0::2, 0], J[0::2, 1], J[0::2, 2] = Mx, -My, 1.0
    J[1::2, 0], J[1::2, 1], J[1::2, 3] = My, Mx, 1.0
    r = _residuals(h, src, dst)
    return J.T @ J, J.T @ r, r


def lm_refine(H, src, dst, max_iters: int, eps: float = FLT_EPSILON):
    """OpenCV's LMSolver (eps = FLT_EPSILON) on (a, b, tx, ty) = (H00, H10, H02, H12).  Returns (H refined, accepted steps)."""
    x = np.array([H[0, 0], H[1, 0], H[0, 2], H[1, 2]], np.float64)
    A, v, r = _normal(x, src, dst)
    S = float(r @ r)
    lg, it = -3, 0
    while True:
        Ap = A.copy()
        lam = np.exp(lg * np.log(10.0))
        Ap[np.diag_indices(4)] *= 1 + lam
        d = np.linalg.solve(Ap, v)
        xd = x - d
        rd = _residuals(xd, src, dst)
        Sd = float(rd @ rd)
        if Sd < S:
            S, x, it = Sd, xd, it + 1
            lg = max(lg - 1, -16)
            A, v, r = _normal(x, src, dst)
        else:
            it += lg == 16
            lg = min(lg + 1, 16)
        if not (it < max_iters and np.abs(d).max() >= eps and S >= eps * eps):
            break
    out = np.array([[x[0], -x[1], x[2]], [x[1], x[0], x[3]]], np.float64)
    return out, it


def estimate_affine_partial_2d(from_pts, to_pts, thr=3.0, max_iters=2000, confidence=0.99, refine_iters=10, minimal="cv2"):
    """(H [2,3] f64 or None, mask uint8 [n], info) like cv2.estimateAffinePartial2D(from, to, RANSAC, thr, max_iters,
    confidence, refine_iters).  info: iterations, winner, samples, counts (per sample), models (per sample, unrefined)."""
    kernel = cv2_kernel if minimal == "cv2" else run_kernel
    f32 = np.ascontiguousarray(np.asarray(from_pts, np.float64).reshape(-1, 2).astype(np.float32))
    t32 = np.ascontiguousarray(np.asarray(to_pts, np.float64).reshape(-1, 2).astype(np.float32))
    n = len(f32)
    if not 0 < confidence < 1:
        raise ValueError("OpenCV's run() asserts 0 < confidence < 1")
    info = {"iterations": 0, "winner": -1, "samples": [], "counts": [], "models": [], "unrefined": None}
    if n < MODEL_POINTS:
        return None, np.zeros(n, np.uint8), info
    if n == MODEL_POINTS:
        H = kernel(f32, t32)
        info["unrefined"] = H
        return H, np.ones(n, np.uint8), info
    thr2 = np.float32(thr * thr)
    rng = CvRNG()
    niters = max(int(max_iters), 1)
    best, best_mask, best_H, it = 0, None, None, 0
    while it < niters:
        idx = draw_subset(rng, n, MODEL_POINTS)
        H = kernel(f32[list(idx)], t32[list(idx)])
        mask = fp32_errors(H, f32, t32) <= thr2
        c = int(mask.sum())
        info["samples"].append(idx)
        info["models"].append(H)
        info["counts"].append(c)
        if c > max(best, MODEL_POINTS - 1):
            best, best_mask, best_H, info["winner"] = c, mask, H, it
            niters = update_num_iters(confidence, (n - c) / n, MODEL_POINTS, niters)
        it += 1
    info["iterations"] = it
    if best_mask is None:
        return None, np.zeros(n, np.uint8), info
    info["unrefined"] = best_H
    H = best_H
    if refine_iters > 0:
        inl = np.nonzero(best_mask)[0]
        H, info["lm_iterations"] = lm_refine(best_H, f32[inl], t32[inl], int(refine_iters))
    return H, best_mask.astype(np.uint8), info


# ---- the detector's box and selection (local_feature_2D_detector.py:76-147) ----

def corners_box(H, db_hw):
    """(affine @ four corners).T.astype(int32), then min / max: [x0, y0, x1, y1] or None where numpy's cast is undefined."""
    h, w = (float(v) for v in db_hw)
    c = np.array([[0, 0, 1], [w, 0, 1], [0, h, 1], [w, h, 1]], np.float64).T
    p = (np.asarray(H, np.float64) @ c).T
    if not np.all(np.isfinite(p)) or np.any(p <= -2147483649.0) or np.any(p >= 2147483648.0):
        return None
    q = p.astype(np.int32)
    return np.concatenate([q.min(axis=0), q.max(axis=0)]).astype(np.int32)
