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
- the refinement: the winner's inliers compressed in order, OpenCV's ``LMSolver`` on ``(a, b, tx, ty)`` for at most
  ``refineIters`` iterations (kept or not), each step ``J^T J + lambda diag(J^T J)_0`` solved against ``J^T r`` by eigen
  decomposition (``lm_refine``; the schedule was worked out from cv2 4.13's results and reproduces them to 1e-13 relative,
  bit for bit at most points, also at coordinates shifted by 1e6, where ``cv::solve``'s dropped eigenvalues stop the
  translation from moving).
``minimal="cv2"`` takes each minimal model from ``cv2.estimateAffinePartial2D`` on exactly the two sampled pairs (OpenCV's own
``runKernel`` result); ``minimal="closed"`` evaluates ``run_kernel`` below, the closed form restated in numpy fp64.  The
generator and the 2-point scan need no cv2, so GPU tests use them without it.
"""
from __future__ import annotations

import numpy as np

from tests.opencv_ransac_reference import CvRNG, draw_subset, update_num_iters

MODEL_POINTS = 2
FLT_EPSILON = float(np.finfo(np.float32).eps)
DBL_EPSILON = float(np.finfo(np.float64).eps)


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


def jacobi(M):
    """``cv::eigen`` of a symmetric fp64 matrix as OpenCV's ``JacobiImpl_`` runs it: cyclic-by-largest Jacobi rotations (the
    largest off-diagonal |a_kl| found through per-row and per-column maxima), stopping when it is <= DBL_EPSILON (absolute) or
    after 30 n^2 rotations, then eigenvalues sorted in descending order.  Returns (w [n], V [n, n], row i the eigenvector of w[i])."""
    A = np.array(M, np.float64)
    n = len(A)
    V, W = np.eye(n), np.diag(A).copy()
    ind_r, ind_c = [0] * n, [0] * n

    def row_max(k):
        m = k + 1
        for i in range(k + 2, n):
            m = i if abs(A[k, m]) < abs(A[k, i]) else m
        return m

    def col_max(k):
        m = 0
        for i in range(1, k):
            m = i if abs(A[m, k]) < abs(A[i, k]) else m
        return m

    for k in range(n):
        ind_r[k] = row_max(k) if k < n - 1 else 0
        ind_c[k] = col_max(k) if k > 0 else 0
    for _ in range(30 * n * n if n > 1 else 0):
        k, mv = 0, abs(A[0, ind_r[0]])
        for i in range(1, n - 1):
            if mv < abs(A[i, ind_r[i]]):
                mv, k = abs(A[i, ind_r[i]]), i
        l = ind_r[k]
        for i in range(1, n):
            if mv < abs(A[ind_c[i], i]):
                mv, k, l = abs(A[ind_c[i], i]), ind_c[i], i
        p = A[k, l]
        if abs(p) <= DBL_EPSILON:
            break
        y = (W[l] - W[k]) * 0.5
        t = abs(y) + np.hypot(p, y)
        s = np.hypot(p, t)
        c = t / s
        s, t = p / s, (p / t) * p
        if y < 0:
            s, t = -s, -t
        A[k, l] = 0.0
        W[k] -= t
        W[l] += t

        def rot(a0, b0):
            return a0 * c - b0 * s, a0 * s + b0 * c
        for i in range(k):
            A[i, k], A[i, l] = rot(A[i, k], A[i, l])
        for i in range(k + 1, l):
            A[k, i], A[i, l] = rot(A[k, i], A[i, l])
        for i in range(l + 1, n):
            A[k, i], A[l, i] = rot(A[k, i], A[l, i])
        for i in range(n):
            V[k, i], V[l, i] = rot(V[k, i], V[l, i])
        for idx in (k, l):
            if idx < n - 1:
                ind_r[idx] = row_max(idx)
            if idx > 0:
                ind_c[idx] = col_max(idx)
    for k in range(n - 1):
        m = k
        for i in range(k + 1, n):
            m = i if W[m] < W[i] else m
        if m != k:
            W[[k, m]], V[[k, m]] = W[[m, k]], V[[m, k]]
    return W, V


def _kept(w):
    """``SVBkSb``'s rule: an eigenvalue counts when |w_i| > 2 DBL_EPSILON * sum(w); the others are dropped (a pseudo-inverse)."""
    thr = 0.0
    for wi in w:
        thr += wi
    return [i for i in range(len(w)) if abs(w[i]) > thr * (2 * DBL_EPSILON)]


def eig_solve(M, b):
    """``cv::solve(M, b, d, DECOMP_EIG)``: sum over the kept eigenpairs of v_i (v_i . b) / w_i, in eigenvalue order."""
    w, V = jacobi(M)
    x = np.zeros(len(w))
    for i in _kept(w):
        s = 0.0
        for j in range(len(w)):
            s += V[i, j] * b[j]
        x = x + (s * (1.0 / w[i])) * V[i]
    return x


def eig_inverse_diagonal(M):
    """The diagonal of ``cv::invert(M, DECOMP_EIG)``, the pseudo-inverse over the kept eigenpairs."""
    w, V = jacobi(M)
    out = np.zeros(len(w))
    for i in _kept(w):
        out = out + V[i] * ((1.0 / w[i]) * V[i])
    return out


def lm_refine(H, src, dst, max_iters: int, eps: float = FLT_EPSILON):
    """OpenCV's ``LMSolver`` (eps = FLT_EPSILON) on (a, b, tx, ty) = (H00, H10, H02, H12).  D = diag(J^T J) at the start,
    lambda = 1, lc = 0.75.  Each iteration solves (J^T J + lambda D) d = J^T r by ``eig_solve`` and tries x - d.  With the
    predicted decrease dS = d . (2 J^T r - J^T J d) and R = (S - Sd) / dS (dS taken as 1 where |dS| <= DBL_EPSILON):
    R > 0.75 halves lambda, to 0 (Gauss-Newton) once it drops below lc; R < 0.25 multiplies it by
    nu = clamp((Sd - S) / (d . J^T r) + 2, 2, 10), and from lambda = 0 first sets lambda = lc = 1 / max |diag((J^T J)^+)| and
    halves nu.  The step is kept when Sd < S.  Every iteration counts, kept or not; the loop stops after max_iters of them, or
    when |d|_inf < eps or when the largest residual |r_i| of the kept model is < eps (not S < eps^2: on sub-pixel fits every
    |r_i| can be below eps while S is still above eps^2, and cv2 stops there).  A NaN residual is passed over, as a running
    std::max from 0 does.  Returns (H refined, iterations)."""
    x = np.array([H[0, 0], H[1, 0], H[0, 2], H[1, 2]], np.float64)
    A, v, r = _normal(x, src, dst)
    S = float(r @ r)
    D = np.diag(A).copy()
    lam, lc, it = 1.0, 0.75, 0
    while True:
        Ap = A.copy()
        Ap[np.diag_indices(4)] += lam * D
        d = eig_solve(Ap, v)
        xd = x - d
        rd = _residuals(xd, src, dst)
        Sd = float(rd @ rd)
        dS = float(d @ (2 * v - A @ d))
        R = (S - Sd) / (dS if abs(dS) > DBL_EPSILON else 1.0)
        if R > 0.75:
            lam *= 0.5
            if lam < lc:
                lam = 0.0
        elif R < 0.25:
            t = float(d @ v)
            nu = min(max((Sd - S) / (t if abs(t) > DBL_EPSILON else 1.0) + 2, 2.0), 10.0)
            if lam == 0:
                lam = lc = 1.0 / max(DBL_EPSILON, float(np.abs(eig_inverse_diagonal(A)).max()))
                nu *= 0.5
            lam *= nu
        if Sd < S:
            S, x = Sd, xd
            A, v, r = _normal(x, src, dst)
        it += 1
        if not (it < max_iters and np.abs(d).max() >= eps and np.fmax.reduce(np.abs(r)) >= eps):
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
