"""numpy restatement of cv2.solvePnPRansac(..., flags=SOLVEPNP_EPNP) -- test infrastructure, not product code.

OpenCV's loop (``RANSACPointSetRegistrator::run`` and ``getSubset`` in calib3d/src/ptsetreg.cpp, ``PnPRansacCallback`` and
``solvePnPRansac`` in calib3d/src/solvepnp.cpp), stage by stage:
- ``CvRNG``             ``cv::RNG``: multiply-with-carry, state = (uint32)state * 4164903690 + (state >> 32), ``uniform(0, n)``
                        = (uint32)state % n; ``run`` builds it from (uint64)-1 on every call;
- ``draw_subset``       ``getSubset``: five indices, an index equal to an earlier one of the same sample is redrawn;
- ``update_num_iters``  ``RANSACUpdateNumIters`` with its clamps, DBL_MIN guards and cvRound (half to even);
- ``scan``              the loop's bookkeeping on given per-sample counts: a sample wins when its count is strictly greater
                        than max(best, modelPoints - 1), the budget is updated after each win, the loop stops at iter >= niters;
- ``solve_pnp_ransac``  everything: inputs rounded to fp32, each minimal model from ``cv2.solvePnP(EPNP)``, OpenCV's fp32
                        error (``projectPoints`` to fp32, squared norm in fp32, against ``fp32_threshold2``), the winner's
                        mask, and the EPnP refit on it.  Frames of 4 or 5 pairs (``model_points == npoints``) are solved
                        directly and every pair is an inlier, as there.
Only ``solve_pnp_ransac`` and ``fp32_errors`` need cv2; the generator and the scan do not, so GPU tests use them without it.
``run`` asserts 0 < confidence < 1; ``update_num_iters`` clamps instead, which is what the GPU mode does at 0 and 1.
"""
from __future__ import annotations

import math

import numpy as np

MWC_A = 4164903690
MWC_M = MWC_A * 2 ** 32 - 1          # the MWC step is the LCG state -> state * MWC_A mod MWC_M in disguise
MODEL_POINTS = 5
DBL_MIN = 2.2250738585072014e-308


class CvRNG:
    def __init__(self, state: int = 2 ** 64 - 1):
        self.state = state

    def next(self) -> int:
        self.state = (self.state & 0xFFFFFFFF) * MWC_A + (self.state >> 32)
        return self.state & 0xFFFFFFFF

    def uniform(self, n: int) -> int:
        return self.next() % n


def draw_subset(rng: CvRNG, n: int, k: int = MODEL_POINTS):
    idx = []
    for _ in range(k):
        v = rng.uniform(n)
        while v in idx:
            v = rng.uniform(n)
        idx.append(v)
    return tuple(idx)


def subsets(n: int, count: int):
    """The first ``count`` samples OpenCV draws for a frame of n pairs (a fresh generator)."""
    rng = CvRNG()
    return [draw_subset(rng, n) for _ in range(count)]


def update_num_iters(p: float, ep: float, model_points: int, max_iters: int) -> int:
    p = min(max(p, 0.0), 1.0)
    ep = min(max(ep, 0.0), 1.0)
    num = max(1.0 - p, DBL_MIN)
    denom = 1.0 - math.pow(1.0 - ep, model_points)
    if denom < DBL_MIN:
        return 0
    num = math.log(num)
    denom = math.log(denom)
    if denom >= 0 or -num >= max_iters * (-denom):
        return max_iters
    return int(np.rint(num / denom))              # cvRound: round half to even


def scan(counts, n: int, confidence: float, max_iters: int):
    """The loop of ``run`` on per-sample inlier counts (``counts[i]`` for sample i; < 0 = no model).  Returns
    (winner index or -1, best count, iterations = the iter at which the loop exits)."""
    niters = max(max_iters, 1)
    best, winner, it = 0, -1, 0
    while it < niters:
        c = int(counts[it])
        if c > max(best, MODEL_POINTS - 1):
            best, winner = c, it
            niters = update_num_iters(confidence, (n - c) / n, MODEL_POINTS, niters)
        it += 1
    return winner, best, it


def fp32_threshold2(thr: float) -> np.float32:
    """findInliers' squared threshold: solvePnPRansac's ``float reprojectionError`` (the threshold rounded to fp32 first),
    squared in double (exact) and rounded to fp32 -- the fp32 product of the fp32 threshold."""
    t = np.float32(thr)
    return t * t


# the boundary scene: integer world points at depths 2 .. 16 seen from the identity pose through K = diag(1000, 1000, 1); every
# normalised coordinate x / z is dyadic, so it survives OpenCV's fp32 undistortPoints, EPnP on any five of them returns the
# identity pose to ~1e-15 and every pixel reprojects to its fp32 value (error below 1e-20).  Row 0 is the probe, a point on the
# optical axis: it projects to (0, 0) and its fp32 error is that of its observation (du, dv) alone.  Sample 0 of 13 pairs is
# (9, 11, 4, 12, 7): with iterationsCount = 1 the mask is that exact pose's, probe included.
BOUNDARY_POINTS = ((0, 0, 7), (1, 0, 16), (-1, -3, 4), (-3, -2, 2), (1, 3, 16), (1, 3, 8), (1, 0, 8), (3, -2, 8), (1, -3, 16),
                   (3, 0, 4), (2, 2, 2), (-2, -3, 16), (-3, 0, 16))


def _round32(q):
    """The rational q rounded to fp32, to nearest with ties to even, exactly."""
    from fractions import Fraction
    a = np.float32(float(q))
    best = None
    for c in (np.nextafter(a, np.float32(-np.inf)), a, np.nextafter(a, np.float32(np.inf))):
        d = abs(Fraction(float(c)) - q)
        if best is None or d < best[0] or (d == best[0] and int(np.float32(c).view(np.uint32)) & 1 == 0):
            best = (d, c)
    return np.float32(best[1])


def probe_offset(err):
    """fp32 (du, dv) whose squared norm is exactly the fp32 value err in fp32 with and without FMA contraction (either
    product fused), so that the probe's error does not depend on how computeError's sum is compiled."""
    from fractions import Fraction
    err = np.float32(err)
    dv0 = np.float32(0.5 if err > 1 else 0.05)
    dvs = (dv0 + np.arange(-4000, 4000, dtype=np.float32) * np.spacing(dv0)).astype(np.float32)
    du0 = np.float32(math.sqrt(float(err) - float(dv0) ** 2))
    for k in range(-20, 21):
        du = np.float32(du0 + np.float32(k) * np.spacing(du0))
        for j in np.nonzero(du * du + dvs * dvs == err)[0]:
            a, b = Fraction(float(du)) ** 2, Fraction(float(dvs[j])) ** 2
            ra, rb = Fraction(float(_round32(a))), Fraction(float(_round32(b)))
            if _round32(ra + rb) == _round32(a + rb) == _round32(ra + b) == err:
                return du, dvs[j]
    raise ValueError(f"no probe offset for {err!r}")


def boundary_scene(err):
    """(K, uv, P) of 13 pairs: the boundary scene with the probe (row 0) observed at fp32 squared error err."""
    P = np.array(BOUNDARY_POINTS, np.float64)
    uv = 1000 * P[:, :2] / P[:, 2:]
    uv[0] = probe_offset(err)
    return np.diag([1000.0, 1000.0, 1.0]), uv, P


def fp32_errors(P32, uv32, K, dist, rvec, tvec):
    """``PnPRansacCallback::computeError``: projectPoints of the fp32 points (fp32 output), squared distance in fp32."""
    import cv2
    proj = cv2.projectPoints(P32, rvec, tvec, K, dist)[0].reshape(-1, 2)
    assert proj.dtype == np.float32
    d = uv32 - proj
    return d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]


def solve_pnp_ransac(P, uv, K, dist=None, thr=5.0, iterations_count=10000, confidence=0.99):
    """(ok, rvec, tvec, inliers [k] int, info) like cv2.solvePnPRansac(P, uv, K, dist, reprojectionError=thr,
    iterationsCount=iterations_count, confidence=confidence, flags=SOLVEPNP_EPNP).  info: iterations, winner, samples (the
    subsets drawn), counts (per sample; -1 = no model)."""
    import cv2
    dist = np.zeros((8, 1)) if dist is None else dist
    K = np.asarray(K, np.float64)
    P32 = np.ascontiguousarray(np.asarray(P, np.float64).reshape(-1, 3).astype(np.float32))
    uv32 = np.ascontiguousarray(np.asarray(uv, np.float64).reshape(-1, 2).astype(np.float32))
    n = len(P32)
    if n < 4:
        raise ValueError("solvePnPRansac needs at least 4 pairs")
    model_points, method = (4, cv2.SOLVEPNP_P3P) if n == 4 else (MODEL_POINTS, cv2.SOLVEPNP_EPNP)
    info = {"iterations": 0, "winner": -1, "samples": [], "counts": []}
    if n == model_points:
        ok, rv, tv = cv2.solvePnP(P32, uv32, K, dist, flags=method)
        return bool(ok), rv, tv, np.arange(n) if ok else np.zeros(0, np.int64), info
    if not 0 < confidence < 1:
        raise ValueError("OpenCV's run() asserts 0 < confidence < 1")
    thr2 = fp32_threshold2(thr)
    rng = CvRNG()
    niters = max(iterations_count, 1)
    best, best_mask, it = 0, None, 0
    while it < niters:
        idx = draw_subset(rng, n)
        info["samples"].append(idx)
        ok, rv, tv = cv2.solvePnP(P32[list(idx)], uv32[list(idx)], K, dist, flags=cv2.SOLVEPNP_EPNP)
        c = -1
        if ok:
            mask = fp32_errors(P32, uv32, K, dist, rv, tv) <= thr2
            c = int(mask.sum())
            if c > max(best, MODEL_POINTS - 1):
                best, best_mask, info["winner"] = c, mask, it
                niters = update_num_iters(confidence, (n - c) / n, MODEL_POINTS, niters)
        info["counts"].append(c)
        it += 1
    info["iterations"] = it
    if best_mask is None:
        return False, None, None, np.zeros(0, np.int64), info
    inl = np.nonzero(best_mask)[0]
    ok, rv, tv = cv2.solvePnP(P32[inl].astype(np.float64), uv32[inl].astype(np.float64), K, dist, flags=cv2.SOLVEPNP_EPNP)
    return bool(ok), rv, tv, inl, info
