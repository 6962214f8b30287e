"""The numpy restatement of OpenCV's EPnP-RANSAC loop (tests/opencv_ransac_reference.py) against cv2.solvePnPRansac itself,
and the facts about cv::RNG and RANSACUpdateNumIters the GPU mode (opb_ransac_epnp_cv, confidence=...) is built on."""
import itertools

import numpy as np
import pytest

from onepose_b200 import synthetic
from tests import opencv_ransac_reference as O

NOISE = (0.0, 1.0, 2.0)
OUTLIERS = (0.0, 0.3, 0.5, 0.7, 0.85)
SIZES = (5, 6, 20, 100, 1000)
CONFIDENCES = (0.9, 0.99, 0.999)
ITERS = (100, 10000)


def _scenes():
    """Every (n, outlier ratio) pair, with noise, confidence and iterationsCount cycled over them; the 10000-iteration runs of
    1000 pairs at >= 70 % outliers (10000 projections of 1000 points each) run at 100 iterations instead."""
    out = []
    for k, (n, f) in enumerate(itertools.product(SIZES, OUTLIERS)):
        it = ITERS[k % 2]
        if n == 1000 and f >= 0.7:
            it = 100
        out.append((300 + k, n, f, NOISE[k % 3], CONFIDENCES[(k // 2) % 3], it))
    return out


@pytest.mark.parametrize("seed,n,frac,noise,conf,iters", _scenes())
def test_restatement_equals_cv2(seed, n, frac, noise, conf, iters):
    cv2 = pytest.importorskip("cv2")
    K, uv, P, _ = synthetic.make_pnp_scene(seed, n, outlier_frac=frac, noise_px=noise)
    P = P * 1000                                          # as the reference's ransac_PnP(scale=1000) calls it
    ok, rv, tv, inl, info = O.solve_pnp_ransac(P, uv, K, None, 5.0, iters, conf)
    ok_cv, rv_cv, tv_cv, inl_cv = cv2.solvePnPRansac(P, uv, K, np.zeros((8, 1)), reprojectionError=5, iterationsCount=iters,
                                                     confidence=conf, flags=cv2.SOLVEPNP_EPNP)
    inl_cv = np.zeros(0, np.int64) if inl_cv is None else inl_cv.reshape(-1)
    assert ok == ok_cv
    assert inl.tolist() == inl_cv.tolist()
    if ok:
        assert rv.tobytes() == rv_cv.tobytes() and tv.tobytes() == tv_cv.tobytes()
    if n > 5:
        assert info["iterations"] == len(info["samples"]) == len(info["counts"]) <= iters
        assert info["samples"] == O.subsets(n, info["iterations"])
        assert O.scan(info["counts"], n, conf, iters) == (info["winner"], len(inl) if ok else 0, info["iterations"])
    print(f"n={n} outliers={frac} noise={noise} conf={conf} iters={iters}: {info['iterations']} iterations, "
          f"winner {info['winner']}, {len(inl)} inliers")


def test_cv2_refuses_confidence_0_and_1():
    """run() asserts 0 < confidence < 1; RANSACUpdateNumIters clamps, and the GPU mode follows the clamped formula."""
    cv2 = pytest.importorskip("cv2")
    K, uv, P, _ = synthetic.make_pnp_scene(11, 50, outlier_frac=0.3)
    for c in (0.0, 1.0):
        with pytest.raises(cv2.error):
            cv2.solvePnPRansac(P, uv, K, None, reprojectionError=5, iterationsCount=100, confidence=c, flags=cv2.SOLVEPNP_EPNP)


def test_mwc_is_a_multiplicative_lcg():
    """state_k = S_0 * MWC_A^k mod (MWC_A * 2^32 - 1) for every k.  The start state 2^64 - 1 and the first state after it lie
    above the modulus (their high word is not below MWC_A), so a jump-ahead must not take the residue's low word for the first
    draw; from the second state on the state is its own residue."""
    rng = O.CvRNG()
    s = (2 ** 64 - 1) % O.MWC_M
    assert 2 ** 64 - 1 >= O.MWC_M
    for k in range(1, 20001):
        rng.next()
        s = s * O.MWC_A % O.MWC_M
        if k == 1:
            assert rng.state == s + O.MWC_M and (rng.state & 0xFFFFFFFF) != s & 0xFFFFFFFF
        else:
            assert rng.state == s < O.MWC_M


def test_subsets_are_distinct_and_redraw_repeats():
    for n in (5, 6, 7, 100):
        for idx in O.subsets(n, 500):
            assert len(set(idx)) == 5 and all(0 <= i < n for i in idx)
    rng = O.CvRNG()
    raw = [rng.next() for _ in range(40)]
    first = O.subsets(6, 1)[0]
    draws = [r % 6 for r in raw]
    kept = []
    for d in draws:                                      # the first five distinct draws, in draw order
        if d not in kept:
            kept.append(d)
        if len(kept) == 5:
            break
    assert first == tuple(kept)


def test_update_num_iters_edges():
    assert O.update_num_iters(0.99, 0.5, 5, 10000) == 145
    assert O.update_num_iters(0.99, 0.8, 5, 10000) == 10000          # 0.2^5 is too small to lower the budget
    assert O.update_num_iters(0.0, 0.5, 5, 10000) == 0                # confidence 0: stop after the first improvement
    assert O.update_num_iters(1.0, 0.5, 5, 10000) == 10000            # confidence 1: the full budget ...
    assert O.update_num_iters(1.0, 0.0, 5, 10000) == 0                # ... except when every pair is an inlier
    assert O.update_num_iters(0.99, 0.5, 5, 100) == 100               # the budget never grows
    assert O.update_num_iters(1.7, -0.2, 5, 50) == 0                  # clamped to 1 and 0
    # the scan: strict improvement over max(best, 4); the earliest sample wins a tie; the loop exits at iter >= niters
    assert O.scan([4, 3, 6, 6, 7] + [0] * 100, 10, 0.99, 100) == (4, 7, 25)
    assert O.scan([4, 3, 6, 6, 7] + [0] * 100, 10, 0.0, 100) == (2, 6, 3)
    assert O.scan([6, 6, 6] + [0] * 100, 10, 0.99, 100)[0] == 0
    assert O.scan([-1] * 10, 10, 0.99, 10) == (-1, 0, 10)


def _pin(P, uv, K, thr, iters, conf):
    """The restatement equals cv2.solvePnPRansac(EPNP) on one scene: success, inlier list, pose bits, and the loop's own
    bookkeeping (samples, scan).  Returns (inliers, info)."""
    cv2 = pytest.importorskip("cv2")
    ok, rv, tv, inl, info = O.solve_pnp_ransac(P, uv, K, None, thr, iters, conf)
    ok_cv, rv_cv, tv_cv, inl_cv = cv2.solvePnPRansac(P, uv, K, np.zeros((8, 1)), reprojectionError=thr, iterationsCount=iters,
                                                     confidence=conf, flags=cv2.SOLVEPNP_EPNP)
    inl_cv = np.zeros(0, np.int64) if inl_cv is None else inl_cv.reshape(-1)
    assert ok == ok_cv
    assert inl.tolist() == inl_cv.tolist()
    if ok:
        assert rv.tobytes() == rv_cv.tobytes() and tv.tobytes() == tv_cv.tobytes()
    n = len(uv)
    if n > 5:
        assert info["iterations"] == len(info["samples"]) <= max(iters, 1)
        assert info["samples"] == O.subsets(n, info["iterations"])
        assert O.scan(info["counts"], n, conf, iters) == (info["winner"], len(inl) if ok else 0, info["iterations"])
    return inl, info


@pytest.mark.parametrize("thr", [0.1, 0.7, 3.3, 5.3, 5.7])
def test_threshold_is_rounded_to_fp32_before_it_is_squared(thr):
    """solvePnPRansac declares ``float reprojectionError``: the inlier bound is fp32(fp32(thr)^2), not fp32(thr^2).  At these
    thresholds the two differ by one ulp.  The boundary scene puts one pair at an exactly known fp32 error: one ulp below the
    lower bound and at it (inlier under both), at the upper bound (the rule decides), one ulp above it (outlier under both).
    The controls pass only if the probe's error is what the scene says it is."""
    cv2 = pytest.importorskip("cv2")
    t_first, t_late = O.fp32_threshold2(thr), np.float32(thr * thr)
    assert t_first != t_late
    lo, hi = min(t_first, t_late), max(t_first, t_late)
    probes = ((np.nextafter(lo, np.float32(0)), True), (lo, True), (hi, hi == t_first), (np.nextafter(hi, np.float32(np.inf)), False))
    for err, inlier in probes:
        K, uv, P = O.boundary_scene(err)
        P32, uv32 = P.astype(np.float32), uv.astype(np.float32)
        ok, rv, tv = cv2.solvePnP(P32[[9, 11, 4, 12, 7]], uv32[[9, 11, 4, 12, 7]], K, np.zeros((8, 1)), flags=cv2.SOLVEPNP_EPNP)
        e = O.fp32_errors(P32, uv32, K, np.zeros((8, 1)), rv, tv)
        assert e[0] == err and np.all(e[1:] < 1e-20), (err, e[0])      # the error model of the probe itself
        inl, info = _pin(P, uv, K, thr, 1, 0.99)
        assert info["samples"] == [(9, 11, 4, 12, 7)]
        assert (0 in inl.tolist()) == inlier and inl.tolist()[-12:] == list(range(1, 13)), (thr, err, inlier)


@pytest.mark.parametrize("thr", [0.05, 0.7, 1.0, 3.0, 5.3, 5.7, 8.0, 1e6, float("inf")])
def test_restatement_equals_cv2_at_thresholds(thr):
    for k, (n, frac, noise) in enumerate(((100, 0.4, 1.0), (60, 0.6, 0.5), (200, 0.3, 2.0))):
        K, uv, P, _ = synthetic.make_pnp_scene(1200 + k, n, outlier_frac=frac, noise_px=noise)
        inl, info = _pin(P * 1000, uv, K, thr, 2000 if thr < 1 else 10000, 0.99)
        if thr == float("inf"):
            assert len(inl) == n and info["iterations"] == 1          # every pair, and the first sample ends the loop
        print(f"thr={thr} n={n}: {info['iterations']} iterations, winner {info['winner']}, {len(inl)} inliers")


@pytest.mark.parametrize("iters", [0, 1, 2, 3])
def test_restatement_equals_cv2_at_tiny_budgets(iters):
    """iterationsCount = 0 runs one iteration in OpenCV (niters = max(iterationsCount, 1))."""
    for k, frac in enumerate((0.0, 0.5, 0.9)):
        K, uv, P, _ = synthetic.make_pnp_scene(1300 + k, 40, outlier_frac=frac, noise_px=1.0)
        inl, info = _pin(P * 1000, uv, K, 5.0, iters, 0.99)
        assert 1 <= info["iterations"] <= max(iters, 1)


@pytest.mark.parametrize("conf", [1e-300, 0.5, 1 - 2 ** -53])
def test_restatement_equals_cv2_at_confidence_edges(conf):
    for k, frac in enumerate((0.2, 0.6)):
        K, uv, P, _ = synthetic.make_pnp_scene(1400 + k, 80, outlier_frac=frac, noise_px=1.0)
        inl, info = _pin(P * 1000, uv, K, 5.0, 3000, conf)
        if conf == 1e-300:
            assert info["iterations"] == info["winner"] + 1                  # the first improvement ends the loop


@pytest.mark.parametrize("n", [5, 6, 7])
def test_restatement_equals_cv2_on_small_frames(n):
    for k, (frac, noise) in enumerate(((0.0, 0.0), (0.0, 1.0), (0.2, 1.0))):
        K, uv, P, _ = synthetic.make_pnp_scene(1500 + 10 * n + k, n, outlier_frac=frac, noise_px=noise)
        for thr in (1.0, 5.0):
            _pin(P * 1000, uv, K, thr, 100, 0.99)


def test_cv2_departures_the_device_refuses():
    """What cv2 accepts and the device entry points refuse or define otherwise: a negative threshold is squared (it acts as
    its absolute value), and iterationsCount = 0 runs one iteration."""
    cv2 = pytest.importorskip("cv2")
    K, uv, P, _ = synthetic.make_pnp_scene(1600, 60, outlier_frac=0.3, noise_px=1.0)
    P = P * 1000
    a = cv2.solvePnPRansac(P, uv, K, np.zeros((8, 1)), reprojectionError=-5, iterationsCount=500, confidence=0.99, flags=cv2.SOLVEPNP_EPNP)
    b = cv2.solvePnPRansac(P, uv, K, np.zeros((8, 1)), reprojectionError=5, iterationsCount=500, confidence=0.99, flags=cv2.SOLVEPNP_EPNP)
    assert a[0] and a[3].tolist() == b[3].tolist() and a[1].tobytes() == b[1].tobytes()


def test_cv2_reads_only_fx_fy_cx_cy():
    """EPnP and projectPoints ignore K's skew, its [1][0] entry and its last row, as the device's frame view does."""
    cv2 = pytest.importorskip("cv2")
    K, uv, P, _ = synthetic.make_pnp_scene(1650, 50, outlier_frac=0.0, noise_px=1.0)
    P = P * 1000
    K2 = K.copy()
    K2[0, 1], K2[1, 0], K2[2] = 3.5, -0.7, (0.3, -0.2, 7.0)
    a = cv2.solvePnP(P, uv, K, None, flags=cv2.SOLVEPNP_EPNP)
    b = cv2.solvePnP(P, uv, K2, None, flags=cv2.SOLVEPNP_EPNP)
    assert a[1].tobytes() == b[1].tobytes() and a[2].tobytes() == b[2].tobytes()
    assert cv2.projectPoints(P, a[1], a[2], K, None)[0].tobytes() == cv2.projectPoints(P, a[1], a[2], K2, None)[0].tobytes()
    r = cv2.solvePnPRansac(P, uv, K, None, reprojectionError=2, iterationsCount=200, flags=cv2.SOLVEPNP_EPNP)
    r2 = cv2.solvePnPRansac(P, uv, K2, None, reprojectionError=2, iterationsCount=200, flags=cv2.SOLVEPNP_EPNP)
    assert r[3].tolist() == r2[3].tolist() and r[1].tobytes() == r2[1].tobytes()
