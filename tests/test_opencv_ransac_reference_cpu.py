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
