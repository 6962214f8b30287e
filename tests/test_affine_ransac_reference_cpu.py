"""The numpy restatement of cv2.estimateAffinePartial2D (tests/affine_ransac_reference.py) against OpenCV itself.

Bars: the inlier mask equal everywhere; at refineIters=0 the affine bit-equal; with refinement the LM port within 1e-10
relative of cv2's (OpenCV sums J^T J and J^T r in its own order and solves by SVD; the measured maximum is printed).  On a
noise-free fit the squared error reaches the rounding floor of the fp32 points, where accepting or rejecting a step turns
on the summation order; there the bar is 1e-6 relative, well inside the points' own fp32 rounding."""
import itertools

import numpy as np
import pytest

from tests import affine_ransac_reference as A

cv2 = pytest.importorskip("cv2")

REFINE_RTOL = 1e-10
EXACT_FIT_RTOL = 1e-6
SIZES = (2, 3, 6, 50, 300, 1000, 4096)
OUTLIERS = (0.0, 0.3, 0.5, 0.9)


def planted(seed, n, frac, noise):
    """n pairs (from in a 640 x 480 view, to under a random similarity), a fraction replaced by uniform outliers."""
    r = np.random.default_rng(seed)
    f = r.uniform([0, 0], [640, 480], (n, 2))
    a, s = r.uniform(-3, 3), r.uniform(0.3, 3)
    R = s * np.array([[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]])
    t = f @ R.T + r.uniform(-300, 300, 2) + r.normal(0, noise, (n, 2))
    out = r.random(n) < frac
    t[out] = r.uniform(0, 1500, (int(out.sum()), 2))
    return f, t


def scenes():
    out = []
    for k, (n, frac) in enumerate(itertools.product(SIZES, OUTLIERS)):
        if n == 2 and frac > 0:
            continue
        out.append((700 + k, n, frac, (0.0, 1.0)[k % 2], (3.0, 6.0)[(k // 2) % 2], (0.9, 0.99, 0.999)[k % 3], (0, 10)[(k // 3) % 2]))
    return out


_worst = {"rel": 0.0}


def _check(f, t, thr, conf, ri, max_iters=2000, rtol=REFINE_RTOL):
    Hc, mc = cv2.estimateAffinePartial2D(np.asarray(f, np.float32), np.asarray(t, np.float32), ransacReprojThreshold=thr, maxIters=max_iters,
                                         confidence=conf, refineIters=ri)
    for minimal in ("cv2", "closed"):
        H, m, info = A.estimate_affine_partial_2d(f, t, thr, max_iters, conf, ri, minimal=minimal)
        assert (H is None) == (Hc is None)
        assert mc.dtype == np.uint8 and mc.shape == (len(f), 1) and np.array_equal(m, mc.reshape(-1))
        if H is None:
            continue
        if ri == 0 or len(f) == 2:
            assert H.tobytes() == Hc.tobytes()
        else:
            rel = float(np.abs(H - Hc).max() / np.abs(Hc).max())
            if rtol == REFINE_RTOL:
                _worst["rel"] = max(_worst["rel"], rel)
            assert rel <= rtol, rel
    return H, info


@pytest.mark.parametrize("seed,n,frac,noise,thr,conf,ri", scenes())
def test_restatement_equals_cv2(seed, n, frac, noise, thr, conf, ri):
    f, t = planted(seed, n, frac, noise)
    H, info = _check(f, t, thr, conf, ri)
    if n > 2:
        assert info["samples"] == A.subsets(n, info["iterations"])
        assert A.scan(info["counts"], n, conf, 2000) == (info["winner"], max(info["counts"]) if info["winner"] >= 0 else 0, info["iterations"])
    print(f"n={n} outliers={frac} noise={noise} thr={thr} conf={conf} refine={ri}: {info['iterations']} iterations, "
          f"winner {info['winner']}; max refined rel. difference so far {_worst['rel']:.2e}")


def test_degenerate_inputs():
    r = np.random.default_rng(3)
    f = r.uniform(0, 100, (40, 2))
    t = f * 1.5 + 7
    same = np.tile(f[:1], (40, 1))
    cases = [
        (same, t),                                                     # every from point coincides: no model
        (same, np.tile(t[:1], (40, 1))),                               # all identical
        (np.concatenate([same[:20], f[20:]]), t),                      # half of them coincide
        (np.repeat(f[:8], 5, axis=0), np.repeat(t[:8], 5, axis=0)),    # repeated pairs
        (np.stack([np.arange(40.0), 2 * np.arange(40.0) + 1], 1), t),  # collinear from points
        (f[:2], t[:2]),                                                # exactly 2 pairs: both inliers
        (f[:3], t[:3]),
    ]
    for ff, tt in cases:
        for ri in (0, 10):
            _check(ff, tt, 3.0, 0.99, ri, rtol=EXACT_FIT_RTOL)
    H, m, _ = A.estimate_affine_partial_2d(same, np.tile(t[:1], (40, 1)), minimal="closed")
    assert H is None and not m.any()
    H, m, _ = A.estimate_affine_partial_2d(f[:2], t[:2])
    assert H is not None and m.tolist() == [1, 1]
    H, m, _ = A.estimate_affine_partial_2d(f[:1], t[:1])
    assert H is None and m.tolist() == [0]


def test_closed_form_model_is_cv2s_bit_for_bit():
    r = np.random.default_rng(11)
    for _ in range(2000):
        f = r.uniform(-50, 2000, (2, 2)).astype(np.float32)
        t = r.uniform(-50, 2000, (2, 2)).astype(np.float32)
        assert A.run_kernel(f, t).tobytes() == A.cv2_kernel(f, t).tobytes()


def test_refinement_moves_the_model_and_float64_input_is_fp32():
    f, t = planted(5, 300, 0.3, 1.0)
    H0, _ = cv2.estimateAffinePartial2D(f, t, ransacReprojThreshold=6, refineIters=0)
    H10, _ = cv2.estimateAffinePartial2D(f, t, ransacReprojThreshold=6)
    assert np.abs(H10 - H0).max() > 1e-3
    H32, _ = cv2.estimateAffinePartial2D(f.astype(np.float32), t.astype(np.float32), ransacReprojThreshold=6)
    assert H32.tobytes() == H10.tobytes()


def test_two_point_scan_rules():
    assert A.scan([1, 2, 2, 1] + [0] * 100, 10, 0.99, 100)[0:2] == (1, 2)      # above max(best, 1); the first of a tie wins
    assert A.scan([1, 1, 1] + [0] * 100, 10, 0.99, 50) == (-1, 0, 50)
    assert A.scan([10] + [0] * 10, 10, 0.99, 100) == (0, 10, 1)               # every pair an inlier: the budget drops to 0
    assert A.subsets(3, 4) == [tuple(s) for s in A.subsets(3, 4)] and all(len(set(s)) == 2 for s in A.subsets(3, 500))
