"""The numpy restatement of cv2.estimateAffinePartial2D (tests/affine_ransac_reference.py) against OpenCV itself.

Bars: the inlier mask equal everywhere; at refineIters=0 the affine bit-equal; with refinement the LM port within 1e-10
relative of cv2's (OpenCV sums J^T J and J^T r in its own order; both solve by the same eigen decomposition; the measured
maximum is printed).  Noise-free fits are held to the same bar: the refinement stops there on the largest residual, as cv2
does, before accepting a step turns on the summation order."""
import itertools

import numpy as np
import pytest

from tests import affine_ransac_reference as A

cv2 = pytest.importorskip("cv2")

REFINE_RTOL = 1e-10
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


def _check(f, t, thr, conf, ri, max_iters=2000):
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
            _worst["rel"] = max(_worst["rel"], rel)
            assert rel <= REFINE_RTOL, rel
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
            _check(ff, tt, 3.0, 0.99, ri)
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


# ---- the refinement's schedule and the loop across the domain cv2 accepts ----

REFINE_STEPS = (1, 2, 3, 5, 10, 50)
SHIFTS = (0.0, 1e3, 1e4, 1e5, 1e6)


def shifted(seed, n, frac, shift):
    """planted() with both point sets moved by (shift, shift): the normal equations' condition grows with shift^2."""
    f, t = planted(seed, n, frac, 1.0)
    return f + shift, t + shift


@pytest.mark.parametrize("shift", SHIFTS)
@pytest.mark.parametrize("ri", REFINE_STEPS)
def test_refinement_schedule_equals_cv2(ri, shift):
    """lm_refine against cv2 after 1 to 50 iterations.  Any accepted damped steps converge to the same least-squares optimum, so
    only the early iterations tell schedules apart: at refineIters=1 cv2's result is one step at lambda = 1, at 2 the second step
    is Gauss-Newton (lambda = 0).  At shifts of 1e5 and 1e6 cv2::solve drops the smallest eigenvalues of J^T J + lambda D and the
    translation stops moving far from the optimum; the restatement drops the same ones."""
    for seed in (41, 42, 43):
        f, t = shifted(seed, 300, 0.5, shift)
        _check(f, t, 3.0, 0.99, ri)


def sub_unit(seed, n=200):
    """n pairs with from in [0, 0.05]^2 and to a random similarity of them plus N(0, 2e-8) noise: after one iteration every
    residual is below FLT_EPSILON while the squared error is still above FLT_EPSILON^2."""
    r = np.random.default_rng(seed)
    f = r.uniform(0, 0.05, (n, 2))
    a, s = r.uniform(-3, 3), r.uniform(0.3, 3)
    R = s * np.array([[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]])
    t = f @ R.T + r.uniform(-0.05, 0.05, 2) + r.normal(0, 2e-8, (n, 2))
    return f.astype(np.float32), t.astype(np.float32)


@pytest.mark.parametrize("ri", (1, 2, 3, 10))
def test_refinement_stops_on_the_largest_residual(ri):
    """cv2's LMSolver stops once every residual of the kept model is below FLT_EPSILON, not on S < FLT_EPSILON^2.  On these
    sub-unit scenes the two rules part after the first iteration (the S rule takes one or two more and ends up to 5.7e-6
    off cv2)."""
    parted = 0
    for seed in (1, 3, 10, 13):
        f, t = sub_unit(seed)
        H, info = _check(f, t, 3.0, 0.99, ri)
        H1, m, _ = A.estimate_affine_partial_2d(f, t, 3.0, 2000, 0.99, 1)
        x = np.array([H1[0, 0], H1[1, 0], H1[0, 2], H1[1, 2]])
        r = A._residuals(x, f[m > 0], t[m > 0])
        parted += np.abs(r).max() < A.FLT_EPSILON <= float(r @ r) ** 0.5
    assert parted == 4


def test_refinement_schedule_distinguishes_the_early_iterations():
    """The probe behind the schedule: cv2's first iteration is one solve with J^T J's diagonal doubled (lambda = 1, not 1e-3),
    and its second a plain Gauss-Newton step (lambda = 0) from there, which lands on the optimum that later iterations keep."""
    f, t = planted(41, 300, 0.5, 1.0)
    f32, t32 = f.astype(np.float32), t.astype(np.float32)
    H0, m, _ = A.estimate_affine_partial_2d(f32, t32, 3.0, 2000, 0.99, 0)
    inl = np.nonzero(m)[0]

    def step(x, lam):
        JtJ, Jtr, _ = A._normal(x, f32[inl], t32[inl])
        return x - A.eig_solve(JtJ + lam * np.diag(np.diag(JtJ)), Jtr)

    def affine(x):
        return np.array([[x[0], -x[1], x[2]], [x[1], x[0], x[3]]])
    x1 = step(np.array([H0[0, 0], H0[1, 0], H0[0, 2], H0[1, 2]]), 1.0)
    x2 = step(x1, 0.0)
    H = {ri: cv2.estimateAffinePartial2D(f32, t32, ransacReprojThreshold=3, refineIters=ri)[0] for ri in (1, 2, 3, 10)}
    assert np.abs(H[1] - affine(x1)).max() <= 1e-13 * np.abs(H[1]).max()
    assert np.abs(H[2] - affine(x2)).max() <= 1e-13 * np.abs(H[2]).max()
    assert np.abs(H[2] - H[1]).max() > 1e-3 * np.abs(H[1]).max() and H[3].tobytes() == H[2].tobytes() == H[10].tobytes()


def test_eigen_solve_and_jacobi():
    r = np.random.default_rng(5)
    for _ in range(50):
        B = r.normal(size=(4, 4)) * r.uniform(0.1, 1e3, 4)
        M = B @ B.T + np.eye(4)
        w, V = A.jacobi(M)
        assert list(w) == sorted(w, reverse=True)
        np.testing.assert_allclose(V.T @ np.diag(w) @ V, M, rtol=1e-12, atol=1e-12 * np.abs(M).max())
        b = r.normal(size=4)
        np.testing.assert_allclose(A.eig_solve(M, b), np.linalg.solve(M, b), rtol=1e-8, atol=1e-12)
        np.testing.assert_allclose(A.eig_inverse_diagonal(M), np.diag(np.linalg.inv(M)), rtol=1e-8)
    M = np.diag([1e16, 1.0, 2.0, 3.0])               # 1, 2, 3 <= 2 DBL_EPSILON * trace = 4.44: dropped, as SVBkSb does
    assert A.eig_solve(M, np.ones(4)).tolist() == [1e-16, 0.0, 0.0, 0.0]
    assert A.eig_inverse_diagonal(np.diag([1e15, 1.0, 2.0, 3.0])).tolist() == [1e-15, 1.0, 0.5, 1 / 3]


THRESHOLDS = (0.0, 1e-30, -3.0, 3.0, 1e19, 1e20, 1e200)


@pytest.mark.parametrize("thr", THRESHOLDS)
def test_thresholds_across_the_domain(thr):
    """thr is squared before the fp32 rounding (-3 acts as 3; 0 and 1e-30 admit only exact fits); from 1e20 fp32(thr^2) is inf,
    every finite pair is an inlier and the refinement runs over all of them."""
    for seed, n, frac in ((51, 60, 0.4), (52, 300, 0.5)):
        f, t = planted(seed, n, frac, 0.0)
        for ri in (0, 10):
            _check(f, t, thr, 0.99, ri)


@pytest.mark.parametrize("max_iters", (0, 1, 2, 3, 31, 32, 33, 63, 64, 65))
def test_max_iters_across_the_wave(max_iters):
    """maxIters 0 runs one sample, as 1 does; 31 to 33 and 63 to 65 sit around the device's 32-sample waves."""
    for seed, n, frac in ((61, 200, 0.9), (62, 40, 0.7)):
        f, t = planted(seed, n, frac, 1.0)
        _, info = _check(f, t, 3.0, 0.999, 10, max_iters=max_iters)
        assert info["iterations"] <= max(max_iters, 1)


def test_budgets_past_int32_are_wrapped_by_cv2():
    """What cv2 does with size_t budgets above 2^31 - 1: it casts them to int.  maxIters 2^31 runs as 1 and 2^32 + 5 as 5;
    refineIters 2^31 and 2^32 + 1 refine for one iteration.  detect._check_params refuses them instead."""
    f, t = planted(63, 200, 0.8, 1.0)
    f, t = f.astype(np.float32), t.astype(np.float32)

    def run(**kw):
        H, m = cv2.estimateAffinePartial2D(f, t, ransacReprojThreshold=3, **kw)
        return H.tobytes() + m.tobytes()
    assert run(maxIters=2**31) == run(maxIters=1) and run(maxIters=2**32 + 5) == run(maxIters=5)
    assert run(refineIters=2**31) == run(refineIters=1) == run(refineIters=2**32 + 1)


@pytest.mark.parametrize("conf", (5e-324, 1e-300, 0.5, 1 - 2.0**-53))
def test_confidences_across_the_domain(conf):
    for seed, n, frac in ((71, 100, 0.5), (72, 30, 0.3)):
        f, t = planted(seed, n, frac, 1.0)
        _, info = _check(f, t, 3.0, conf, 10, max_iters=5000 if conf > 0.5 else 2000)
        assert info["iterations"] >= 1


@pytest.mark.parametrize("n", range(2, 9))
def test_small_problems(n):
    for seed, frac, thr, conf in ((81, 0.0, 3.0, 0.99), (82, 0.4, 3.0, 0.99), (83, 0.0, 0.0, 1 - 2.0**-53)):
        f, t = planted(seed + 10 * n, n, frac, 0.0)
        _check(f, t, thr, conf, 10)


@pytest.mark.parametrize("side", ("from", "to"))
def test_non_finite_rows(side):
    """NaN and +-inf rows in from or in to: their error is never <= a finite bound, and a sample that draws one gives a non-finite
    model that counts nothing; at threshold 1e20 an infinite error is inside the inf bound."""
    f, t = planted(91, 120, 0.3, 1.0)
    p = f if side == "from" else t
    p[[3, 50]] = np.nan
    p[7, 0], p[60, 1], p[99] = np.inf, -np.inf, (np.inf, -np.inf)
    for thr in (3.0, 1e20):
        for ri in (0, 10):
            _check(f, t, thr, 0.99, ri)
