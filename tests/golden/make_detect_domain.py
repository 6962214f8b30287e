"""Generate the fixture of the detector's domain test (tests/test_detect_domain_gpu.py) on a machine with OpenCV:

    python tests/golden/make_detect_domain.py

Writes ``pnp_detect_domain_cases.npz``: cv2.estimateAffinePartial2D(from, to, RANSAC, ...) across the domain it accepts --
thresholds from 0 to 1e200, maxIters around the device's 32-sample waves, confidences from 5e-324 to 1 - 2^-53, 2 to 8 pairs,
NaN and +-inf rows in from and in to, refineIters 1 to 1000 near the origin and at coordinates shifted by 1e3 to 1e6, and
refineIters 1 to 10 on sub-unit fits where only the largest-residual stopping test agrees with cv2.
Per case ``c{i}_from`` / ``c{i}_to`` (fp32 [n, 2]), ``c{i}_thr``, ``c{i}_conf``, ``c{i}_max_iters``, ``c{i}_refine``, cv2's
``c{i}_ok``, ``c{i}_affine`` (zeros where cv2 returns None) and ``c{i}_mask``, and the restatement's
(tests/affine_ransac_reference.py) ``c{i}_iterations``, ``c{i}_winner``, ``c{i}_counts``, ``c{i}_samples`` and ``c{i}_models``
(every sample's unrefined model); ``c_tags`` names them.  The restatement's mask equals cv2's on every case, its unrefined
model bit for bit and its refined model to 1e-10 relative (asserted here).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))

from tests import affine_ransac_reference as A  # noqa: E402

REFINE_RTOL = 1e-10


def planted(seed, n, frac, noise=1.0, shift=0.0):
    """n pairs (from in a 640 x 480 view, to under a random similarity), a fraction replaced by uniform outliers, both point
    sets moved by (shift, shift)."""
    r = np.random.default_rng(seed)
    f = r.uniform([0, 0], [640, 480], (n, 2))
    a, s = r.uniform(-3, 3), r.uniform(0.3, 3)
    R = s * np.array([[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]])
    t = f @ R.T + r.uniform(-300, 300, 2) + r.normal(0, noise, (n, 2))
    out = r.random(n) < frac
    t[out] = r.uniform(0, 1500, (int(out.sum()), 2))
    return (f + shift).astype(np.float32), (t + shift).astype(np.float32)


def sub_unit(seed, n=200):
    """from in [0, 0.05]^2, to a similarity of them plus N(0, 2e-8) noise: every residual falls below FLT_EPSILON while the
    squared error is still above FLT_EPSILON^2, so only the refinement's residual stopping test ends the loop as cv2 does."""
    r = np.random.default_rng(seed)
    f = r.uniform(0, 0.05, (n, 2))
    a, s = r.uniform(-3, 3), r.uniform(0.3, 3)
    R = s * np.array([[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]])
    t = f @ R.T + r.uniform(-0.05, 0.05, 2) + r.normal(0, 2e-8, (n, 2))
    return f.astype(np.float32), t.astype(np.float32)


def non_finite(f, t, side):
    p = (f if side == "from" else t).copy()
    p[[3, 50]] = np.nan
    p[7, 0], p[60, 1], p[99] = np.inf, -np.inf, (np.inf, -np.inf)
    return (p, t) if side == "from" else (f, p)


def cases():
    """(tag, from, to, thr, conf, max_iters, refine)"""
    out = []
    for thr in (0.0, 1e-30, -3.0, 1e19, 1e20, 1e200):
        for seed, n, frac in ((1800, 60, 0.4), (1801, 300, 0.5)):
            out.append((f"thr{thr}_n{n}", *planted(seed, n, frac, 0.0), thr, 0.99, 2000, 10))
    for conf in (5e-324, 1e-300, 0.5, 1 - 2.0**-53):
        for seed, n, frac in ((1810, 100, 0.5), (1811, 30, 0.3)):
            out.append((f"conf{conf!r}_n{n}", *planted(seed, n, frac), 3.0, conf, 2000, 10))
    for it in (0, 1, 2, 3, 31, 32, 33, 63, 64, 65):
        out.append((f"iters{it}", *planted(1820, 200, 0.9), 3.0, 0.999, it, 10))
    for n in range(2, 9):
        out.append((f"n{n}_exact", *planted(1830 + n, n, 0.0, 0.0), 3.0, 0.99, 2000, 10))
        out.append((f"n{n}_outliers", *planted(1840 + n, n, 0.4, 1.0), 3.0, 0.99, 2000, 10))
    for n, seed in ((3, 1850), (4, 1854)):   # threshold 0, confidence 1 - 2^-53: no sample wins, all 3000 run
        out.append((f"n{n}_thr0", *planted(seed, n, 0.0, 1.0), 0.0, 1 - 2.0**-53, 3000, 10))
    for side in ("from", "to"):
        for thr in (3.0, 1e20):
            for ri in (0, 10):
                out.append((f"nonfinite_{side}_thr{thr}_ri{ri}", *non_finite(*planted(1860, 120, 0.3), side), thr, 0.99, 2000, ri))
    for shift in (0.0, 1e3, 1e4, 1e5, 1e6):
        for ri in (1, 2, 3, 1000):
            for seed in (1870, 1871):
                out.append((f"refine{ri}_shift{shift:g}_s{seed}", *planted(seed, 300, 0.5, 1.0, shift), 3.0, 0.99, 2000, ri))
    for ri in (1, 2, 3, 10):
        for seed in (3, 10):
            out.append((f"subunit{ri}_s{seed}", *sub_unit(seed), 3.0, 0.99, 2000, ri))
    return out


def main():
    import cv2
    res = {"cv2_version": np.array(cv2.__version__)}
    tags = []
    for i, (tag, f, t, thr, conf, it, ri) in enumerate(cases()):
        Hc, mc = cv2.estimateAffinePartial2D(f, t, ransacReprojThreshold=thr, maxIters=it, confidence=conf, refineIters=ri)
        H, m, info = A.estimate_affine_partial_2d(f, t, thr, it, conf, ri, minimal="closed")
        assert (H is None) == (Hc is None) and np.array_equal(m, mc.reshape(-1)), tag
        if H is not None:
            if ri == 0 or len(f) == 2:
                assert H.tobytes() == Hc.tobytes(), tag
            else:
                assert np.abs(H - Hc).max() <= REFINE_RTOL * np.abs(Hc).max(), tag
        k = len(info["samples"])
        res.update({f"c{i}_from": f, f"c{i}_to": t, f"c{i}_thr": np.float64(thr), f"c{i}_conf": np.float64(conf),
                    f"c{i}_max_iters": np.int64(it), f"c{i}_refine": np.int64(ri), f"c{i}_ok": np.bool_(Hc is not None),
                    f"c{i}_affine": Hc if Hc is not None else np.zeros((2, 3)), f"c{i}_mask": mc.reshape(-1),
                    f"c{i}_iterations": np.int64(info["iterations"]), f"c{i}_winner": np.int64(info["winner"]),
                    f"c{i}_counts": np.asarray(info["counts"], np.int32).reshape(k),
                    f"c{i}_samples": np.asarray(info["samples"], np.int32).reshape(k, 2),
                    f"c{i}_models": np.asarray(info["models"], np.float64).reshape(k, 2, 3)})
        tags.append(tag)
        print(tag, "iterations", info["iterations"], "winner", info["winner"], "inliers", int(m.sum()))
    res["c_tags"] = np.array(tags)
    np.savez_compressed(os.path.join(HERE, "pnp_detect_domain_cases.npz"), **res)
    print(len(tags), "cases")


if __name__ == "__main__":
    main()
