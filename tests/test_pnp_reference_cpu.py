"""CPU checks of the references the GPU RANSAC-PnP tests rely on (tests/pnp_reference.py) -- the referee is checked first:
p3p_all recovers planted poses on generic, planar, symmetric, near-symmetric and far scenes; refine_lsq stops at a stationary
point; the sampler never repeats an index.  Also the argument checks of opb_ransac_pnp, which run before any CUDA call."""
import ctypes as C

import numpy as np
import pytest

from onepose_b200 import _lib
from tests import pnp_reference as ref


def _rotation(rs):
    w = rs.randn(3)
    return ref._rodrigues(w / np.linalg.norm(w) * rs.uniform(0.1, 3.0))


def _check_recovers(P, R, t, tol=1e-10):
    X = P @ R.T + t
    j = X / np.linalg.norm(X, axis=1, keepdims=True)
    sols = ref.p3p_all(P, j)
    assert 1 <= len(sols) <= 4, len(sols)
    err = min(ref.pose_error(s["R"], s["t"], R, t) for s in sols)
    assert err <= tol, (err, [s["cond"] for s in sols])
    for s in sols:                                        # every solution is a rotation that maps P onto the three rays
        assert np.allclose(s["R"] @ s["R"].T, np.eye(3), atol=1e-12) and np.linalg.det(s["R"]) > 0
        Y = P @ s["R"].T + s["t"]
        assert np.allclose(np.cross(Y, j), 0, atol=1e-9 * np.max(np.abs(Y))) and np.all(Y[:, 2] > 0)
    return sols


@pytest.mark.parametrize("scale", [1.0, 1000.0])
def test_p3p_all_recovers_generic_and_planar_scenes(scale):
    rs = np.random.RandomState(1)
    done = 0
    while done < 300:
        R = _rotation(rs)
        t = np.array([0.03 * rs.randn(), 0.03 * rs.randn(), 0.5 + 0.3 * rs.rand()]) * scale
        P = 0.05 * rs.randn(3, 3) * scale
        if done % 2:
            P[:, 2] = 0.0                                # planar object
        X = P @ R.T + t
        if np.any(X[:, 2] <= 0.1 * scale) or ref.min_angle_deg(P) < 10:
            continue
        _check_recovers(P, R, t)
        done += 1


@pytest.mark.parametrize("offset_mm", [0.0, 1e-3, 0.1, 5.0])
@pytest.mark.parametrize("shape", ["equilateral", "isosceles"])
def test_p3p_all_recovers_symmetric_triangles(shape, offset_mm):
    """A 50 mm triangle 600 mm in front of the camera, seen from (or near) its symmetry plane: Grunert's linear back-substitution
    is singular exactly here; the reference must not be."""
    L = 0.05
    apex = L * np.sqrt(3) / 2 if shape == "equilateral" else 0.7 * L
    P = np.array([[-L / 2, 0, 0], [L / 2, 0, 0], [0, apex, 0]])
    P -= P.mean(0)
    for R in (np.eye(3), ref._rodrigues(np.array([0.0, 0.3, 0.0]))):   # head-on, and tilted about the symmetry axis
        sols = _check_recovers(P, R, np.array([offset_mm * 1e-3, 0.0, 0.6]))
        if offset_mm == 0.0 and shape == "equilateral" and np.array_equal(R, np.eye(3)):
            assert len(sols) == 4                         # the true pose, two mirror-like poses sharing a depth, and one more
            best = min(sols, key=lambda s: ref.pose_error(s["R"], s["t"], R, np.array([0, 0, 0.6])))
            assert best["cond"] < 3.0                     # ~[[1,1,0],[1,0,1],[0,1,1]]: condition number 2


def test_p3p_all_recovers_far_narrow_scenes():
    """A 10 cm object 3-8 m away (a field of view of ~1 degree): the rays are nearly parallel, the root cluster is tight."""
    rs = np.random.RandomState(2)
    done = 0
    while done < 200:
        R = _rotation(rs)
        t = np.array([0.05 * rs.randn(), 0.05 * rs.randn(), rs.uniform(3.0, 8.0)])
        P = 0.05 * rs.randn(3, 3)
        if ref.min_angle_deg(P) < 20:
            continue
        X = P @ R.T + t
        j = X / np.linalg.norm(X, axis=1, keepdims=True)
        sols = ref.p3p_all(P, j)
        true = min(sols, key=lambda s: ref.pose_error(s["R"], s["t"], R, t))
        # the depths' sensitivity grows with the distance; the data are exact to rounding, so the pose is exact to cond * eps
        assert ref.pose_error(true["R"], true["t"], R, t) <= max(1e-10, 1e-15 * true["cond"]), true["cond"]
        done += 1


def test_refine_lsq_reaches_a_stationary_point():
    rs = np.random.RandomState(3)
    for seed in range(10):
        n = 50
        R = _rotation(rs)
        t = np.array([0.02, -0.01, 0.6])
        P = 0.05 * rs.randn(n, 3)
        K = np.array([[620.0, 0, 250], [0, 610.0, 260], [0, 0, 1]])
        X = P @ R.T + t
        uv = X[:, :2] / X[:, 2:] * [K[0, 0], K[1, 1]] + K[:2, 2] + rs.randn(n, 2)
        start = np.concatenate([ref._rodrigues(0.01 * rs.randn(3)) @ R, (t + 0.005 * rs.randn(3))[:, None]], 1)
        pose, res = ref.refine_lsq(start, K, uv, P)
        assert res.success
        # the gradient of the cost vanishes: J^T r is tiny relative to |J| |r|
        g = res.jac.T @ res.fun
        assert np.linalg.norm(g) <= 1e-9 * np.linalg.norm(res.jac) * np.linalg.norm(res.fun), np.linalg.norm(g)
        # and nothing nearby is lower
        c0 = np.sum(ref.reprojection_residuals(pose, K, uv, P) ** 2)
        for _ in range(20):
            d = np.concatenate([ref._rodrigues(1e-6 * rs.randn(3)) @ pose[:, :3], (pose[:, 3] + 1e-7 * rs.randn(3))[:, None]], 1)
            assert np.sum(ref.reprojection_residuals(d, K, uv, P) ** 2) >= c0 * (1 - 1e-12)
        np.testing.assert_allclose(pose[:, :3] @ pose[:, :3].T, np.eye(3), atol=1e-12)


def test_sample_indices_are_distinct_and_in_range():
    for n in (3, 4, 5, 37, 1000):
        for b in (0, 1, 70000):
            for h in range(200):
                idx = ref.sample_indices(12345, b, h, n)
                assert len(set(idx)) == 3 and all(0 <= i < n for i in idx), (n, b, h, idx)
    assert ref.sample_indices(0, 0, 0, 10) != ref.sample_indices(0, 1, 0, 10) or ref.sample_indices(0, 0, 1, 10) != ref.sample_indices(0, 1, 1, 10)


def test_classify_marks_threshold_points_as_border():
    K = np.array([[600.0, 0, 256], [0, 600.0, 256], [0, 0, 1]])
    pose = np.concatenate([np.eye(3), [[0], [0], [1.0]]], 1)
    P = np.array([[0, 0, 0], [0, 0, 0], [0, 0, 0], [0, 0, -2.0]])
    uv = np.array([[256 + 5.0, 256], [256 + 4.0, 256], [256 + 6.0, 256], [256, 256]])
    inl, border = ref.classify(pose, K, uv, P, 5.0)
    assert inl.tolist() == [False, True, False, False]
    assert border.tolist() == [True, False, False, False]


def test_ransac_pnp_rejects_bad_arguments():
    lib = _lib.load()
    buf = C.c_void_p(16)     # never dereferenced: every call below fails its argument check first

    def call(K=buf, p2=buf, p3=buf, off=buf, B=2, H=64, thr=5.0, ws=buf, pose=buf, mask=buf, cnt=buf):
        return lib.opb_ransac_pnp(K, p2, p3, off, B, H, thr, 0, ws, pose, mask, cnt, None)

    for kw in (dict(K=None), dict(p2=None), dict(p3=None), dict(off=None), dict(ws=None), dict(pose=None), dict(mask=None),
               dict(cnt=None), dict(B=0), dict(B=-1), dict(H=0), dict(H=-5), dict(H=65535 * 128 + 1), dict(H=(1 << 31) - 1),
               dict(thr=0.0), dict(thr=-1.0), dict(thr=float("nan")), dict(thr=-float("inf"))):
        assert call(**kw) == -1, kw
