"""CPU checks of the EPnP referee (tests/epnp_reference.py) against OpenCV's solvePnP(EPNP) fixtures
(tests/golden/pnp_epnp_cases.npz, made by tests/golden/make_epnp.py), its five-index sampler, the argument checks of opb_epnp /
opb_ransac_epnp (they fail before any CUDA call), the method option's validation, and the new symbols declared, bound and
exported."""
import ctypes as C
import itertools
import os

import numpy as np
import pytest

from onepose_b200 import _lib, pnp
from tests import epnp_reference as E
from tests import pnp_reference as ref
from tests.golden_util import GOLDEN_DIR

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "onepose_b200.h")


def _fixture():
    return dict(np.load(os.path.join(GOLDEN_DIR, "pnp_epnp_cases.npz"), allow_pickle=False))


def test_reference_equals_cv2_on_noise_free_generic_sets():
    """Noise-free generic sets of 5 or more pairs, in metres and millimetres: the restatement, OpenCV and the ground truth
    agree to 1e-9 (OpenCV reaches the ground truth to ~1e-12 there)."""
    g = _fixture()
    checked = 0
    for i, tag in enumerate(str(t) for t in g["p_tags"]):
        if not (tag.startswith("generic") and "noise0.0" in tag) or "_n4_" in tag:
            continue
        r = E.epnp(g[f"p{i}_K"], g[f"p{i}_uv"], g[f"p{i}_P"])
        gt, cv = g[f"p{i}_gt"], g[f"p{i}_cv"]
        assert ref.pose_error(r["R"], r["t"], gt[:, :3], gt[:, 3]) <= 1e-9, tag
        assert ref.pose_error(r["R"], r["t"], cv[:, :3], cv[:, 3]) <= 1e-9, tag
        assert np.allclose(r["alphas"].sum(1), 1.0) and np.allclose(r["alphas"] @ r["cw"], g[f"p{i}_P"], atol=1e-9 * np.abs(g[f"p{i}_P"]).max())
        checked += 1
    assert checked == 12


def test_reference_stages_are_consistent():
    g = _fixture()
    i = [str(t) for t in g["p_tags"]].index("generic_n50_noise0.0_m")
    K, uv, P, gt = g[f"p{i}_K"], g[f"p{i}_uv"], g[f"p{i}_P"], g[f"p{i}_gt"]
    r = E.epnp(K, uv, P)
    # the true control points' camera coordinates are in M's null space
    cc = r["cw"] @ gt[:, :3].T + gt[:, 3]
    x = cc.reshape(12)
    assert np.linalg.norm(r["MtM"] @ x) <= 1e-9 * np.linalg.norm(r["MtM"]) * np.linalg.norm(x)
    # rho is reproduced by the refined betas of the chosen candidate
    pr = E._products(r["betas"][r["best"]])
    np.testing.assert_allclose(r["L"] @ pr, r["rho"], rtol=1e-9)
    assert min(r["errors"]) <= 1e-9


def test_reference_equals_cv2_on_noisy_sets_up_to_the_axis_signs():
    """On noisy data EPnP's algebraic least squares depends on the control points, so the sign each principal axis is taken
    with changes the answer; OpenCV takes the signs its SVD returns, this project the largest-magnitude-component-positive
    rule.  With one of the eight sign choices the restatement equals cv2's pose to 1e-12 on every noisy generic set of 6 to
    1000 pairs, but one: 6 pairs at 2 px, where no choice comes within 5e-2 (named and printed here; cause unknown)."""
    g = _fixture()
    for i, tag in enumerate(str(t) for t in g["p_tags"]):
        if not tag.startswith("generic") or "noise0.0" in tag or any(f"_n{n}_" in tag for n in (4, 5)):
            continue
        K, uv, P, cv = (g[f"p{i}_{k}"] for k in ("K", "uv", "P", "cv"))
        d = []
        for s in itertools.product((1.0, -1.0), repeat=3):
            r = E.epnp(K, uv, P, s)
            d.append(ref.pose_error(r["R"], r["t"], cv[:, :3], cv[:, 3]))
        if tag.startswith("generic_n6_noise2.0"):
            print(f"{tag}: closest sign choice {min(d):.2e} from cv2")
            assert min(d) > 1e-2
            continue
        assert min(d) <= 1e-12, (tag, d)


def test_planar_sets_reach_ground_truth_and_four_point_sets_are_recorded():
    """Noise-free planar sets (the flat axis's control point at full length along the normal) reach the ground truth to 1e-10,
    as cv2 does on these sets; an exactly planar set in a general orientation as well.  Noise-free 4-pair sets are printed only:
    EPnP on 4 points is poor in both implementations (DESIGN 5.4)."""
    g = _fixture()
    for i, tag in enumerate(str(t) for t in g["p_tags"]):
        if not (tag.startswith("planar") or ("_n4_" in tag and "noise0.0" in tag)):
            continue
        K, uv, P, gt, cv = (g[f"p{i}_{k}"] for k in ("K", "uv", "P", "gt", "cv"))
        r = E.epnp(K, uv, P)
        mine = ref.pose_error(r["R"], r["t"], gt[:, :3], gt[:, 3])
        theirs = ref.pose_error(cv[:, :3], cv[:, 3], gt[:, :3], gt[:, 3])
        print(f"{tag}: restatement vs ground truth {mine:.2e}, OpenCV vs ground truth {theirs:.2e}")
        if tag.startswith("planar"):
            assert r["planar"] and mine <= 1e-10, (tag, mine)
            Rw = ref._rodrigues(np.array([0.3, -0.7, 0.2]))          # the same plane in a general orientation
            r = E.epnp(K, uv, P @ Rw.T)
            assert r["planar"]
            assert ref.pose_error(r["R"], r["t"], gt[:, :3] @ Rw.T, gt[:, 3]) <= 1e-10, tag


def test_degenerate_sets_have_no_control_points():
    P = np.tile([[0.01, 0.02, 0.03]], (8, 1))
    assert E.control_points(P)[0] is None
    assert E.control_points(np.linspace(0, 1, 8)[:, None] * [[0.1, 0.2, 0.3]])[0] is None


def test_cv2_ransac_fits_a_four_pair_scene():
    """A five-point sample cannot be drawn from 4 pairs, yet solvePnPRansac(EPNP) returns a pose with all 4 as inliers: it
    switches to a 4-point (P3P) model there, which opb_ransac_epnp follows."""
    g = _fixture()
    i = [str(t) for t in g["r_tags"]].index("four")
    assert len(g[f"r{i}_uv"]) == 4 and sorted(g[f"r{i}_inliers"].tolist()) == [0, 1, 2, 3]


def test_sample_indices5_are_distinct_and_extend_the_three_index_draw():
    for n in (5, 6, 37, 1000):
        for b in (0, 1, 70000):
            for h in range(200):
                idx = E.sample_indices5(12345, b, h, n)
                assert len(set(idx)) == 5 and all(0 <= i < n for i in idx), (n, b, h, idx)
                assert idx[:3] == ref.sample_indices(12345, b, h, n)


def test_count_inliers_has_no_depth_test():
    K = np.array([[600.0, 0, 256], [0, 600.0, 256], [0, 0, 1]])
    pose = np.concatenate([np.eye(3), [[0], [0], [1.0]]], 1)
    P = np.array([[0.1, 0.0, 0.0], [-0.1, 0.0, -2.0], [0, 0, 0]])    # the second is behind the camera, at the same pixel
    uv = np.array([[316.0, 256], [316.0, 256], [261.0, 256]])
    inl, border = E.count_inliers(pose, K, uv, P, 5.0)
    assert inl.tolist() == [True, True, True] and border.tolist() == [False, False, True]


def test_epnp_entry_points_reject_bad_arguments():
    lib = _lib.load()
    buf = C.c_void_p(16)     # never dereferenced: every call below fails its argument check first

    def epnp(K=buf, p2=buf, p3=buf, off=buf, B=2, pose=buf, status=buf):
        return lib.opb_epnp(K, p2, p3, off, B, pose, status, None)

    for kw in (dict(K=None), dict(p2=None), dict(p3=None), dict(off=None), dict(pose=None), dict(status=None), dict(B=0), dict(B=-3)):
        assert epnp(**kw) == -1, kw

    def ransac(K=buf, p2=buf, p3=buf, off=buf, B=2, H=64, thr=5.0, ws=buf, pose=buf, mask=buf, cnt=buf):
        return lib.opb_ransac_epnp(K, p2, p3, off, B, H, thr, 0, ws, pose, mask, cnt, None)

    for kw in (dict(K=None), dict(p2=None), dict(p3=None), dict(off=None), dict(ws=None), dict(pose=None), dict(mask=None),
               dict(cnt=None), dict(B=0), dict(H=0), dict(H=65535 * 128 + 1), dict(thr=0.0), dict(thr=float("nan")), dict(thr=-1.0),
               dict(thr=-float("inf"))):
        assert ransac(**kw) == -1, kw


def test_method_option_is_checked_and_defaults_kept():
    assert pnp._hypotheses("p3p", None) == pnp.DEFAULT_HYPOTHESES == 4096
    assert pnp._hypotheses("epnp", None) == pnp.EPNP_HYPOTHESES == 10000
    assert pnp._hypotheses("epnp", 7) == 7
    with pytest.raises(ValueError):
        pnp._hypotheses("EPnP", None)
    import inspect
    for fn in (pnp.ransac_pnp_batch, pnp.poses_from_matches, pnp.poses_from_matches_objects, pnp.ransac_PnP):
        assert inspect.signature(fn).parameters["method"].default == "p3p", fn.__name__


def test_new_symbols_declared_bound_and_exported():
    header = open(HEADER).read()
    lib = _lib.load()
    for name in ("opb_epnp", "opb_ransac_epnp"):
        assert f"int {name}(" in header and name in _lib.SYMBOLS
        assert getattr(lib, name).restype is C.c_int
