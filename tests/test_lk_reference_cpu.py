"""tests/lk_reference.py against live cv2.calcOpticalFlowPyrLK / buildOpticalFlowPyramid (OpenCV 4.13): the pyramids and
derivatives bit for bit, and status, points and err bit for bit on seeded textured scenes (affine and perspective motion,
points near and past the borders, a flat region that fails the eigenvalue test, large motion that loses points) for every
window of 3 / 7 / 15 / 21 / 31 and max_level 0 .. 4."""
import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")

from tests import lk_reference as L  # noqa: E402
from tests.flow_scenes import lk_scene  # noqa: E402


@pytest.mark.parametrize("win", [(3, 3), (7, 7), (15, 15), (21, 21), (31, 31), (9, 13)])
@pytest.mark.parametrize("max_level", [0, 1, 2, 3, 4])
def test_pyramid_bit_equal(win, max_level):
    img, _, _ = lk_scene(7, 150, 190, "affine")
    P, dP = L.build_pyramid(img, win, max_level)
    n, pyr = cv2.buildOpticalFlowPyramid(img, win, max_level, withDerivatives=True)
    assert n == len(P) - 1
    for level in range(n + 1):
        np.testing.assert_array_equal(pyr[2 * level], P[level])
        np.testing.assert_array_equal(pyr[2 * level + 1], dP[level])


@pytest.mark.parametrize("win", [(3, 3), (7, 7), (15, 15), (21, 21), (31, 31), (5, 11)])
@pytest.mark.parametrize("max_level", [0, 1, 2, 3, 4])
@pytest.mark.parametrize("motion", ["affine", "perspective", "large"])
def test_lk_bit_equal(win, max_level, motion):
    img, nxt, pts = lk_scene(3 + max_level, 110, 140, motion)
    crit = (3, 10, 0.03) if max_level % 2 else (3, 30, 0.01)
    a, s, e = L.calc_optical_flow_pyr_lk(img, nxt, pts, win, max_level, crit)
    b, cs, ce = cv2.calcOpticalFlowPyrLK(img, nxt, pts[:, None], None, winSize=win, maxLevel=max_level, criteria=crit)
    cs, b, ce = cs[:, 0], b[:, 0], ce[:, 0]
    np.testing.assert_array_equal(s, cs)
    m = cs == 1
    assert 0 < m.sum() < len(m)
    np.testing.assert_array_equal(a[m], b[m])
    np.testing.assert_array_equal(e[m], ce[m])


@pytest.mark.parametrize("crit", [(1, 1, 0), (1, 100, 0), (2, 0, 0.0), (2, 0, 0.5), (3, 5, 20.0)])
def test_lk_criteria(crit):
    img, nxt, pts = lk_scene(9, 90, 120, "perspective")
    a, s, e = L.calc_optical_flow_pyr_lk(img, nxt, pts, (15, 15), 2, crit)
    b, cs, ce = cv2.calcOpticalFlowPyrLK(img, nxt, pts[:, None], None, winSize=(15, 15), maxLevel=2, criteria=crit)
    m = cs[:, 0] == 1
    np.testing.assert_array_equal(s, cs[:, 0])
    np.testing.assert_array_equal(a[m], b[:, 0][m])
    np.testing.assert_array_equal(e[m], ce[:, 0][m])


def test_golden_matches_model():
    """The GPU goldens are what the model computes."""
    import os
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", "pnp_flow_cases.npz"))
    for i in range(6):
        p = z[f"lk{i}_params"]
        win, lev, crit = (int(p[0]), int(p[1])), int(p[2]), (int(p[3]), int(p[4]), float(p[5]))
        a, s, e = L.calc_optical_flow_pyr_lk(z[f"lk{i}_prev"], z[f"lk{i}_next"], z[f"lk{i}_pts"], win, lev, crit)
        m = z[f"lk{i}_status"] == 1
        np.testing.assert_array_equal(s, z[f"lk{i}_status"])
        np.testing.assert_array_equal(a[m], z[f"lk{i}_next_pts"][m])
        np.testing.assert_array_equal(e[m], z[f"lk{i}_err"][m])
