"""tests/lk_reference.py against live cv2.calcOpticalFlowPyrLK / buildOpticalFlowPyramid (OpenCV 4.13): the pyramids and
derivatives bit for bit, and status, points and err bit for bit on seeded textured scenes (affine and perspective motion,
points near and past the borders, a flat region that fails the eigenvalue test, large motion that loses points) for every
window of 3 / 7 / 15 / 21 / 31 and max_level 0 .. 4.  On the cv2-free scenes of the GPU suite (flow_scenes.warp_scene), images
of 1 x 1 to 47 x 63, every min_eig_threshold it uses and the points on each pyramid level's edges, the positions of every
point are pinned too, status-0 points included."""
import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")

from tests import lk_reference as L  # noqa: E402
from tests import flow_scenes as FS  # noqa: E402
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


# ----------------------------------------------------------------------------- every row, on the GPU suite's cv2-free scenes
# tests/test_flow_domain_gpu.py compares the device with the model in every row, status 0 included; these pin the model to cv2
# there: the positions of every point (NaN equal to NaN), the status, and err where cv2 sets it (status 1).
SMALL_SIZES = [(1, 1), (1, 9), (9, 1), (2, 2), (3, 5), (4, 40), (5, 7), (9, 9), (12, 30), (16, 16), (20, 20), (31, 33), (33, 31),
               (47, 63)]
SMALL_WINS = [(3, 3), (5, 11), (15, 15), (31, 31)]


def _all_rows(prev, nxt, pts, win, lev, crit, min_eig=1e-4):
    a, s, e = L.calc_optical_flow_pyr_lk(prev, nxt, pts, win, lev, crit, min_eig)
    b, cs, ce = cv2.calcOpticalFlowPyrLK(prev, nxt, pts[:, None], None, winSize=win, maxLevel=lev, criteria=crit, minEigThreshold=min_eig)
    cs, b, ce = cs[:, 0], b[:, 0], ce[:, 0]
    np.testing.assert_array_equal(s, cs)
    np.testing.assert_array_equal(a, b)
    m = cs == 1
    np.testing.assert_array_equal(e[m], ce[m])
    assert not e[~m].any()
    return int(m.sum()), int((~m).sum())


@pytest.mark.parametrize("motion", ["affine", "large"])
@pytest.mark.parametrize("win,lev,crit,min_eig", [((15, 15), 2, (3, 10, 0.03), 1e-4), ((21, 21), 3, (3, 30, 0.01), 1e-2),
                                                  ((15, 15), 4, (1, 100, 0), 0.0), ((31, 31), 4, (2, 0, 20.0), 1e-3),
                                                  ((3, 29), 1, (1, 1, 0), 1e-3), ((29, 3), 0, (3, 5, 20.0), 1e-2)])
def test_lk_warp_scene_every_row(motion, win, lev, crit, min_eig):
    """warp_scene at 128 x 160 (and the benchmarked 512 x 512 for the tracker's parameters) with scene and border points."""
    h, w = (512, 512) if win == (15, 15) and lev == 2 else (128, 160)
    prev, nxt = FS.warp_scene(11 + lev, h, w, motion)
    pts = np.concatenate([FS.scene_points(11 + lev, h, w, 600), FS.border_points(h, w, win, lev)])
    with np.errstate(invalid="ignore"):
        n1, n0 = _all_rows(prev, nxt, pts, win, lev, crit, min_eig)
    assert n1 > 0 and n0 > 0


@pytest.mark.parametrize("min_eig", [0.0, 1e-4, 1e-3, 1e-2])
def test_lk_min_eig_every_row(min_eig):
    prev, nxt = FS.warp_scene(4, 96, 128)
    pts = FS.scene_points(4, 96, 128, 400)
    n1, n0 = _all_rows(prev, nxt, pts, (9, 13), 2, (3, 10, 0.03), min_eig)
    assert n1 > 0 and n0 > 0


@pytest.mark.parametrize("win", SMALL_WINS)
@pytest.mark.parametrize("lev", [0, 2, 4])
def test_lk_small_images_every_row(win, lev):
    """Images from 1 x 1 to 47 x 63, most of them smaller than the window: pyramids, derivatives and every row."""
    for h, w in SMALL_SIZES:
        prev, nxt = FS.warp_scene(h * 100 + w, h, w)
        P, dP = L.build_pyramid(prev, win, lev)
        n, pyr = cv2.buildOpticalFlowPyramid(prev, win, lev, withDerivatives=True)
        assert n == len(P) - 1, (h, w)
        for level in range(n + 1):
            np.testing.assert_array_equal(pyr[2 * level], P[level])
            np.testing.assert_array_equal(pyr[2 * level + 1], dP[level])
        pts = np.concatenate([FS.scene_points(h + w, h, w, 40, margin=3.0), FS.border_points(h, w, win, lev)])
        with np.errstate(invalid="ignore"):
            _all_rows(prev, nxt, pts, win, lev, (3, 10, 0.03))
