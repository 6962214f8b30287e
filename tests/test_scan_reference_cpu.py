"""The reference model of an annotated scan's processing (tests/scan_reference.py) and the package's host readers, without a GPU:
transforms3d's quat2mat, the pairing of ARposes rows and video frames, the skip rule's four bounds, and the two facts the
device colour crop rests on -- cv2 warps a colour image as it warps each channel plane, and cropping the colour frame then
turning the crop grey (the reference's order) differs from cropping the grey frame."""
import os

import cv2
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from onepose_b200 import scan
from tests import crop_reference as cr
from tests import grey_reference as G
from tests import scan_reference as sr
from tests.golden_util import GOLDEN_DIR


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(os.path.join(GOLDEN_DIR, "pnp_scan_cases.npz"), allow_pickle=False))


# ---- transforms3d ----

def test_quat2mat_is_scipys_rotation_on_unit_quaternions():
    q = Rotation.random(2000, random_state=3).as_quat()                    # x, y, z, w
    for x, y, z, w in q:
        want = Rotation.from_quat([x, y, z, w]).as_matrix()
        np.testing.assert_allclose(sr.quat2mat([w, x, y, z]), want, atol=2e-15, rtol=0)
        assert np.array_equal(scan.quat2mat([w, x, y, z]), sr.quat2mat([w, x, y, z]))


def test_quat2mat_on_non_unit_quaternions_is_the_formula_not_a_normalisation():
    rng = np.random.default_rng(4)
    for _ in range(2000):
        q = rng.normal(size=4) * np.exp(rng.uniform(-6, 6))
        w, x, y, z = q
        Nq = w * w + x * x + y * y + z * z
        s = 2.0 / Nq
        want = np.array([[1.0 - (y * y * s + z * z * s), x * y * s - w * z * s, x * z * s + w * y * s],
                         [x * y * s + w * z * s, 1.0 - (x * x * s + z * z * s), y * z * s - w * x * s],
                         [x * z * s - w * y * s, y * z * s + w * x * s, 1.0 - (x * x * s + y * y * s)]])
        got = sr.quat2mat(q)
        np.testing.assert_allclose(got, want, atol=1e-15, rtol=0)
        np.testing.assert_allclose(got, Rotation.from_quat([x, y, z, w]).as_matrix(), atol=2e-15, rtol=0)   # scipy normalises
        assert np.array_equal(scan.quat2mat(q), got)
    eps = np.finfo(np.float64).eps
    assert np.array_equal(sr.quat2mat([np.sqrt(eps) * 0.99, 0, 0, 0]), np.eye(3))                  # below eps: the identity
    assert np.array_equal(scan.quat2mat([0, 0, 0, 0]), np.eye(3))
    assert not np.array_equal(sr.quat2mat([0, 0, np.sqrt(eps) * 1.01, 0]), np.eye(3))


def test_compose_with_unit_zooms_is_R_t():
    R = Rotation.random(random_state=1).as_matrix()
    t = [0.1, -0.2, 0.3]
    A = sr.compose(t, R, np.ones(3))
    assert np.array_equal(A[:3, :3], R) and np.array_equal(A[:3, 3], t) and A[3].tolist() == [0, 0, 0, 1]
    assert np.array_equal(scan.compose(t, R), A)


# ---- readers ----

def test_readers_equal_the_reference_lines(golden, tmp_path):
    g = golden
    paths = {}
    for name in ("frames", "box", "arposes"):
        paths[name] = tmp_path / f"{name}.txt"
        paths[name].write_text(str(g[f"{name}_txt"]))
    K = scan.read_intrinsics(paths["frames"])
    fx, fy, cx, cy = sr.intrinsics(str(g["frames_txt"]).splitlines(keepends=True))
    assert np.array_equal(K, [[fx, 0, cx], [0, fy, cy], [0, 0, 1]]) and np.array_equal(K, g["K"])
    bbox3d, T_ow = scan.read_box(paths["box"])
    lines = str(g["box_txt"]).splitlines(keepends=True)
    assert np.array_equal(bbox3d, sr.get_bbox3d(lines)[0]) and np.array_equal(T_ow, sr.parse_box(lines))
    rows = scan.read_arposes(paths["arposes"])
    text = str(g["arposes_txt"])
    assert rows.shape == (len(g["keep"]), 8)
    data = [ln.strip() for ln in text.splitlines() if ln.strip() and not ln.strip().startswith("#")]
    assert np.array_equal(rows, [[float(e) for e in ln.split(",")] for ln in data])


def test_readers_refuse_malformed_files(tmp_path):
    p = tmp_path / "a.txt"
    p.write_text("1,2,3\n")
    with pytest.raises(ValueError, match="8 numbers"):
        scan.read_arposes(p)
    p.write_text("header\n1,2,3,4,5,6,7\n")
    with pytest.raises(ValueError, match="10 numbers"):
        scan.read_box(p)
    p.write_text("# only a comment\n")
    with pytest.raises(ValueError, match="at least 6"):
        scan.read_intrinsics(p)


def test_model_reproduces_the_golden(golden):
    g = golden
    saved, keep = sr.process_poses(g["K"], str(g["box_txt"]).splitlines(keepends=True), str(g["arposes_txt"]).splitlines(keepends=True))
    assert np.array_equal(keep, g["keep"]) and len(saved) == int(g["count"])
    for i in range(int(g["count"])):
        assert np.array_equal(saved[i][0], g["pose"][i]) and np.array_equal(saved[i][1], g["proj"][i]) and saved[i][2] == g["row"][i]
    v = g["proj"].reshape(-1)
    assert np.abs(v - np.rint(v)).min() >= 1e-6                       # truncation is not decided by the last bits
    assert keep.sum() < len(keep) and {k for k in keep} == {0, 1}


# ---- the pairing ----

def _rows_text(kinds):
    """ARposes text with one row per entry of kinds: 'in' (kept), 'far' (skipped), '#' (a comment) or '' (a blank line)."""
    lines = []
    for k in kinds:
        if k == "#":
            lines.append("# comment\n")
        elif k == "":
            lines.append("   \n")
        else:
            x = 0.0 if k == "in" else 10.0                            # 10 m to the side, the object projects far left of -1000
            lines.append(f"0.0,{x},0.0,0.5,1.0,0.0,0.0,0.0\n")
    return lines


BOX = ["header\n", "0.0,0.0,0.0,0.1,0.1,0.1,1.0,0.0,0.0,0.0\n"]
K0 = np.array([[500.0, 0, 320], [0, 500.0, 240], [0, 0, 1]])


@pytest.mark.parametrize("kinds,rows_of_frames", [
    (["in", "in", "in"], [0, 1, 2, None]),
    (["#", "in", "far", "in", "", "far", "in"], [0, 2, 4, None, None]),        # data rows 0..4: the skipped ones give no frame
    (["far", "far", "in"], [2, None, None]),
    (["in", "far", "#", "far", "in", "in"], [0, 3, 4]),
])
def test_frame_i_gets_the_ith_kept_row_and_frames_past_them_nothing(kinds, rows_of_frames):
    saved, keep = sr.process_poses(K0, BOX, _rows_text(kinds))
    data_kinds = [k for k in kinds if k in ("in", "far")]
    assert keep.tolist() == [1 if k == "in" else 0 for k in data_kinds]
    _, homo = sr.get_bbox3d(BOX)
    frames = [np.zeros((480, 640, 3), np.uint8)] * len(rows_of_frames)
    got = [None if r is None else r["row"] for r in sr.parse_video(frames, saved, K0, homo, 64)]
    assert got == rows_of_frames


def test_the_flip_turns_arkits_camera_into_opencvs():
    """ARKit's camera looks down -z; the flip diag(1, -1, -1) turns it into OpenCV's camera, which looks down +z: with the
    identity quaternion the object 0.5 m in front along ARKit's -z must sit at T_oc's +z."""
    saved, _ = sr.process_poses(K0, BOX, ["0.0,0.0,0.0,0.5,1.0,0.0,0.0,0.0\n"])
    T_oc = saved[0][0]
    assert T_oc[2, 3] == pytest.approx(0.5) and np.allclose(T_oc[:3, :3], np.diag([1, -1, -1]))


@pytest.mark.parametrize("axis,side", [(0, "lo"), (1, "lo"), (0, "hi"), (1, "hi")])
def test_each_skip_bound_alone(axis, side):
    base = np.array([[10.25, 20.5], [300.75, 400.5]])
    bound = -1000.0 if side == "lo" else 3000.0
    for delta, skip in ((-1e-9, side == "lo"), (0.0, False), (1e-9, side == "hi")):
        p = base.copy()
        p[0 if side == "lo" else 1, axis] = bound + delta
        assert sr.skipped(p) == skip, (axis, side, delta)
    p = base.copy()
    p[0, axis] = np.nan                                           # numpy's min propagates NaN, and NaN compares false
    assert not sr.skipped(p)


# ---- the colour crop ----

def _cases(n):
    return [c for c in cr.sweep_cases(n, seed=77)]


@pytest.mark.parametrize("C", [3, 4])
def test_cv2_colour_warp_is_its_per_channel_grey_warp(C):
    """Over boxes inside, across every edge, wholly outside and larger than the frame, 1-pixel and large sides: cv2.warpAffine
    of a C-channel image equals, channel by channel, its warp of each plane -- both stages of the crop."""
    frames = {}
    n_mismatch = 0
    for f, box, S, _ in _cases(200) + [(3, np.array([5, 7, 6, 8], np.int32), 16, None), (5, np.array([-900, -700, 2900, 2100], np.int32), 64, None)]:
        if not cr.box_ok(box):
            continue
        H, W = cr.SWEEP_FRAMES[f]
        img = frames.setdefault((f, C), sr.colour_frame(H, W, f, C))
        x0, y0, x1, y1 = (int(v) for v in box)
        im1, _ = sr.get_image_crop_resize(img, box, [y1 - y0, x1 - x0])
        im2, _ = sr.get_image_crop_resize(im1, [0, 0, x1 - x0, y1 - y0], [S, S])
        for c in range(C):
            p1, _ = sr.get_image_crop_resize(np.ascontiguousarray(img[..., c]), box, [y1 - y0, x1 - x0])
            p2, _ = sr.get_image_crop_resize(p1, [0, 0, x1 - x0, y1 - y0], [S, S])
            n_mismatch += int(np.count_nonzero(im2.reshape(S, S, C)[..., c] != p2)) + int(np.count_nonzero(im1.reshape(p1.shape + (C,))[..., c] != p1))
    assert n_mismatch == 0


def test_colour_first_and_grey_first_crops_differ():
    """The reason the device crops colour frames: the reference crops the BGR frame, writes it, and reads it back grey.  Turning
    the frame grey first and cropping that gives other pixels on a realistic box."""
    rng = np.random.default_rng(9)
    bgr = rng.integers(0, 256, (1440, 1920, 3), dtype=np.uint8)
    bgr = cv2.GaussianBlur(bgr, (0, 0), 3)
    box = np.array([600, 300, 1300, 1000])
    im1, _ = sr.get_image_crop_resize(bgr, box, [700, 700])
    colour_first = sr.png_grey(sr.get_image_crop_resize(im1, [0, 0, 700, 700], [512, 512])[0])
    grey = G.grey_from_bgr(bgr)
    g1, _ = sr.get_image_crop_resize(grey, box, [700, 700])
    grey_first = sr.get_image_crop_resize(g1, [0, 0, 700, 700], [512, 512])[0]
    differ = np.count_nonzero(colour_first != grey_first) / colour_first.size
    assert differ > 0.05, differ
    assert np.abs(colour_first.astype(int) - grey_first.astype(int)).max() <= 2
