"""The numpy model of the reference's crop (tests/crop_reference.py, the oracle of csrc/crop.cu) against the golden vectors the
reference's own functions produced with OpenCV (tests/golden/make_crop.py): images and transforms bit for bit."""
import os

import numpy as np
import pytest

from tests import crop_reference as cr
from tests.golden_util import GOLDEN_DIR


@pytest.fixture(scope="module")
def golden():
    g = dict(np.load(os.path.join(GOLDEN_DIR, "pnp_crop_cases.npz"), allow_pickle=False))
    g["frame_images"] = [cr.synthetic_frame(*(int(v) for v in f)) for f in g["frames"]]
    return g


def test_fixture_covers_the_listed_boxes(golden):
    g = golden
    box, (H, W) = g["box"], (480, 640)
    f0 = g["case_frame"] == 0
    w, h = box[:, 2] - box[:, 0], box[:, 3] - box[:, 1]
    assert len(box) >= 30 and len(g["sc_box"]) >= 10
    assert (f0 & (box[:, 0] < 0) & (box[:, 2] > 0)).any() and (f0 & (box[:, 1] < 0) & (box[:, 3] > 0)).any()      # crossing left, top
    assert (f0 & (box[:, 0] < W) & (box[:, 2] > W)).any() and (f0 & (box[:, 1] < H) & (box[:, 3] > H)).any()      # right, bottom
    assert (f0 & ((box[:, 0] >= W) | (box[:, 2] <= 0))).any()                                                     # wholly outside
    assert (w == 1).any() and (h == 1).any() and (w % 2 == 1).any() and (w % 2 == 0).any() and (w != h).any()
    f1 = g["case_frame"] == 1
    assert (f1 & (w > 128) & (h > 96)).any()                                                                      # larger than the frame
    assert (g["sc_box"] < 0).any() and set(g["crop_size"].tolist()) >= {8, 64, 512}


def test_oracle_equals_every_golden_crop(golden):
    g = golden
    for i in range(len(g["box"])):
        im1, im2, T1, T2, K_crop = cr.crop_img_by_bbox(g["frame_images"][g["case_frame"][i]], g["box"][i], g["K"][i], int(g["crop_size"][i]))
        assert np.array_equal(T1, g["T1"][i]) and np.array_equal(T2, g["T2"][i]), i
        assert im1.shape == g[f"stage1_{i}"].shape and np.array_equal(im1, g[f"stage1_{i}"]), i
        assert np.array_equal(im2, g[f"stage2_{i}"]), i
        np.testing.assert_allclose(K_crop, g["K_crop"][i], rtol=1e-12, atol=0)


def test_oracle_boxes_equal_the_golden_boxes(golden):
    g = golden
    for i in range(len(g["sc_box"])):
        np.testing.assert_allclose(cr.reproj(g["sc_K"][i], g["sc_pose"][i], g["sc_corners"][i]), g["sc_proj"][i], rtol=1e-12)
        assert np.array_equal(cr.box_from_pose(g["sc_K"][i], g["sc_pose"][i], g["sc_corners"][i]), g["sc_box"][i]), i
    bad = g["sc_pose"][0].copy()
    bad[0, 3] = np.nan
    assert np.array_equal(cr.box_from_pose(g["sc_K"][0], bad, g["sc_corners"][0]), [0, 0, 0, 0])
    far = g["sc_pose"][0].copy()
    far[0, 3] = 1e9
    assert np.array_equal(cr.box_from_pose(g["sc_K"][0], far, g["sc_corners"][0]), [0, 0, 0, 0])


def test_weight_table_is_the_closed_form_the_kernel_uses():
    """crop.cu computes the bilinear weights as 32 * (32 - fx | fx) * (32 - fy | fy).  That is cv2's table everywhere but at
    fx = fy = 0, where the table holds (32767, 1, 0, 0) for (32768, 0, 0, 0): the rounded pixel is the same for every pair."""
    T = cr.weight_table()
    for fy in range(32):
        for fx in range(32):
            if fx or fy:
                assert np.array_equal(T[fy, fx], cr.closed_form_weights(fx, fy)), (fy, fx)
    assert T[0, 0].tolist() == [32767, 1, 0, 0]
    p0, p1 = np.meshgrid(np.arange(256), np.arange(256), indexing="ij")
    assert np.array_equal((32767 * p0 + p1 + (1 << 14)) >> 15, (32768 * p0 + (1 << 14)) >> 15)


def test_oracle_equals_live_opencv():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(7)
    img = cr.synthetic_frame(300, 400, 3)
    for t in range(200):
        x0, y0 = rng.integers(-150, 450, 2)
        w, h = rng.integers(1, 420, 2)
        box = [int(x0), int(y0), int(x0 + w), int(y0 + h)]
        S = int(rng.choice([8, 64, 160]))
        im1, im2, T1, T2, _ = cr.crop_img_by_bbox(img, box, np.eye(3), S)
        for src, T, (ow, oh), got in ((img, T1, (w, h), im1), (im1, T2, (S, S), im2)):
            c = np.float32([[box[0] + w / 2, box[1] + h / 2], [0, 0], [0, 0]]) if src is img else np.float32([[w / 2, h / 2], [0, 0], [0, 0]])
            d = np.float32([[ow / 2, oh / 2], [0, 0], [0, 0]])
            c[1] = c[0] + np.float32([0, w * -0.5])
            d[1] = d[0] + np.float32([0, ow * -0.5])
            for p in (c, d):
                p[2] = p[1] + np.float32([-(p[0] - p[1])[1], (p[0] - p[1])[0]])
            M = cv2.getAffineTransform(c, d)
            assert np.array_equal(M, T), (t, box)
            assert np.array_equal(cv2.warpAffine(src, M, (int(ow), int(oh)), flags=cv2.INTER_LINEAR), got), (t, box, S)
