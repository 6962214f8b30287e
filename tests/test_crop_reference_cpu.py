"""The numpy model of the reference's crop (tests/crop_reference.py, the oracle of csrc/crop.cu) against the golden vectors the
reference's own functions produced with OpenCV (tests/golden/make_crop.py) and against live cv2 at the extremes of the domain:
images and transforms bit for bit.  Also what the GPU sweep's boxes can catch: its rounding ties and the planted variants."""
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


def _cv2_transforms(cv2, box, S):
    """T1, T2 as the reference builds them: get_affine_transform's float32 points through cv2.getAffineTransform."""
    x0, y0, x1, y1 = (int(v) for v in box)
    w, h = x1 - x0, y1 - y0
    out = []
    for c0, (ow, oh) in (((x0 + w / 2, y0 + h / 2), (w, h)), ((w / 2, h / 2), (S, S))):
        c = np.float32([c0, [0, 0], [0, 0]])
        d = np.float32([[ow / 2, oh / 2], [0, 0], [0, 0]])
        c[1] = c[0] + np.float32([0, w * -0.5])
        d[1] = d[0] + np.float32([0, ow * -0.5])
        for p in (c, d):
            p[2] = p[1] + np.float32([-(p[0] - p[1])[1], (p[0] - p[1])[0]])
        out.append(cv2.getAffineTransform(c, d))
    return out


def _probe_positions(h, w, n, rng):
    """Every pixel of the first and last rows and columns, and n seeded random positions: (xs, ys)."""
    ex = np.concatenate([np.arange(w), np.arange(w), np.zeros(h, np.int64), np.full(h, w - 1)])
    ey = np.concatenate([np.zeros(w, np.int64), np.full(w, h - 1), np.arange(h), np.arange(h)])
    return np.concatenate([ex, rng.integers(0, w, n)]), np.concatenate([ey, rng.integers(0, h, n)])


def test_per_pixel_model_equals_the_array_model(golden):
    g = golden
    cases = [(g["frame_images"][g["case_frame"][i]], g["box"][i], int(g["crop_size"][i])) for i in range(len(g["box"]))]
    rng = np.random.default_rng(11)
    frames = [cr.synthetic_frame(h, w, k) for k, (h, w) in enumerate(((300, 400), (1, 37), (29, 1), (37, 53)))]
    for _ in range(300):
        f = frames[int(rng.integers(len(frames)))]
        w, h = (int(v) for v in np.exp(rng.uniform(0, np.log(500), 2)).astype(int))
        x0, y0 = int(rng.integers(-w - 50, f.shape[1] + 50)), int(rng.integers(-h - 50, f.shape[0] + 50))
        cases.append((f, [x0, y0, x0 + w, y0 + h], 8 * int(rng.integers(1, 33))))
    for frame, box, S in cases:
        im1, im2, T1, _, _ = cr.crop_img_by_bbox(frame, box, np.eye(3), S)
        ys, xs = np.mgrid[0:S, 0:S]
        assert np.array_equal(cr.crop_pixels(frame, box, S, xs, ys), im2), (box, S)
        ys, xs = np.mgrid[0:im1.shape[0], 0:im1.shape[1]]
        assert np.array_equal(cr.warp_pixels(frame, T1, xs, ys), im1), (box, S)


M20 = 1 << 20
EXTREMES = [((480, 640), (-3000, -2500, 3000, 3500), 64),              # about 6000 a side, crossing the frame
            ((480, 640), (-2900, 100, 3100, 6100), 512),
            ((480, 640), (-M20, 0, -M20 + 5000, 40), 64),               # at -2^20
            ((480, 640), (M20 - 300, -M20, M20, -M20 + 200), 128),       # at +2^20 and -2^20
            ((480, 640), (-(M20 - 4000), 5, -(M20 - 4000) + 4000, 9), 8),
            ((480, 640), (300, 200, 301, 201), 2048),                   # 1 x 1, dense with ties
            ((480, 640), (10, -5, 11, 400), 1024),                      # 1 x N
            ((480, 640), (639, 479, 640, 480), 1024),
            ((480, 640), (0, 0, 4000, 1), 8),                           # N x 1
            ((480, 640), (-50, 100, 950, 101), 512),
            ((1, 640), (-20, -3, 700, 4), 64),                          # 1 x W, H x 1 and 37 x 53 frames
            ((480, 1), (-3, -10, 2, 500), 128),
            ((37, 53), (-7, -5, 60, 41), 256),
            ((37, 53), (20, 30, 21, 37), 2048)]


@pytest.mark.parametrize("shape,box,S", EXTREMES)
def test_oracle_equals_live_opencv_at_the_extremes(shape, box, S):
    """Both stages against cv2 itself: T1 and T2 bit for bit, every stage-2 pixel, and stage 1 (up to 6000 x 6000, too large
    for the array model) at its edges and 20000 random positions through the per-pixel model."""
    cv2 = pytest.importorskip("cv2")
    img = cr.synthetic_frame(*shape, 5)
    x0, y0, x1, y1 = box
    T1, T2 = cr.crop_transforms(box, S)
    C1, C2 = _cv2_transforms(cv2, box, S)
    assert np.array_equal(C1, T1) and np.array_equal(C2, T2)
    c1 = cv2.warpAffine(img, C1, (x1 - x0, y1 - y0), flags=cv2.INTER_LINEAR)
    c2 = cv2.warpAffine(c1, C2, (S, S), flags=cv2.INTER_LINEAR)
    xs, ys = _probe_positions(y1 - y0, x1 - x0, 20000, np.random.default_rng(3))
    assert np.array_equal(cr.warp_pixels(img, T1, xs, ys), c1[ys, xs])
    ys, xs = np.mgrid[0:S, 0:S]
    assert np.array_equal(cr.crop_pixels(img, box, S, xs, ys), c2)


@pytest.fixture(scope="module")
def sweep():
    return cr.sweep_cases(), [cr.synthetic_frame(h, w, k) for k, (h, w) in enumerate(cr.SWEEP_FRAMES)]


def test_sweep_covers_its_domain(sweep):
    cases, _ = sweep
    box = np.stack([c[1] for c in cases[:-len(cr.SWEEP_TIE_CASES)]]).astype(np.int64)
    HW = np.array([cr.SWEEP_FRAMES[c[0]] for c in cases[:-len(cr.SWEEP_TIE_CASES)]])
    w, h = box[:, 2] - box[:, 0], box[:, 3] - box[:, 1]
    inside = (box[:, 0] >= 0) & (box[:, 1] >= 0) & (box[:, 2] <= HW[:, 1]) & (box[:, 3] <= HW[:, 0])
    outside = (box[:, 2] <= 0) | (box[:, 0] >= HW[:, 1]) | (box[:, 3] <= 0) | (box[:, 1] >= HW[:, 0])
    larger = (box[:, 0] <= 0) & (box[:, 1] <= 0) & (box[:, 2] >= HW[:, 1]) & (box[:, 3] >= HW[:, 0]) & ((w > HW[:, 1]) | (h > HW[:, 0]))
    crossing = ~inside & ~outside & ~larger
    assert min(inside.sum(), outside.sum(), larger.sum(), crossing.sum()) >= 50
    assert all(cr.box_ok(b) for b in box) and w.min() == 1 and h.min() == 1 and max(w.max(), h.max()) > 2000
    S = {c[2] for c in cases}
    assert S >= {8, 512, 2048} and len(S) >= 60


def _tie_counts(cases):
    """Round-half-even ties of adelta, bdelta, X0 and Y0 over both stages of every case: all of them, and those with an odd
    floor, where rounding half down would give another term."""
    ties, odd = np.zeros(4, np.int64), np.zeros(4, np.int64)
    for _, box, S, _ in cases:
        x0, y0, x1, y1 = (int(v) for v in box)
        for T, (w, h) in zip(cr.crop_transforms(box, S), ((x1 - x0, y1 - y0), (S, S))):
            _, raw = cr.fixed_point_terms(cr.inverse_transform(T), np.arange(w), np.arange(h))
            for k, r in enumerate(raw):
                t = r - np.floor(r) == 0.5
                ties[k] += t.sum()
                odd[k] += (t & (np.floor(r) % 2 == 1)).sum()
    return ties, odd


def test_sweep_meets_rounding_ties(sweep):
    """adelta and Y0 meet ties, half of them where half-even and half-down differ.  bdelta and X0 cannot: with rot = 0 the
    inverse map has m[3] = m[1] = 0, so bdelta is 0 and X0 is one integer per stage."""
    ties, odd = _tie_counts(sweep[0])
    print("ties (adelta, bdelta, X0, Y0):", ties.tolist(), "with an odd floor:", odd.tolist())
    assert ties[0] >= 1 and ties[3] >= 1 and odd[0] >= 1 and odd[3] >= 1
    assert ties[1] == 0 and ties[2] == 0


@pytest.mark.parametrize("variant", ["tie_floor", "no_round_delta", "stage1_unrounded"])
def test_sweep_catches_the_planted_variant(sweep, variant):
    """The GPU sweep's list tells each of these slips of the warp from the model: some pixel at the probed positions differs."""
    cases, frames = sweep
    rng = np.random.default_rng(1)
    for i, (f, box, S, _) in enumerate(cases):
        xs, ys = _probe_positions(S, S, 256, rng)
        if not np.array_equal(cr.crop_pixels(frames[f], box, S, xs, ys), cr.crop_pixels(frames[f], box, S, xs, ys, variant)):
            print(f"{variant}: case {i} differs")
            return
    pytest.fail(f"no case of the sweep tells {variant} apart")


def test_the_other_planted_variants_cannot_change_a_result(sweep):
    """Three slips are harmless for every box the crop accepts, so no sweep could catch them:
    - table_unfixed: cv2's (32767, 0, 0, 0) for (32768, 0, 0, 0) at fx = fy = 0 still rounds to p0 for every uint8 p0;
    - no_saturation: a coordinate saturated to int16 and its neighbour lie outside every image of sides <= 32767, as do the
      unsaturated ones, so the four reads are the zero border either way;
    - f64_points: get_affine_transform's points are multiples of 0.5 below 2^22 in magnitude, exact in float32."""
    p0 = np.arange(256)
    assert np.array_equal((32767 * p0 + (1 << 14)) >> 15, p0)
    for raw in (-40000, -32769, -32768, 32767, 32768, 40000):
        for sx in (raw, int(np.clip(raw, -32768, 32767))):
            assert not (0 <= sx < cr.MAX_SIDE) and not (0 <= sx + 1 < cr.MAX_SIDE)
    cases = sweep[0] + [(0, np.array(b, np.int32), S, None) for _, b, S in EXTREMES]
    cases += [(0, np.array([M20 - 32767, -M20, M20, -M20 + 32767], np.int32), 8, None)]
    for _, box, S, _ in cases:
        T, T64 = cr.crop_transforms(box, S), cr.crop_transforms(box, S, "f64_points")
        assert np.array_equal(T[0], T64[0]) and np.array_equal(T[1], T64[1]), box
    f, box, S, _ = cases[0]
    ys, xs = np.mgrid[0:S, 0:S]
    want = cr.crop_pixels(sweep[1][f], box, S, xs, ys)
    for v in ("table_unfixed", "no_saturation", "f64_points"):
        assert np.array_equal(cr.crop_pixels(sweep[1][f], box, S, xs, ys, v), want), v
