"""An annotated scan on the GPU (onepose_b200.scan, crop.crop_frames_colour; csrc/scan.cu, csrc/crop.cu) against the reference
model of parse_scanned_data.py (tests/scan_reference.py) and the golden it made (tests/golden/make_scan.py): poses, boxes and
the pairing exactly or to fp64 rounding, the colour crops bit for bit against cv2, and the evaluation's grey read of them."""
import os
import re

import numpy as np
import pytest
import torch

from onepose_b200 import _lib, crop, frames, pnp, scan, synthetic
from tests import scan_reference as sr
from tests.golden_util import GOLDEN_DIR

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SLEEP = 1 << 29              # device cycles of torch.cuda._sleep: about 0.25 s on an H100


@pytest.fixture(scope="module")
def golden():
    g = dict(np.load(os.path.join(GOLDEN_DIR, "pnp_scan_cases.npz"), allow_pickle=False))
    H, W = (int(v) for v in g["frame_hw"])
    g["frames"] = np.stack([sr.colour_frame(H, W, f) for f in range(int(g["n_frames"]))])
    g["arposes"] = np.array([[float(e) for e in ln.strip().split(",")] for ln in str(g["arposes_txt"]).splitlines()
                             if ln.strip() and not ln.strip().startswith("#")])
    _, g["bbox_homo"] = sr.get_bbox3d(str(g["box_txt"]).splitlines(keepends=True))
    return g


def _args(g):
    return tuple(torch.from_numpy(np.ascontiguousarray(g[k])).to(DEV) for k in ("K", "arposes", "T_ow", "bbox3d"))


def _close(a, b, rel):
    """|a - b| <= rel * max |b| over the whole matrix or box (a box's small coordinate carries its large ones' rounding)."""
    a, b = np.asarray(a), np.asarray(b)
    assert np.all(np.abs(a - b) <= rel * np.abs(b).max()), np.abs(a - b).max()


def test_object_poses_equal_the_reference(golden):
    g = golden
    out = scan.object_poses(*_args(g))
    n, c = len(g["keep"]), int(g["count"])
    assert out["count"].item() == c and out["keep"].cpu().numpy().tolist() == g["keep"].tolist()
    assert out["row"][:c].cpu().numpy().tolist() == g["row"].tolist() and out["row"][c:].cpu().numpy().tolist() == [-1] * (n - c)
    np.testing.assert_allclose(out["pose"][:c].cpu().numpy(), g["pose"], atol=1e-12, rtol=0)
    np.testing.assert_allclose(out["proj"][:c].cpu().numpy(), g["proj"], atol=1e-7, rtol=0)
    assert np.array_equal(out["box"][:c].cpu().numpy(), np.stack([np.concatenate([p.astype(int).min(0), p.astype(int).max(0)]) for p in g["proj"]]))
    assert not out["pose"][c:].any() and not out["proj"][c:].any() and not out["box"][c:].any()
    again = scan.object_poses(g["K"], g["arposes"], g["T_ow"], g["bbox3d"])               # numpy inputs: the same results
    for k in out:
        assert torch.equal(again[k], out[k]), k


def test_each_skip_bound_and_the_pairing_on_the_device():
    """Rows past each bound alone, around kept rows: keep, count and the slots of the kept rows, with comment and blank lines
    removed by read_arposes."""
    K0 = np.array([[500.0, 0, 320], [0, 500.0, 240], [0, 0, 1]])
    box = ["header\n", "0.0,0.0,0.0,0.1,0.1,0.1,1.0,0.0,0.0,0.0\n"]
    moves = {"in": "0.01,0.02,0.5", "x0": "2.2,0.0,0.5", "y0": "0.0,-2.2,0.5", "x1": "-2.9,0.0,0.5", "y1": "0.0,2.9,0.5"}
    kinds = ["in", "x0", "in", "y0", "x1", "in", "y1", "in"]
    lines = [f"{i * 0.1},{moves[k]},1.0,0.0,0.0,0.0\n" for i, k in enumerate(kinds)]
    saved, keep = sr.process_poses(K0, box, lines)
    assert keep.tolist() == [int(k == "in") for k in kinds]
    rows = np.array([[float(e) for e in ln.split(",")] for ln in lines])
    bbox3d, T_ow = sr.get_bbox3d(box)[0], sr.parse_box(box)
    out = scan.object_poses(K0, rows, T_ow, bbox3d, device=DEV)
    assert out["keep"].tolist() == keep.tolist() and out["count"].item() == len(saved)
    assert out["row"].tolist() == [saved[i][2] for i in range(len(saved))] + [-1] * (len(rows) - len(saved))
    for i in range(len(saved)):
        np.testing.assert_allclose(out["pose"][i].cpu().numpy(), saved[i][0], atol=1e-12, rtol=0)


def _reference_frames(g, F=None):
    F = int(g["n_frames"]) if F is None else F
    saved, _ = sr.process_poses(g["K"], str(g["box_txt"]).splitlines(keepends=True), str(g["arposes_txt"]).splitlines(keepends=True))
    return sr.parse_video(list(g["frames"][:F]), saved, g["K"], g["bbox_homo"], int(g["crop_size"]))


def test_annotate_equals_the_reference(golden):
    g = golden
    F, c, S = int(g["n_frames"]), int(g["count"]), int(g["crop_size"])
    ref = _reference_frames(g)
    ann = scan.annotate(torch.from_numpy(g["frames"]).to(DEV), *_args(g), crop_size=S)
    assert ann["image"].dtype == torch.uint8 and tuple(ann["image"].shape) == (F, S, S, 3)
    assert ann["status"].tolist() == [1] * c + [0] * (F - c)
    img = ann["image"].cpu().numpy()
    grey = frames.grey_frames(ann["image"]).cpu().numpy()
    for f in range(c):
        r = ref[f]
        assert np.array_equal(img[f], r["image"]), f
        assert np.array_equal(grey[f], sr.png_grey(r["image"])), f                    # the evaluation's cv2.imwrite / imread
        assert np.array_equal(ann["box"][f].cpu().numpy(), r["box"]) and np.array_equal(r["box"], g["box"][f])
        np.testing.assert_allclose(ann["pose"][f].cpu().numpy(), r["pose"], atol=1e-12, rtol=0)
        _close(ann["K_crop"][f].cpu().numpy(), r["K_crop"], 1e-12)
        _close(ann["M"][f].cpu().numpy(), r["M"], 1e-12)
        _close(ann["box_crop"][f].cpu().numpy(), r["box_crop"], 1e-12)
        _close(ann["K_crop"][f].cpu().numpy(), g["K_crop"][f], 1e-12)
        _close(ann["M"][f].cpu().numpy(), g["M"][f], 1e-12)
        _close(ann["box_crop"][f].cpu().numpy(), g["box_crop"][f], 1e-12)
    for k in ("pose", "box", "image", "M", "box_crop"):
        assert not ann[k][c:].any(), k


def test_annotate_with_fewer_frames_than_kept_rows_and_padded_frames(golden):
    g = golden
    F, S = 5, 64
    big = torch.zeros(F, *g["frames"].shape[1:3], 4, dtype=torch.uint8, device=DEV)    # rows and frames padded: a C = 3 view of C = 4
    view = big[:, :, :, :3]
    assert view.stride(2) == 4
    with pytest.raises(ValueError, match="packed pixels"):
        scan.annotate(view, *_args(g), crop_size=S)
    wide = torch.zeros(F, g["frames"].shape[1], g["frames"].shape[2] + 7, 3, dtype=torch.uint8, device=DEV)
    wide[:, :, :g["frames"].shape[2]] = torch.from_numpy(g["frames"][:F]).to(DEV)
    ann = scan.annotate(wide[:, :, :g["frames"].shape[2]], *_args(g), crop_size=S)
    ref = _reference_frames({**g, "crop_size": np.array(S)}, F)
    assert ann["status"].tolist() == [1] * F
    for f in range(F):
        assert np.array_equal(ann["image"][f].cpu().numpy(), ref[f]["image"]), f
        np.testing.assert_allclose(ann["pose"][f].cpu().numpy(), ref[f]["pose"], atol=1e-12, rtol=0)


@pytest.mark.parametrize("C", [3, 4])
def test_crop_frames_colour_is_cv2s_and_the_grey_crop_of_each_plane(C):
    H, W, S = 97, 131, 48
    px = np.stack([sr.colour_frame(H, W, f, C) for f in range(3)])
    boxes = np.array([[10, 12, 60, 70], [-20, 30, 40, 150], [90, -5, 140, 30], [3, 4, 4, 5], [200, 200, 260, 240], [5, 5, 5, 9]], np.int32)
    index = np.array([0, 1, 2, 1, 0, 2], np.int32)
    K = np.array([[300.0, 0, 65.5], [0, 301.0, 48.25], [0, 0, 1]])
    big = torch.zeros(3, H + 3, W + 9, C, dtype=torch.uint8, device=DEV)
    big[:, :H, :W] = torch.from_numpy(px).to(DEV)
    fr = big[:, :H, :W]                                                            # padded rows and frames
    Kd, bd = torch.from_numpy(K).to(DEV), torch.from_numpy(boxes).to(DEV)
    out = crop.crop_frames_colour(fr, bd, Kd, S, frame_index=torch.from_numpy(index).to(DEV))
    assert out["status"].tolist() == [1, 1, 1, 1, 1, 0]
    img = out["image"].cpu().numpy()
    for b, (box, f) in enumerate(zip(boxes, index)):
        if out["status"][b]:
            x0, y0, x1, y1 = (int(v) for v in box)
            im1, _ = sr.get_image_crop_resize(px[f], box, [y1 - y0, x1 - x0])
            im2, _ = sr.get_image_crop_resize(im1, [0, 0, x1 - x0, y1 - y0], [S, S])
            assert np.array_equal(img[b], im2), b
        else:
            assert not img[b].any()
    for c in range(C):                                                                # each plane through the grey crop
        plane = fr[..., c].contiguous()
        grey = crop.crop_frames(plane, bd, Kd, S, frame_index=torch.from_numpy(index).to(DEV))
        assert torch.equal((grey["image"][:, 0] * 255).round().to(torch.uint8), out["image"][..., c])
        for k in ("K_crop", "trans", "status"):
            assert torch.equal(grey[k], out[k]), k
    one = crop.crop_frames_colour(fr[1:2].expand(2, -1, -1, -1), bd[1:3], Kd, S)     # frame stride 0, no frame_index
    two = crop.crop_frames_colour(fr[[1, 1]].contiguous(), bd[1:3], Kd, S)
    for k in one:
        assert torch.equal(one[k], two[k]), k


def test_refusals_name_their_entry_point_and_condition():
    fr = torch.zeros(2, 16, 16, 3, dtype=torch.uint8, device=DEV)
    bx = torch.tensor([[0, 0, 8, 8], [4, 4, 4, 12]], dtype=torch.int32, device=DEV)
    K = torch.eye(3, dtype=torch.float64, device=DEV)
    assert crop.crop_frames_colour(fr, bx, K, 8)["status"].tolist() == [1, 0]                     # an empty box: status 0
    with pytest.raises(ValueError, match="C = 3 or 4"):
        crop.crop_frames_colour(torch.zeros(2, 16, 16, 2, dtype=torch.uint8, device=DEV), bx, K, 8)
    with pytest.raises(ValueError, match="packed pixels"):
        crop.crop_frames_colour(torch.zeros(2, 16, 16, 6, dtype=torch.uint8, device=DEV)[..., ::2], bx, K, 8)
    with pytest.raises(ValueError, match="crop_size"):
        crop.crop_frames_colour(fr, bx, K, 12)
    with pytest.raises(ValueError, match="boxes"):
        crop.crop_frames_colour(fr, bx.to(torch.int64), K, 8)
    out = [torch.empty(2, 8, 8, 3, dtype=torch.uint8, device=DEV), torch.empty(2, 9, dtype=torch.float64, device=DEV),
           torch.empty(2, 12, dtype=torch.float64, device=DEV), torch.empty(2, dtype=torch.int32, device=DEV)]
    base = [fr, 16 * 16 * 3, 16 * 3, 2, 16, 16, 3, None, 2, bx, K.expand(2, 3, 3).contiguous(), 8, *out]
    for i, val, cond in ((6, 2, "C == 3 || C == 4"), (2, 16 * 2, "row_pitch >= (int64_t)W * C"), (11, 12, "crop_size % 8 == 0"),
                         (3, 1, "frame_index != nullptr || n_frames == B")):
        a = list(base)
        a[i] = val
        with pytest.raises(_lib.OpbError, match=r"opb_crop_resize_colour: .*" + re.escape(cond)):
            _lib.call(torch.device(DEV), "opb_crop_resize_colour", *a)
    rows = torch.zeros(1, 8, dtype=torch.float64, device=DEV)
    with pytest.raises(_lib.OpbError, match=r"opb_scan_poses: .*n_corners > 0"):
        _lib.call(torch.device(DEV), "opb_scan_poses", K, rows, 1, torch.eye(4, dtype=torch.float64, device=DEV), K, 0, 1,
                  torch.empty(16, dtype=torch.float64, device=DEV), None, torch.empty(4, dtype=torch.int32, device=DEV), None, None,
                  torch.empty(1, dtype=torch.int32, device=DEV))
    with pytest.raises(ValueError, match="arposes must be"):
        scan.object_poses(K, torch.zeros(3, 7, dtype=torch.float64, device=DEV), torch.eye(4), torch.zeros(8, 3))
    with pytest.raises(ValueError, match="bbox3d must be"):
        scan.object_poses(K, rows, torch.eye(4), torch.zeros(0, 3))


# ---- past the kernel's first 256-row tile: a real capture has one ARposes row per video frame ----

K0 = np.array([[500.0, 0, 320], [0, 500.0, 240], [0, 0, 1]])
BOX = ["header\n", "0.0,0.0,0.0,0.1,0.1,0.1,1.0,0.0,0.0,0.0\n"]
# the moves of test_each_skip_bound_and_the_pairing_on_the_device, and a camera at the box corner (0.05, 0.05, 0.05): that
# corner projects to 0 / 0, so the extent is NaN, which compares false against every bound and the row is kept
SKIPS = {"x0": "2.2,0.0,0.5", "y0": "0.0,-2.2,0.5", "x1": "-2.9,0.0,0.5", "y1": "0.0,2.9,0.5"}
SCAN_N = [255, 256, 257, 511, 512, 513, 1000, 4097]
PATTERNS = ["all", "none", "alternating", "runs", "nan"]


def _move(kind, i, skips=SKIPS):
    if kind == "in":            # kept, a pose of its own on every row, and no corner that projects to a whole pixel (where
        # astype(int) would turn an ulp of difference between two correct fp64 evaluations into a pixel)
        x, y, z = (0.01 + 0.002 * (i * 0.6180339887498949 % 1), 0.02 - 0.002 * (i * 0.41421356237309515 % 1),
                   0.5 + 0.01 * (i * 0.7320508075688772 % 1))
        return f"{x!r},{y!r},{z!r}"
    if kind == "nan":
        return "0.05,0.05,0.05"
    return skips[kind]


def _kinds(n, pattern):
    """Per row "in", "nan" or one of the skip moves.  runs: skipped runs [m - 37, m) below odd multiples m of 256 and [m, m + 53)
    from even ones (0 included), so runs end and start exactly on tile boundaries.  nan: NaN extents at rows 0, 255, 256, 511,
    512, 767, 768 and n - 1, among rows of which every third is skipped."""
    skip = list(SKIPS)
    k = [skip[i % 4] if pattern == "none" or (pattern == "alternating" and i % 2) or (pattern == "nan" and i % 3 == 1) else "in"
         for i in range(n)]
    if pattern == "runs":
        for m in range(0, n + 1, 256):
            for i in (range(m - 37, m) if (m // 256) % 2 else range(m, m + 53)):
                if 0 <= i < n:
                    k[i] = skip[i % 4]
    if pattern == "nan":
        for i in (0, 255, 256, 511, 512, 767, 768, n - 1):
            if i < n:
                k[i] = "nan"
    return k


def _scan_case(kinds, K=K0, corners=None, skips=SKIPS):
    """(rows f64 [n, 8], T_ow, corners, the model's saved slots and keep) for rows of the given kinds."""
    lines = [f"{i * 0.1},{_move(k, i, skips)},1.0,0.0,0.0,0.0\n" for i, k in enumerate(kinds)]
    with np.errstate(all="ignore"):
        saved, keep = sr.process_poses(K, BOX, lines, corners)
    assert keep.tolist() == [int(k in ("in", "nan")) for k in kinds]
    rows = np.array([[float(e) for e in ln.split(",")] for ln in lines])
    return rows, sr.parse_box(BOX), sr.get_bbox3d(BOX)[0] if corners is None else corners, saved, keep


def _ref_box(p):
    """The kernel's box of projected corners p: [x0, y0, x1, y1] truncated towards zero (astype(int) of the min / max), or 0
    when an extent is not a finite int32 (NaN: numpy's min / max propagate it)."""
    with np.errstate(all="ignore"):
        ext = np.concatenate([p.min(0), p.max(0)])
    return np.trunc(ext).astype(np.int32) if np.all(np.isfinite(ext)) else np.zeros(4, np.int32)


def _check_slots(got, saved, keep, n_out):
    """got (numpy) of opb_scan_poses with n_out slots against the model: keep, the full kept count, and per slot below
    min(count, n_out) the row, pose (1e-12), projections (1e-7; NaN and infinities where the model has them) and box; slots from
    the count to n_out cleared."""
    c = len(saved)
    m = min(c, n_out)
    assert got["keep"].tolist() == keep.tolist() and int(got["count"][0]) == c
    assert got["row"][:m].tolist() == [saved[i][2] for i in range(m)]
    if m:
        np.testing.assert_allclose(got["pose"][:m], np.stack([saved[i][0] for i in range(m)]), atol=1e-12, rtol=0)
        ref = np.stack([saved[i][1] for i in range(m)])
        p = got["proj"][:m]
        assert np.array_equal(np.isnan(p), np.isnan(ref)) and np.array_equal(np.isinf(p), np.isinf(ref))
        fin = np.isfinite(ref)
        np.testing.assert_allclose(p[fin], ref[fin], atol=1e-7, rtol=0)
        assert np.array_equal(got["box"][:m], np.stack([_ref_box(saved[i][1]) for i in range(m)]))
    assert not got["pose"][c:n_out].any() and not got["proj"][c:n_out].any() and not got["box"][c:n_out].any()
    assert (got["row"][c:n_out] == -1).all()


def _numpy(out):
    return {k: v.cpu().numpy() for k, v in out.items()}


@pytest.mark.parametrize("pattern", PATTERNS)
@pytest.mark.parametrize("n", SCAN_N)
def test_object_poses_past_one_tile(n, pattern):
    kinds = _kinds(n, pattern)
    rows, T_ow, corners, saved, keep = _scan_case(kinds)
    out = _numpy(scan.object_poses(K0, rows, T_ow, corners, device=DEV))
    _check_slots(out, saved, keep, n)
    if pattern == "none":
        assert int(out["count"][0]) == 0 and (out["row"] == -1).all()
    if pattern == "nan":
        nan_slots = [i for i in range(len(saved)) if kinds[saved[i][2]] == "nan"]
        assert len(nan_slots) == sum(k == "nan" for k in kinds) and not out["box"][nan_slots].any()


PAD = 8                      # spare rows past n_out and past n_rows that the call must leave alone
FILL = 0xA5


def _filled(shape, dtype):
    """A device tensor of the given shape whose bytes are all FILL."""
    n = int(np.prod(shape)) * torch.empty(0, dtype=dtype).element_size()
    return torch.full((n,), FILL, dtype=torch.uint8, device=DEV).view(dtype).reshape(shape)


def _untouched(t):
    return bool((t.contiguous().view(torch.uint8) == FILL).all())


@pytest.mark.parametrize("n,pattern", [(1000, "runs"), (4097, "alternating"), (513, "nan"), (600, "all")])
def test_scan_poses_writes_its_slots_only(n, pattern):
    """opb_scan_poses into outputs filled with a byte pattern first, with PAD rows past n_out (and past n_rows for keep): n_out
    below the kept count and above it, each across a multiple of 256 from it, equal to it, 1, and past n_rows.  count is the full
    kept count whatever n_out is, slots from it to n_out are cleared, and nothing past n_out / n_rows is written."""
    rows, T_ow, corners, saved, keep = _scan_case(_kinds(n, pattern))
    c, nc = len(saved), len(corners)
    assert c >= 256
    lo = c // 256 * 256                                   # a multiple of 256 at or below the count
    args = [torch.from_numpy(np.ascontiguousarray(a)).to(DEV) for a in (K0, rows, T_ow, corners)]
    for n_out in sorted({1, lo - 1, c - 1, c, c + 1, lo + 257, n + 300}):
        out = {"pose": _filled((n_out + PAD, 4, 4), torch.float64), "proj": _filled((n_out + PAD, nc, 2), torch.float64),
               "box": _filled((n_out + PAD, 4), torch.int32), "row": _filled((n_out + PAD,), torch.int32),
               "keep": _filled((n + PAD,), torch.int32), "count": _filled((1 + PAD,), torch.int32)}
        _lib.call(torch.device(DEV), "opb_scan_poses", args[0], args[1], n, args[2], args[3], nc, n_out, out["pose"], out["proj"],
                  out["box"], out["row"], out["keep"], out["count"])
        got = _numpy({k: v[:n if k == "keep" else 1 if k == "count" else n_out] for k, v in out.items()})
        _check_slots(got, saved, keep, n_out)
        for k, v in out.items():
            assert _untouched(v[n if k == "keep" else 1 if k == "count" else n_out:]), (n_out, k)


@pytest.mark.parametrize("nc", [1, 9, 1024])
def test_object_poses_with_any_number_of_corners(nc):
    """n_corners of 1, 9 and the bound 1024, over 600 rows with skipped runs across the tile boundaries, against the model's
    reproj and skip rule over the same corners."""
    rs = np.random.RandomState(nc)
    corners = rs.uniform(-0.05, 0.05, (nc, 3))
    far = {"x0": "3.0,0.0,0.5", "y0": "0.0,-3.0,0.5", "x1": "-6.0,0.0,0.5", "y1": "0.0,6.0,0.5"}   # past the bounds from any corner
    rows, T_ow, corners, saved, keep = _scan_case(_kinds(600, "runs"), corners=corners, skips=far)
    out = _numpy(scan.object_poses(K0, rows, T_ow, corners, device=DEV))
    assert out["proj"].shape == (600, nc, 2)
    _check_slots(out, saved, keep, 600)


def test_annotate_past_one_tile():
    """annotate of F = 600 small frames (32 x 48, crop_size 8) and 800 ARposes rows of which fewer than F are kept: the pairing,
    status, poses, boxes and crops against the model's parse_video, and frames past the kept count cleared, across three tiles."""
    K = np.array([[40.0, 0, 24], [0, 40.0, 16], [0, 0, 1]])     # the kept boxes fall inside the 48 x 32 frame
    F, S, n = 600, 8, 800
    far = {"x0": "30.0,0.0,0.5", "y0": "0.0,-30.0,0.5", "x1": "-80.0,0.0,0.5", "y1": "0.0,80.0,0.5"}
    kinds = ["in" if i % 5 in (0, 2, 3) or 250 <= i < 270 else list(far)[i % 4] for i in range(n)]
    rows, T_ow, corners, saved, keep = _scan_case(kinds, K, skips=far)
    assert 256 < len(saved) < F
    frames_np = np.stack([sr.colour_frame(32, 48, f) for f in range(F)])
    ref = sr.parse_video(list(frames_np), saved, K, sr.get_bbox3d(BOX)[1], S)
    ann = scan.annotate(torch.from_numpy(frames_np).to(DEV), K, rows, T_ow, corners, crop_size=S)
    status = ann["status"].cpu().numpy()
    assert status.tolist() == [int(r is not None) for r in ref]
    c = len(saved)
    assert int(status.sum()) == c
    img, pose, box = (ann[k].cpu().numpy() for k in ("image", "pose", "box"))
    for f in range(c):
        np.testing.assert_allclose(pose[f], ref[f]["pose"], atol=1e-12, rtol=0)
        assert np.array_equal(box[f], ref[f]["box"]) and np.array_equal(img[f], ref[f]["image"]), f
    for k in ("pose", "box", "image", "M", "box_crop"):
        assert not ann[k][c:].any(), k


# ---- the evaluation step on the crops ----

def _chain(image_u8, K_crop, pose, sp, mm, kp3):
    _, inp = frames.grey_frames(image_u8, normalised=True)
    det = sp.forward_padded(inp, cap=1024)
    out = mm.match_frames(det["descriptors"], return_conf=False, lengths=det["counts"])
    res = pnp.poses_from_matches(K_crop, det["keypoints"], kp3, out["matches0"], out["matching_scores0"], scale=1000)
    rot, trans = pnp.pose_errors(res["pose"], pose)
    return res["n_inliers"], rot, trans, det["counts"], det["keypoints"]


def test_evaluation_step_on_device_crops_equals_it_on_the_reference_crops(golden):
    """grey_frames(image) -> extractor -> matcher -> poses_from_matches(K_crop) -> pose_errors(pose), once on annotate's results
    and once on the reference model's crops read back through PNG with its K_crop and pose.  Synthetic weights: the poses are
    not the planted ones, but every count and error must be the same."""
    from onepose_b200 import GATsSuperGlue, SuperPoint
    g = golden
    c, S = min(int(g["count"]), 8), int(g["crop_size"])
    sp = SuperPoint({"nms_radius": 3, "max_keypoints": 1024}).eval()
    sp.load_state_dict({k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in synthetic.make_superpoint_state_dict(0, 4.0).items()},
                       strict=True)
    sp = sp.cuda()
    s = synthetic.make_planted_scene(4, [401], 1024, 600)
    mm = GATsSuperGlue(dict(synthetic.DEFAULT_HPARAMS)).eval()
    mm.load_state_dict({k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in synthetic.make_state_dict(0).items()})
    mm = mm.cuda()
    mm.set_object(torch.as_tensor(s["desc3d"]).cuda(), torch.as_tensor(s["desc2d_db"]).cuda())
    kp3 = torch.as_tensor(s["keypoints3d"]).cuda()
    ann = scan.annotate(torch.from_numpy(g["frames"][:c]).to(DEV), *_args(g), crop_size=S)
    ref = _reference_frames(g, c)
    dev = _chain(ann["image"], ann["K_crop"], ann["pose"], sp, mm, kp3)
    grey = np.stack([sr.png_grey(r["image"]) for r in ref])
    ref_img = torch.from_numpy(np.stack([r["image"] for r in ref])).to(DEV)
    assert torch.equal(frames.grey_frames(ref_img).cpu(), torch.from_numpy(grey))
    host = _chain(ref_img, torch.from_numpy(np.stack([r["K_crop"] for r in ref])).to(DEV),
                  torch.from_numpy(np.stack([r["pose"] for r in ref])).to(DEV), sp, mm, kp3)
    assert int(dev[3].min()) > 0
    assert torch.equal(dev[0], host[0]) and torch.equal(dev[3], host[3])
    for b in range(c):
        n = int(dev[3][b])
        assert torch.equal(dev[4][b, :n], host[4][b, :n]), b
    torch.testing.assert_close(dev[1], host[1], atol=1e-6, rtol=0)
    torch.testing.assert_close(dev[2], host[2], atol=1e-6, rtol=0)


# ---- the caller's streams and devices (tests/test_streams_devices_gpu.py's conventions) ----

def test_runs_on_the_callers_stream_without_synchronising(golden):
    g = golden
    real = torch.from_numpy(g["frames"][:4]).to(DEV)
    stale = torch.zeros_like(real)
    args = _args(g)
    want = scan.annotate(real, *args, crop_size=64)
    buf = torch.empty_like(real)
    torch.cuda.synchronize()
    s = torch.cuda.Stream(DEV)
    asleep = torch.cuda.Event()
    with torch.cuda.stream(s):
        buf.copy_(stale)
        torch.cuda._sleep(SLEEP)
        asleep.record(s)
        buf.copy_(real)
        out = scan.annotate(buf, *args, crop_size=64)
        busy = not asleep.query()
    torch.cuda.synchronize()
    assert busy, "annotate synchronised the host with the caller's stream"
    for k in want:
        assert torch.equal(out[k], want[k]), k


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two visible GPUs")
def test_on_the_second_device(golden):
    g = golden
    torch.cuda.set_device(0)
    want = scan.annotate(torch.from_numpy(g["frames"][:3]).to("cuda:0"), *_args(g), crop_size=64)
    got = scan.annotate(torch.from_numpy(g["frames"][:3]).to("cuda:1"), g["K"], g["arposes"], g["T_ow"], g["bbox3d"], crop_size=64)
    assert torch.cuda.current_device() == 0
    for k in want:
        assert got[k].device == torch.device("cuda:1") and torch.equal(got[k].cpu(), want[k].cpu()), k
