"""The PNG byte model (tests/png_reference.py) against cv2.imencode('.png', ...) of OpenCV 4.13, and the numpy emulation of the
device encoder against zlib and the model."""
import struct
import zlib

import cv2
import numpy as np
import pytest

from tests import png_reference as ref

SIZES = [(1, 1), (1, 2), (2, 1), (1, 300), (300, 1), (3, 3), (7, 13), (16, 16), (31, 64), (64, 31), (100, 100), (127, 129),
         (200, 150), (300, 300)]
KINDS = ["noise", "flat", "levels", "gradient", "columns", "ramp"]


def content(kind, shape, rng):
    H, W = shape[:2]
    extra = (1,) * (len(shape) - 2)
    if kind == "noise":
        return rng.integers(0, 256, shape, dtype=np.uint8)
    if kind == "flat":
        return np.full(shape, int(rng.integers(0, 256)), np.uint8)
    if kind == "levels":
        return (rng.integers(0, 3, shape) * 100).astype(np.uint8)
    if kind == "gradient":
        g = (np.arange(H)[:, None] + 3 * np.arange(W)[None, :]).astype(np.uint8).reshape(H, W, *extra)
        return np.ascontiguousarray(np.broadcast_to(g, shape))
    if kind == "columns":
        return np.ascontiguousarray(np.broadcast_to(rng.integers(0, 256, (1, W) + shape[2:], dtype=np.uint8), shape))
    if kind == "ramp":          # SUB rows of 1s: runs that cross rows
        g = (np.arange(W)[None, :] + 1 + np.zeros((H, 1), np.int64)).astype(np.uint8).reshape(H, W, *extra)
        return np.ascontiguousarray(np.broadcast_to(g, shape))
    raise ValueError(kind)


def cv2_png(img):
    return cv2.imencode(".png", img)[1].tobytes()


@pytest.mark.parametrize("C", [1, 3, 4])
@pytest.mark.parametrize("kind", KINDS)
def test_model_and_emulation_equal_cv2_on_the_sweep(C, kind):
    rng = np.random.default_rng(10 * KINDS.index(kind) + C)
    for H, W in SIZES:
        img = content(kind, (H, W) if C == 1 else (H, W, C), rng)
        want = cv2_png(img)
        assert ref.encode(img) == want, (H, W, C, kind)
        filt = ref.filtered(img)
        assert ref.emulate_zlib(filt) == ref.zlib_stream(filt), (H, W, C, kind)


@pytest.mark.parametrize("shape", [(512, 512, 3), (1440, 1920, 3), (1440, 1920)])
@pytest.mark.parametrize("kind", ["noise", "gradient"])
def test_camera_frames_and_crops(shape, kind):
    img = content(kind, shape, np.random.default_rng(1))
    want = cv2_png(img)
    assert ref.encode(img) == want
    filt = ref.filtered(img)
    assert ref.emulate_zlib(filt) == ref.zlib_stream(filt)


def test_scan_fixture_crops():
    """parse_video's 512 x 512 colour crops of the scan fixture's projected boxes, cropped from the scan model's frames."""
    from tests import scan_reference as sr
    g = np.load(sr.__file__.replace("scan_reference.py", "golden/pnp_scan_cases.npz"))
    h, w = (int(v) for v in g["frame_hw"])
    for i in range(3):
        frame = sr.colour_frame(h, w, i)
        crop = sr.crop_frame(frame, g["proj"][i], g["K"], 512)["image"]
        assert crop.shape == (512, 512, 3)
        assert ref.encode(crop) == cv2_png(crop)
        filt = ref.filtered(crop)
        assert ref.emulate_zlib(filt) == ref.zlib_stream(filt)


def test_width_one_rows_are_not_filtered():
    img = np.arange(40, dtype=np.uint8).reshape(40, 1) * 7
    filt = ref.filtered(img)
    assert (filt[:, 0] == 0).all() and (filt[:, 1] == img[:, 0]).all()
    assert ref.encode(img) == cv2_png(img)
    wide = np.repeat(img, 2, axis=1)
    assert (ref.filtered(wide)[:, 0] == 1).all()
    assert ref.encode(wide) == cv2_png(wide)


def test_strided_views():
    rng = np.random.default_rng(7)
    big = rng.integers(0, 256, (90, 120, 4), dtype=np.uint8)
    big[:, :50] = big[:1, :50]
    for view in (big[3:80:2, 5:100:3, :3], big[::-1, ::2, 1], big[10:60, 7:90, [2, 0, 1]], big[:, :, :]):
        assert ref.encode(view) == cv2_png(np.ascontiguousarray(view)) == cv2_png(view)


def test_window_and_header_rules():
    """png_deflate_claim's window (with +262) and optimize_cmf's CINFO (without, halved at least once when the data fits the
    window) differ; zlib runs window 8 as 9.  cv2's own header bytes decide."""
    assert ref.window_bits(16385) == 15 and ref.window_bits(16384) == 15 and ref.window_bits(8000) == 14
    assert ref.window_bits(250) == 9 and ref.window_bits(2) == 9
    for n, cinfo in [(8000, 5), (8192, 5), (8193, 6), (200, 0), (16384, 6), (16385, 7)]:
        img = np.zeros((1, n - 1), np.uint8)
        z = ref.zlib_stream(ref.filtered(img))
        assert z[0] >> 4 == cinfo and z[0] & 15 == 8, n
        assert ((z[0] << 8) | z[1]) % 31 == 0
        assert cv2_png(img)[41:43] == z[:2], n
    # without optimize_cmf zlib's header (CINFO = window - 8) differs from cv2's in the header only
    img = np.zeros((1, 7999), np.uint8)
    filt = ref.filtered(img)
    co = zlib.compressobj(1, zlib.DEFLATED, ref.window_bits(filt.size), 8, zlib.Z_RLE)
    raw = co.compress(filt.tobytes()) + co.flush()
    assert raw[0] >> 4 == 6 and raw[:2] != ref.zlib_stream(filt)[:2] and raw[2:] == ref.zlib_stream(filt)[2:]
    assert ref.encode(img) == cv2_png(img)


def test_idat_chunks_of_8192_bytes():
    img = np.random.default_rng(2).integers(0, 256, (100, 300, 3), dtype=np.uint8)
    data = cv2_png(img)
    pos, sizes = 33, []
    while True:
        (n,) = struct.unpack(">I", data[pos:pos + 4])
        kind = data[pos + 4:pos + 8]
        if kind == b"IEND":
            break
        assert kind == b"IDAT"
        sizes.append(n)
        pos += 12 + n
    assert all(s == 8192 for s in sizes[:-1]) and 0 < sizes[-1] <= 8192 and len(sizes) > 5
    assert len(data) <= ref.png_bound(ref.filtered(img).size)


def test_fibonacci_frequencies_reach_the_length_repair():
    """Literal counts in the Fibonacci sequence make zlib's Huffman tree deeper than 15 bits: gen_bitlen's repair runs and the
    emulation follows it."""
    img = ref.fibonacci_row()
    filt = ref.filtered(img)
    d = filt[0, 1:]
    assert (d[1:] != d[:-1]).all()
    lfreq = np.bincount(filt.reshape(-1), minlength=286)
    lfreq[256] = 1
    free, _, _, _ = ref.build_tree(lfreq, ref.STATIC_LLEN, ref.EXTRA_LBITS, 257, 40)
    lens, _, _, _ = ref.build_tree(lfreq, ref.STATIC_LLEN, ref.EXTRA_LBITS, 257, 15)
    assert free.max() > 15 and lens.max() == 15
    assert np.sum(2.0 ** -lens[lens > 0]) == 1.0
    assert ref.emulate_zlib(filt) == ref.zlib_stream(filt)
    assert ref.encode(img) == cv2_png(img)


def test_stored_fixed_and_dynamic_blocks_all_occur():
    """Noise frames store most blocks; smooth ones use dynamic trees; tiny ones use the fixed codes."""
    def types(img):
        z = ref.zlib_stream(ref.filtered(img))
        return z[2] >> 1 & 3                      # the first block's type
    rng = np.random.default_rng(0)
    assert types(rng.integers(0, 256, (200, 200, 3), dtype=np.uint8)) == 0
    assert types(content("gradient", (200, 200, 3), rng)) == 2
    assert types(np.zeros((2, 2), np.uint8)) == 1


def test_planted_defects_break_equality():
    img = content("levels", (64, 64, 3), np.random.default_rng(9))
    filt = ref.filtered(img)
    want = ref.zlib_stream(filt)
    assert ref.emulate_zlib(filt) == want
    orig = ref.BLOCK_SYMBOLS
    try:
        ref.BLOCK_SYMBOLS = 4000                  # a wrong block size
        assert ref.emulate_zlib(filt) != want
    finally:
        ref.BLOCK_SYMBOLS = orig
    swapped = filt.copy()
    swapped[0, 1], swapped[0, 3] = filt[0, 3], filt[0, 1]     # RGB left as BGR
    assert filt[0, 1] == filt[0, 3] or ref.frame_png(ref.zlib_stream(swapped), 64, 64, 3) != cv2_png(img)
