"""The PNG reader's models (tests/png_decode_reference.py) against cv2.imdecode (OpenCV 4.13) and zlib: pixels and accept / reject
on files cv2 writes at every compression level and strategy, on zlib streams of every window, strategy and row filter in any IDAT
split, on ancillary chunks, and on malformed files."""
import struct
import zlib

import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")

from tests import png_decode_reference as ref  # noqa: E402


def _cv2(buf, mode):
    return cv2.imdecode(np.frombuffer(buf, np.uint8), mode)


@pytest.fixture(scope="module")
def corpus():
    rng = np.random.default_rng(2026)
    return ref.cv2_corpus(rng) + ref.zlib_corpus(rng)


def test_model_equals_cv2_on_the_corpus(corpus):
    for name, buf in corpus:
        for mode in (ref.GREY, ref.BGR):
            st, px = ref.model_decode(buf, mode)
            assert st == ref.OK, name
            np.testing.assert_array_equal(px, _cv2(buf, mode), err_msg=name)


def test_emulated_inflate_equals_zlib_on_the_corpus(corpus):
    for name, buf in corpus:
        W, H = struct.unpack(">II", buf[16:24])
        st, C, idat, z = ref.walk_chunks(buf, H, W, ref.BGR)
        n = H * (1 + W * C)
        got_st, got = ref.inflate(z, ref.pieces(buf, idat, len(z)), n, 1 + W * C)
        assert got_st == ref.OK and got == zlib.decompress(z)[:n], name


@pytest.mark.parametrize("C", [1, 3, 4])
def test_full_frame_and_300_square(C):
    rng = np.random.default_rng(C)
    for H, W in [(300, 300), (1440, 1920)]:
        img = ref.image(rng, H, W, C)
        for p in ([], [cv2.IMWRITE_PNG_COMPRESSION, 9]):
            buf = cv2.imencode(".png", img if C > 1 else img[..., 0], p)[1].tobytes()
            for mode in (ref.GREY, ref.BGR):
                st, px = ref.model_decode(buf, mode, emulate=False)
                assert st == ref.OK
                np.testing.assert_array_equal(px, _cv2(buf, mode))


def test_malformed_files_follow_cv2():
    for name, buf, H, W, want in ref.malformed(np.random.default_rng(5)):
        st, px = ref.model_decode(buf, ref.BGR, H, W)
        assert st == want, name
        got = _cv2(buf, ref.BGR)
        if name != "other shape":        # cv2 reads the file's own shape
            assert (got is not None) == (st == ref.OK), name
        if st == ref.OK:
            np.testing.assert_array_equal(px, got, err_msg=name)


@pytest.mark.parametrize("kind,data,colour_grey_ok", [
    (b"gAMA", struct.pack(">I", 45455), False),
    (b"gAMA", struct.pack(">I", 100000), True),
    (b"sRGB", b"\x00", False),
    (b"cHRM", bytes(32), True),
    (b"sBIT", b"\x08\x08\x08", True),
    (b"bKGD", bytes(6), True),
    (b"pHYs", bytes(9), True),
])
def test_colour_chunks(kind, data, colour_grey_ok):
    rng = np.random.default_rng(9)
    for C, ct in ((1, 0), (3, 2)):
        img = ref.image(rng, 10, 13, C)
        buf = ref.png_file(10, 13, ct, zlib.compress(ref.filter_rows(img, [1] * 10)), before=ref.chunk(kind, data))
        for mode in (ref.GREY, ref.BGR):
            st, px = ref.model_decode(buf, mode)
            if C == 1 or mode == ref.BGR or colour_grey_ok:
                assert st == ref.OK
                np.testing.assert_array_equal(px, _cv2(buf, mode))
            else:
                assert st == ref.UNSUPPORTED
                # cv2 gives other grey values here: libpng's rgb_to_gray in linear light
                assert not np.array_equal(ref.convert(img, ref.GREY), _cv2(buf, mode))


def test_iccp_on_a_colour_file_read_grey_is_unsupported():
    img = ref.image(np.random.default_rng(3), 6, 7, 3)
    buf = ref.png_file(6, 7, 2, zlib.compress(ref.filter_rows(img, [0] * 6)),
                       before=ref.chunk(b"iCCP", b"x\0\0" + zlib.compress(b"not a profile")))
    assert ref.model_decode(buf, ref.GREY)[0] == ref.UNSUPPORTED
    assert ref.model_decode(buf, ref.BGR)[0] == ref.OK


def test_fuzzed_streams_follow_cv2():
    for name, buf in ref.fuzzed(np.random.default_rng(77), 1500):
        st, px = ref.model_decode(buf, ref.BGR)
        got = _cv2(buf, ref.BGR)
        assert (got is not None) == (st == ref.OK), f"{name}: status {st}"
        if st == ref.OK:
            np.testing.assert_array_equal(px, got, err_msg=name)
