"""Refusals of the PNG reader's entry points: OPB_E_INVALID with a message that names the entry point and the refused condition,
before any CUDA call (so no GPU is needed), and the Python layer's ValueError for flags, buffers and shapes."""
import ctypes as C

import pytest
import torch

from onepose_b200 import _lib, png

OPB_E_INVALID = -1
P = 256
BIG = 1 << 40


def _decode(**kw):
    a = dict(data=P, offsets=P, F=2, H=3, W=5, mode=0, workspace=P, workspace_bytes=BIG, out=P, out_frame_pitch=15, out_row_pitch=5,
             image=None, status=P, stream=None)
    a.update(kw)
    return tuple(a.values())


CASES = [
    (_decode(data=None), "data && offsets && workspace && out && status"),
    (_decode(offsets=None), "data && offsets && workspace && out && status"),
    (_decode(status=None), "data && offsets && workspace && out && status"),
    (_decode(F=0), "F > 0 && F <= OPB_PNG_MAX_FRAMES"),
    (_decode(F=65536), "F > 0 && F <= OPB_PNG_MAX_FRAMES"),
    (_decode(H=0), "H > 0 && W > 0"),
    (_decode(W=-1), "H > 0 && W > 0"),
    (_decode(H=20000, W=20000), "(int64_t)H * (1 + 4 * (int64_t)W) <= opb::kMaxFilteredBytes"),
    (_decode(mode=2), "mode == OPB_PNG_READ_GREY || mode == OPB_PNG_READ_BGR"),
    (_decode(mode=1, image=P, out_row_pitch=15, out_frame_pitch=45), "image == nullptr || mode == OPB_PNG_READ_GREY"),
    (_decode(out_row_pitch=4), "out_row_pitch >= (int64_t)W * px"),
    (_decode(mode=1, out_row_pitch=5), "out_row_pitch >= (int64_t)W * px"),
    (_decode(out_frame_pitch=14), "out_frame_pitch >= (int64_t)H * out_row_pitch"),
    (_decode(workspace=P + 16), "((uintptr_t)workspace & 255) == 0"),
    (_decode(workspace_bytes=100), "workspace_bytes >= (int64_t)L.total"),
]


@pytest.mark.parametrize("args,cond", CASES)
def test_decode_refused_with_a_message(args, cond):
    lib = _lib.load()
    assert lib.opb_png_decode(*args) == OPB_E_INVALID
    msg = lib.opb_last_error(None).decode()
    assert msg.startswith("opb_png_decode:") and cond in msg, msg


@pytest.mark.parametrize("args", [(0, 4, 4, 10), (65536, 4, 4, 10), (1, 0, 4, 10), (1, 4, 0, 10), (1, 4, 4, -1), (1, 20000, 20000, 10)])
def test_workspace_query_refuses_bad_arguments(args):
    lib = _lib.load()
    out = C.c_int64(-5)
    assert lib.opb_png_decode_workspace_bytes(*args, C.byref(out)) == OPB_E_INVALID
    assert lib.opb_last_error(None).decode().startswith("opb_png_decode_workspace_bytes:")
    assert out.value == -5
    assert lib.opb_png_decode_workspace_bytes(1, 4, 4, 10, None) == OPB_E_INVALID


def test_workspace_grows_with_the_files():
    lib = _lib.load()
    a, b = C.c_int64(), C.c_int64()
    assert lib.opb_png_decode_workspace_bytes(2, 8, 8, 100, C.byref(a)) == 0
    assert lib.opb_png_decode_workspace_bytes(2, 8, 8, 100000, C.byref(b)) == 0
    assert b.value - a.value >= 100000 - 100 - 255


@pytest.mark.parametrize("flags", [-1, 2, 4, 1.0, None, True])
def test_flags_other_than_grey_and_colour_raise(flags, tmp_path):
    with pytest.raises(ValueError, match="flags"):
        png.imread([tmp_path / "a.png"], flags)
    with pytest.raises(ValueError, match="flags"):
        png.imdecode(b"", flags)
    with pytest.raises(ValueError, match="flags"):
        png.decode(torch.zeros(8, dtype=torch.uint8), torch.zeros(2, dtype=torch.int64), 1, 1, flags)


def test_decode_argument_errors():
    d, o = torch.zeros(8, dtype=torch.uint8), torch.tensor([0, 8])
    with pytest.raises(ValueError, match="normalised"):
        png.decode(d, o, 1, 1, png.IMREAD_COLOR, normalised=True)
    with pytest.raises(ValueError, match="data"):
        png.decode(d.float(), o, 1, 1, png.IMREAD_GRAYSCALE)
    with pytest.raises(ValueError, match="data"):
        png.decode(torch.zeros(2, 4, dtype=torch.uint8), o, 1, 1, png.IMREAD_GRAYSCALE)
    with pytest.raises(ValueError, match="offsets"):
        png.decode(d, o.int(), 1, 1, png.IMREAD_GRAYSCALE)
    with pytest.raises(RuntimeError, match="CUDA device"):
        png.decode(d, o, 1, 1, png.IMREAD_GRAYSCALE)


def test_imread_refuses_files_on_the_host(tmp_path):
    from tests import png_decode_reference as ref
    import numpy as np
    import zlib
    z = zlib.compress(bytes(4 * 5))
    a, b, c, d = (tmp_path / f"{k}.png" for k in "abcd")
    a.write_bytes(ref.png_file(4, 4, 0, z))
    b.write_bytes(ref.png_file(4, 5, 0, z))
    c.write_bytes(b"not a png at all, but long enough to hold an IHDR")
    d.write_bytes(ref.SIGNATURE + ref.ihdr(4, 4, 0, depth=16) + ref.chunk(b"IEND", b""))
    with pytest.raises(ValueError, match="at least one"):
        png.imread([], png.IMREAD_GRAYSCALE)
    with pytest.raises(ValueError, match="5 x 4, the first file 4 x 4"):
        png.imread([a, b], png.IMREAD_GRAYSCALE)
    with pytest.raises(ValueError, match="not a PNG"):
        png.imread([a, c], png.IMREAD_GRAYSCALE)
    with pytest.raises(ValueError, match="unsupported PNG format: bit depth 16"):
        png.imread([d], png.IMREAD_COLOR)
    assert png.imdecode(np.frombuffer(b"garbage", np.uint8), png.IMREAD_COLOR) is None
