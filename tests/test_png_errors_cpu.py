"""Refusals of the PNG encoder's entry points: OPB_E_INVALID with a message that names the entry point and the refused condition,
before any CUDA call (so no GPU is needed), and the Python layer's ValueError for shapes, channel counts and strides."""
import ctypes as C

import pytest
import torch

from onepose_b200 import _lib, png

OPB_E_INVALID = -1
P = 256                     # a non-null, 256-byte aligned address; never dereferenced (the call is refused first)
BIG = 1 << 40


def _encode(**kw):
    a = dict(frames=P, frame_pitch=3 * 4 * 5, row_pitch=15, F=2, H=3, W=5, C=3, workspace=P, workspace_bytes=BIG, out=P,
             out_pitch=BIG, sizes=P, stream=None)
    a.update(kw)
    return tuple(a.values())


CASES = [
    ("opb_png_encode", _encode(frames=None), "frames && workspace && out && sizes"),
    ("opb_png_encode", _encode(sizes=None), "frames && workspace && out && sizes"),
    ("opb_png_encode", _encode(F=0), "F > 0 && F <= OPB_PNG_MAX_FRAMES"),
    ("opb_png_encode", _encode(F=65536), "F > 0 && F <= OPB_PNG_MAX_FRAMES"),
    ("opb_png_encode", _encode(H=0), "H > 0 && W > 0"),
    ("opb_png_encode", _encode(W=-1), "H > 0 && W > 0"),
    ("opb_png_encode", _encode(C=2), "(C == 1 || C == 3 || C == 4)"),
    ("opb_png_encode", _encode(C=0), "(C == 1 || C == 3 || C == 4)"),
    ("opb_png_encode", _encode(H=20000, W=20000, C=4, row_pitch=80000, frame_pitch=BIG), "n <= opb::kMaxFiltered"),
    ("opb_png_encode", _encode(row_pitch=14), "row_pitch >= (int64_t)W * C"),
    ("opb_png_encode", _encode(frame_pitch=44), "frame_pitch >= (int64_t)H * row_pitch"),
    ("opb_png_encode", _encode(workspace=P + 16), "((uintptr_t)workspace & 255) == 0"),
    ("opb_png_encode", _encode(workspace_bytes=1000), "workspace_bytes >= (int64_t)L.total"),
    ("opb_png_encode", _encode(out_pitch=100), "out_pitch >= opb::png_bound(n)"),
]


@pytest.mark.parametrize("name,args,cond", CASES)
def test_refused_with_a_message(name, args, cond):
    lib = _lib.load()
    rc = getattr(lib, name)(*args)
    assert rc == OPB_E_INVALID
    msg = lib.opb_last_error(None).decode()
    assert msg.startswith(name + ":") and cond in msg, msg


@pytest.mark.parametrize("args", [(0, 4, 4, 3), (1, 0, 4, 3), (1, 4, 0, 3), (1, 4, 4, 2), (65536, 4, 4, 1), (1, 20000, 20000, 4)])
def test_workspace_query_refuses_bad_shapes(args):
    lib = _lib.load()
    out = C.c_int64(-5)
    assert lib.opb_png_workspace_bytes(*args, C.byref(out)) == OPB_E_INVALID
    assert lib.opb_last_error(None).decode().startswith("opb_png_workspace_bytes:")
    assert out.value == -5
    assert lib.opb_png_workspace_bytes(1, 4, 4, 3, None) == OPB_E_INVALID


def test_frame_bytes_is_deflate_bound_plus_framing():
    from tests import png_reference as ref
    for H, W, Ch in [(1, 1, 1), (512, 512, 3), (1440, 1920, 3), (100, 100, 4), (40, 40, 1)]:
        assert png.frame_bytes(H, W, Ch) == ref.png_bound(H * (1 + W * Ch))
    with pytest.raises(_lib.OpbError, match="opb_png_frame_bytes"):
        png.frame_bytes(4, 4, 2)


@pytest.mark.parametrize("frames,match", [
    (torch.zeros(2, 4, 4, 2, dtype=torch.uint8), "uint8"),
    (torch.zeros(2, 4, 4, 3, dtype=torch.float32), "uint8"),
    (torch.zeros(4, 4, dtype=torch.uint8), "uint8"),
    (torch.zeros(0, 4, 4, 3, dtype=torch.uint8), "images"),
    (torch.zeros(2, 4, 8, 3, dtype=torch.uint8)[:, :, ::2], "packed pixels"),
    (torch.zeros(2, 4, 4, 4, dtype=torch.uint8)[..., :3], "packed pixels"),
    (torch.zeros(2, 4, 4, dtype=torch.uint8).transpose(1, 2), "packed pixels"),
    ([[0]], "torch.Tensor"),
])
def test_python_refuses_shapes_channels_and_strides(frames, match):
    with pytest.raises(ValueError, match=match):
        png.encode(frames)


def test_imencode_takes_one_frame_and_imwrite_one_path_per_frame():
    with pytest.raises(ValueError, match="uint8"):
        png.imencode(torch.zeros(1, 4, 4, 3, dtype=torch.uint8))
    with pytest.raises(ValueError, match="paths"):
        png.imwrite(["a.png"], torch.zeros(2, 4, 4, 3, dtype=torch.uint8))
