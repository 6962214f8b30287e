"""The device PNG encoder (csrc/png.cu, onepose_b200.png) against the byte model and cv2.imencode: grey, BGR and BGRA frames of
every kind in the model's sweep, padded and strided frames, batches against single frames, full camera frames, a poisoned
workspace and output, and a caller's stream."""
import ctypes as C

import cv2
import numpy as np
import pytest
import torch

from onepose_b200 import _lib, png
from tests import png_reference as ref

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _content(kind, shape, rng):
    H, W = shape[:2]
    if kind == "noise":
        return rng.integers(0, 256, shape, dtype=np.uint8)
    if kind == "flat":
        return np.full(shape, 77, np.uint8)
    if kind == "levels":
        return (rng.integers(0, 3, shape) * 100).astype(np.uint8)
    if kind == "gradient":
        g = (np.arange(H)[:, None] + 3 * np.arange(W)[None, :]).astype(np.uint8)
        return np.ascontiguousarray(np.broadcast_to(g.reshape(H, W, *([1] * (len(shape) - 2))), shape))
    if kind == "columns":
        c = rng.integers(0, 256, (1, W) + shape[2:], dtype=np.uint8)
        return np.ascontiguousarray(np.broadcast_to(c, shape))
    if kind == "ramp":          # SUB rows of 1s: runs that cross rows
        g = (np.arange(W)[None, :] + 1 + np.zeros((H, 1), np.int64)).astype(np.uint8)
        return np.ascontiguousarray(np.broadcast_to(g.reshape(H, W, *([1] * (len(shape) - 2))), shape))
    raise ValueError(kind)


def _bytes(buf, sizes, f=0):
    n = int(sizes[f])
    assert n > 0
    return buf[f, :n].cpu().numpy().tobytes()


SIZES = [(1, 1), (1, 9), (9, 1), (2, 2), (7, 13), (64, 64), (33, 257), (300, 300)]
KINDS = ["noise", "flat", "levels", "gradient", "columns", "ramp"]


@pytest.mark.parametrize("C", [1, 3, 4])
@pytest.mark.parametrize("kind", KINDS)
def test_sweep_equals_model_and_cv2(C, kind):
    rng = np.random.default_rng(10 * KINDS.index(kind) + C)
    for H, W in SIZES:
        img = _content(kind, (H, W) if C == 1 else (H, W, C), rng)
        want = cv2.imencode(".png", img)[1].tobytes()
        assert ref.encode(img) == want
        buf, sizes = png.encode(torch.from_numpy(img).to(DEV).unsqueeze(0))
        assert _bytes(buf, sizes) == want, (H, W, C, kind)


@pytest.mark.parametrize("shape", [(512, 512, 3), (1440, 1920, 3), (1440, 1920), (600, 800, 4)])
@pytest.mark.parametrize("kind", ["noise", "gradient", "levels"])
def test_camera_frames_and_crops(shape, kind):
    img = _content(kind, shape, np.random.default_rng(5))
    want = cv2.imencode(".png", img)[1].tobytes()
    got = png.imencode(torch.from_numpy(img).to(DEV))
    assert got.tobytes() == want
    dec = cv2.imdecode(got, cv2.IMREAD_UNCHANGED)
    assert np.array_equal(dec, img)


def test_fibonacci_symbol_counts_reach_the_length_repair():
    img = ref.fibonacci_row()                 # a literal tree deeper than 15 bits before zlib's repair
    buf, sizes = png.encode(torch.from_numpy(img).to(DEV).unsqueeze(0))
    assert _bytes(buf, sizes) == cv2.imencode(".png", img)[1].tobytes()


@pytest.mark.parametrize("C", [1, 3, 4])
def test_batch_of_32_equals_frames_one_by_one_and_cv2(C):
    rng = np.random.default_rng(C)
    kinds = KINDS * 6
    imgs = np.stack([_content(kinds[i], (45, 70) if C == 1 else (45, 70, C), rng) for i in range(32)])
    buf, sizes = png.encode(torch.from_numpy(imgs).to(DEV))
    for f in range(32):
        one, s1 = png.encode(torch.from_numpy(imgs[f]).to(DEV).unsqueeze(0))
        want = cv2.imencode(".png", imgs[f])[1].tobytes()
        assert _bytes(buf, sizes, f) == _bytes(one, s1) == want, f


@pytest.mark.parametrize("C", [1, 3, 4])
def test_padded_rows_and_strided_frames(C):
    rng = np.random.default_rng(10 + C)
    big = torch.from_numpy(rng.integers(0, 256, (8, 50, 90, C), dtype=np.uint8)).to(DEV)
    big[:, :, :40] = big[:, :1, :40]                                  # runs as well as noise
    view = big[::2, 3:43, 5:66]                                       # padded rows, strided frames
    if C == 1:
        view = view[..., 0]
    buf, sizes = png.encode(view)
    for f in range(view.shape[0]):
        img = view[f].cpu().numpy()
        assert _bytes(buf, sizes, f) == cv2.imencode(".png", img)[1].tobytes(), f
    # frame stride 0: one frame for all F
    one = big[0, :30, :30]
    rep = one.unsqueeze(0).expand(4, *one.shape)
    buf, sizes = png.encode(rep[..., 0] if C == 1 else rep)
    want = cv2.imencode(".png", one.cpu().numpy()[..., 0] if C == 1 else one.cpu().numpy())[1].tobytes()
    for f in range(4):
        assert _bytes(buf, sizes, f) == want


def _raw_encode(frames, ws_fill, out_fill, stream=None):
    F, H, W, Ch = frames.shape
    lib = _lib.load()
    ws = C.c_int64()
    _lib.check(lib.opb_png_workspace_bytes(F, H, W, Ch, C.byref(ws)))
    slot = png.frame_bytes(H, W, Ch)
    workspace = torch.full((ws.value,), ws_fill, dtype=torch.uint8, device=DEV)
    out = torch.full((F, slot), out_fill, dtype=torch.uint8, device=DEV)
    sizes = torch.full((F,), -7, dtype=torch.int64, device=DEV)
    st = stream if stream is not None else torch.cuda.current_stream()
    rc = lib.opb_png_encode(frames.data_ptr(), frames.stride(0), frames.stride(1), F, H, W, Ch, workspace.data_ptr(), ws.value,
                            out.data_ptr(), slot, sizes.data_ptr(), st.cuda_stream)
    _lib.check(rc)
    torch.cuda.synchronize()
    return out, sizes


def test_poisoned_workspace_and_output_change_nothing():
    rng = np.random.default_rng(4)
    imgs = np.stack([_content(k, (120, 200, 3), rng) for k in KINDS])
    frames = torch.from_numpy(imgs).to(DEV)
    a, sa = _raw_encode(frames, 0, 0)
    b, sb = _raw_encode(frames, 0xFF, 0xA5)
    assert torch.equal(sa, sb)
    for f in range(len(KINDS)):
        n = int(sa[f])
        assert torch.equal(a[f, :n], b[f, :n])
        assert bool((b[f, n:] == 0xA5).all()), "bytes past the file were written"
        assert a[f, :n].cpu().numpy().tobytes() == cv2.imencode(".png", imgs[f])[1].tobytes()


def test_non_default_stream_equals_default_stream():
    rng = np.random.default_rng(6)
    frames = torch.from_numpy(np.stack([_content(k, (200, 300, 4), rng) for k in KINDS])).to(DEV)
    a, sa = _raw_encode(frames, 0, 0)
    s = torch.cuda.Stream()
    busy = torch.empty(1 << 26, device=DEV)
    with torch.cuda.stream(s):
        busy.normal_()                       # the stream is busy when the encode is enqueued behind it
        b, sb = _raw_encode(frames, 3, 3, stream=s)
    assert torch.equal(sa, sb)
    for f in range(len(KINDS)):
        assert torch.equal(a[f, :int(sa[f])], b[f, :int(sb[f])])


def test_imwrite_writes_cv2s_files(tmp_path):
    rng = np.random.default_rng(8)
    imgs = np.stack([_content(k, (64, 96, 3), rng) for k in KINDS])
    paths = [tmp_path / f"{i}.png" for i in range(len(KINDS))]
    png.imwrite(paths, torch.from_numpy(imgs).to(DEV))
    for p, img in zip(paths, imgs):
        cv2.imwrite(str(p) + ".cv2.png", img)
        assert p.read_bytes() == open(str(p) + ".cv2.png", "rb").read()
