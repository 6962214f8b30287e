"""The device PNG reader (csrc/png_decode.cu, onepose_b200.png.decode / imdecode / imread) against cv2.imdecode and the models of
tests/png_decode_reference.py: pixels in both modes over the corpus, statuses of malformed files with untouched outputs and a
poisoned workspace, batches against single files, round trips through the encoder and the scan's crops, and a caller's busy
stream and second device."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

cv2 = pytest.importorskip("cv2")

from onepose_b200 import _lib, frames, png, scan  # noqa: E402
from tests import png_decode_reference as ref  # noqa: E402
from tests import scan_reference as sr  # noqa: E402
from tests.golden_util import GOLDEN_DIR  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _pack(files, dev=DEV):
    offsets = np.zeros(len(files) + 1, np.int64)
    offsets[1:] = np.cumsum([len(f) for f in files])
    data = torch.from_numpy(np.frombuffer(b"".join(files), np.uint8).copy()).to(dev)
    return data, torch.from_numpy(offsets).to(dev)


def _raw(files, H, W, mode, ws_fill=0xA5, out_fill=0x5A, pad=7, image=False, stream=None, dev=DEV):
    """opb_png_decode with a poisoned workspace and padded output rows and frames."""
    F = len(files)
    data, offsets = _pack(files, dev)
    px = 1 if mode == 0 else 3
    ws = C.c_int64()
    _lib.check(_lib.load().opb_png_decode_workspace_bytes(F, H, W, data.numel(), C.byref(ws)))
    workspace = torch.full((ws.value,), ws_fill, dtype=torch.uint8, device=dev)
    rp, fp = W * px + pad, (W * px + pad) * H + pad
    out = torch.full((F * fp,), out_fill, dtype=torch.uint8, device=dev)
    img = torch.full((F, 1, H, W), -1.0, device=dev) if image else None
    status = torch.full((F,), -9, dtype=torch.int32, device=dev)
    st = stream if stream is not None else torch.cuda.current_stream(dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.load().opb_png_decode(data.data_ptr(), offsets.data_ptr(), F, H, W, mode, workspace.data_ptr(), ws.value,
                                              out.data_ptr(), fp, rp, img.data_ptr() if image else None, status.data_ptr(),
                                              st.cuda_stream))
    return out, fp, rp, img, status


def _pixels(out, fp, rp, f, H, W, px):
    o = out[f * fp:(f + 1) * fp].cpu().numpy()
    return np.stack([o[y * rp:y * rp + W * px] for y in range(H)]).reshape((H, W) if px == 1 else (H, W, 3)), o


@pytest.fixture(scope="module")
def corpus():
    rng = np.random.default_rng(2026)
    return ref.cv2_corpus(rng) + ref.zlib_corpus(rng)


def test_corpus_equals_cv2_in_both_modes(corpus):
    for name, buf in corpus:
        W, H = (int(v) for v in np.frombuffer(buf[16:24], ">u4"))
        for mode in (0, 1):
            out, fp, rp, img, status = _raw([buf], H, W, mode, image=mode == 0)
            assert int(status[0]) == ref.OK, name
            got, o = _pixels(out, fp, rp, 0, H, W, 1 if mode == 0 else 3)
            want = cv2.imdecode(np.frombuffer(buf, np.uint8), mode)
            np.testing.assert_array_equal(got, want, err_msg=f"{name} mode {mode}")
            if mode == 0:
                assert torch.equal(img.cpu(), torch.from_numpy(want).float()[None, None] / 255), name


@pytest.mark.parametrize("C", [1, 3, 4])
def test_full_frames_and_crops_equal_cv2(C):
    rng = np.random.default_rng(40 + C)
    for H, W in [(512, 512), (1440, 1920)]:
        img = ref.image(rng, H, W, C)
        for p in ([], [cv2.IMWRITE_PNG_COMPRESSION, 9], [cv2.IMWRITE_PNG_COMPRESSION, 0]):
            buf = cv2.imencode(".png", img if C > 1 else img[..., 0], p)[1].tobytes()
            for flags in (cv2.IMREAD_GRAYSCALE, cv2.IMREAD_COLOR):
                got = png.imdecode(buf, flags)
                np.testing.assert_array_equal(got, cv2.imdecode(np.frombuffer(buf, np.uint8), flags), err_msg=f"{H}x{W}x{C} {p}")


def test_malformed_statuses_and_untouched_outputs():
    for name, buf, H, W, want in ref.malformed(np.random.default_rng(5)):
        for mode in (0, 1):
            out, fp, rp, img, status = _raw([buf], H, W, mode, image=mode == 0)
            assert int(status[0]) == want, f"{name}: {int(status[0])} != {want}"
            px = 1 if mode == 0 else 3
            got, o = _pixels(out, fp, rp, 0, H, W, px)
            for y in range(H):                 # the row padding and the frame's tail are never written
                assert (o[y * rp + W * px:(y + 1) * rp] == 0x5A).all(), name
            assert (o[H * rp:] == 0x5A).all(), name
            if want == ref.OK:
                np.testing.assert_array_equal(got, ref.model_decode(buf, mode, H, W)[1], err_msg=name)
            else:
                assert (got == 0x5A).all(), name
                if mode == 0:
                    assert (img == -1.0).all(), name


def test_workspace_contents_do_not_matter(corpus):
    files = [b for _, b in corpus if b[16:24] == corpus[-1][1][16:24]]
    W, H = (int(v) for v in np.frombuffer(files[0][16:24], ">u4"))
    a = _raw(files, H, W, 1, ws_fill=0x00)
    b = _raw(files, H, W, 1, ws_fill=0xFF)
    assert torch.equal(a[0], b[0]) and torch.equal(a[4], b[4]) and (a[4] == 0).all()


def _bad_files(rng, H, W):
    """Files of the batch's shape that fail in the inflate, Adler-32 and filter checks, and in the chunk walk."""
    import zlib
    raw = ref.filter_rows(ref.image(rng, H, W, 3), rng.integers(0, 5, H))
    z = zlib.compress(raw, 6)
    d = ref.Deflater()
    d.bits(0b111, 3)
    return {
        ref.BAD_DEFLATE: ref.png_file(H, W, 2, d.stream()),
        ref.BAD_ADLER: ref.png_file(H, W, 2, z[:-1] + bytes([z[-1] ^ 1])),
        ref.TOO_LITTLE: ref.png_file(H, W, 2, zlib.compress(raw + bytes(40))[:-4], 7),
        ref.BAD_FILTER: ref.png_file(H, W, 2, zlib.compress(raw[:1 + W * 3] + b"\x07" + raw[2 + W * 3:])),
        ref.BAD_CRC: ref.png_file(H, W, 2, z)[:-16] + b"\0\0\0\0" + ref.chunk(b"IEND", b""),
    }


@pytest.mark.parametrize("F", [1, 2, 7, 32, 128])
def test_batches_equal_single_files(F):
    """Good files, files that fail in every kernel and files of another shape, side by side."""
    rng = np.random.default_rng(F)
    H, W = 23, 41
    bad = list(_bad_files(rng, H, W).items())
    other = [b for _, b, h, w, _ in ref.malformed(rng) if (h, w) == (12, 20)]
    files, want = [], []
    for f in range(F):
        if f % 3 == 1:
            st, b = bad[f // 3 % len(bad)]
        elif f % 7 == 5:
            st, b = ref.BAD_SHAPE, other[f % len(other)]
        else:
            p = [cv2.IMWRITE_PNG_COMPRESSION, int(rng.integers(0, 10))]
            st, b = ref.OK, cv2.imencode(".png", ref.image(rng, H, W, 3), p)[1].tobytes()
        files.append(b)
        want.append(st)
    for mode in (0, 1):
        out, fp, rp, _, status = _raw(files, H, W, mode)
        for f, b in enumerate(files):
            o1, fp1, rp1, _, s1 = _raw([b], H, W, mode)
            assert int(status[f]) == int(s1[0]), f
            if want[f] != ref.BAD_SHAPE:
                assert int(s1[0]) == want[f] == ref.model_decode(b, mode, H, W)[0], f
            assert torch.equal(out[f * fp:(f + 1) * fp], o1[:fp1]), f


def test_decreasing_offsets_refuse_every_file():
    img = ref.image(np.random.default_rng(1), 8, 9, 3)
    files = [cv2.imencode(".png", img)[1].tobytes()] * 3
    data, offsets = _pack(files)
    o = offsets.cpu()
    o[2] = o[1] - 1                      # file 1 ends before it starts, file 2 would overlap file 1
    grey, status = png.decode(data, o.to(DEV), 8, 9, cv2.IMREAD_GRAYSCALE)
    assert (status.cpu() == ref.NOT_PNG).all()


@pytest.mark.parametrize("C", [1, 3, 4])
def test_imread_of_imwrite_returns_the_frames(C, tmp_path):
    rng = np.random.default_rng(C)
    fr = torch.from_numpy(ref.image(rng, 5 * 64, 96, C).reshape(5, 64, 96, C)).to(DEV)
    fr = fr[..., 0] if C == 1 else fr
    paths = [tmp_path / f"{i}.png" for i in range(5)]
    png.imwrite(paths, fr)
    bgr = png.imread(paths, cv2.IMREAD_COLOR)
    want = fr[..., None].expand(-1, -1, -1, 3) if C == 1 else fr[..., :3]
    assert torch.equal(bgr, want)
    grey, image = png.imread(paths, cv2.IMREAD_GRAYSCALE, normalised=True)
    if C == 1:
        assert torch.equal(grey, fr)
    else:
        g, im = frames.grey_frames(fr, "bgr" if C == 3 else "bgra", normalised=True)
        assert torch.equal(grey, g) and torch.equal(image, im)


def test_scan_crops_round_trip(tmp_path):
    g = dict(np.load(os.path.join(GOLDEN_DIR, "pnp_scan_cases.npz"), allow_pickle=False))
    H, W = (int(v) for v in g["frame_hw"])
    fr = np.stack([sr.colour_frame(H, W, f) for f in range(int(g["n_frames"]))])
    arposes = np.array([[float(e) for e in ln.strip().split(",")] for ln in str(g["arposes_txt"]).splitlines()
                        if ln.strip() and not ln.strip().startswith("#")])
    args = [torch.from_numpy(np.ascontiguousarray(v)).to(DEV) for v in (g["K"], arposes, g["T_ow"], g["bbox3d"])]
    ann = scan.annotate(torch.from_numpy(fr).to(DEV), *args, crop_size=int(g["crop_size"]))
    paths = [tmp_path / f"{i}.png" for i in range(ann["image"].shape[0])]
    png.imwrite(paths, ann["image"])
    grey, inp = png.imread(paths, cv2.IMREAD_GRAYSCALE, normalised=True)
    g2, i2 = frames.grey_frames(ann["image"], normalised=True)
    assert torch.equal(grey, g2) and torch.equal(inp, i2)


def test_imread_names_every_failed_file(tmp_path):
    img = ref.image(np.random.default_rng(0), 12, 20, 3)
    good = cv2.imencode(".png", img)[1].tobytes()
    bad = {n: b for n, b, h, w, s in ref.malformed(np.random.default_rng(5)) if (h, w) == (12, 20) and s not in (ref.OK, ref.NOT_PNG)
           and b[:16] == good[:16] and s != ref.UNSUPPORTED}
    paths = []
    for i, b in enumerate([good] + list(bad.values()) + [good]):
        p = tmp_path / f"{i}.png"
        p.write_bytes(b)
        paths.append(p)
    with pytest.raises(_lib.OpbError) as e:
        png.imread(paths, cv2.IMREAD_COLOR)
    for p in paths[1:-1]:
        assert str(p) in str(e.value)
    assert str(paths[0]) + ":" not in str(e.value)


def test_busy_stream_and_second_device(corpus):
    files = [b for _, b in corpus[:40]]
    shapes = {b[16:24] for b in files}
    files = [b for b in files if b[16:24] == sorted(shapes)[0]]
    W, H = (int(v) for v in np.frombuffer(files[0][16:24], ">u4"))
    want = _raw(files, H, W, 1)
    s = torch.cuda.Stream(DEV)
    busy = torch.empty(1 << 26, device=DEV)
    with torch.cuda.stream(s):
        busy.normal_()
        got = _raw(files, H, W, 1, stream=s)
    s.synchronize()
    assert torch.equal(got[0], want[0]) and torch.equal(got[4], want[4])
    if torch.cuda.device_count() > 1:
        other = _raw(files, H, W, 1, dev="cuda:1")
        assert torch.equal(other[0].cpu(), want[0].cpu()) and torch.equal(other[4].cpu(), want[4].cpu())
