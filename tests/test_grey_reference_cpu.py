"""The grey frames the reference reads, without a GPU: tests/grey_reference.py against live OpenCV (cv2.imread(...,
IMREAD_GRAYSCALE) of a colour PNG) on every colour, the probes that settle each of its constants, and the argument checks of
frames.grey_frames and opb_grey_frames, which run before anything reaches a device."""
import numpy as np
import pytest
import torch

from onepose_b200 import _lib, frames
from tests import grey_reference as G

cv2 = pytest.importorskip("cv2")

OPB_E_INVALID = -1
P = 64                      # a non-null address; never dereferenced (the call is refused first)


def _png_grey(pixels):
    """cv2.imread(path, IMREAD_GRAYSCALE) of the PNG cv2.imwrite makes of `pixels` (BGR or BGRA), in memory."""
    ok, buf = cv2.imencode(".png", pixels, [cv2.IMWRITE_PNG_COMPRESSION, 1])
    assert ok
    return cv2.imdecode(buf, cv2.IMREAD_GRAYSCALE)


def test_cv2_is_the_version_the_model_was_probed_on():
    assert cv2.__version__.startswith("4.13"), cv2.__version__


def test_the_model_equals_cv2_on_every_colour():
    bgr = G.every_colour_bgr()
    want = _png_grey(bgr)
    got = G.grey_from_bgr(bgr)
    assert got.dtype == np.uint8 and got.shape == (4096, 4096)
    assert np.array_equal(got, want), f"{int((got != want).sum())} colours differ"
    # the decoder's grey is a function of the pixel alone: a permuted copy of the image gives the permuted map
    perm = np.random.default_rng(0).permutation(1 << 24)
    assert np.array_equal(_png_grey(bgr.reshape(-1, 3)[perm].reshape(4096, 4096, 3)).reshape(-1), want.reshape(-1)[perm])
    # a 2^14 scale does not fit: the only integer weights its one-channel ramps admit miss many colours
    b, g, r = (bgr[..., c].astype(np.int32) for c in range(3))
    for wg in (9617, 9618):
        assert int((((4899 * r + wg * g + 1869 * b) >> 14) != want).sum()) >= 130838
    # and it is not cvtColor's: one level apart on half of the colours
    diff = cv2.cvtColor(bgr, cv2.COLOR_BGR2GRAY).astype(np.int16) - want
    assert np.abs(diff).max() == 1 and int((diff != 0).sum()) == 8389722


SIZES = [(1, 1), (1, 63), (47, 1), (2, 3), (3, 2), (5, 7), (17, 29), (31, 33), (47, 63)]


@pytest.mark.parametrize("h,w", SIZES, ids=[f"{h}x{w}" for h, w in SIZES])
def test_the_model_equals_cv2_on_random_frames(h, w):
    rng = np.random.default_rng(h * 100 + w)
    for _ in range(4):
        bgr = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        assert np.array_equal(G.grey_from_bgr(bgr), _png_grey(bgr))


@pytest.mark.parametrize("order", G.ORDERS)
def test_each_channel_order_gives_the_bgr_result(order):
    rng = np.random.default_rng(7)
    bgr = rng.integers(0, 256, (29, 37, 3), dtype=np.uint8)
    alpha = rng.integers(0, 256, (29, 37), dtype=np.uint8)
    px = G.from_bgr(bgr, order, alpha)
    assert px.shape == (29, 37, len(order))
    assert np.array_equal(px[..., len(order) - 1] if order.endswith("a") else G.to_bgr(px, order), alpha if order.endswith("a") else bgr)
    assert np.array_equal(G.grey_from_bgr(G.to_bgr(px, order)), _png_grey(bgr))
    if order == "bgra":                       # the reference ignores alpha too: a BGRA PNG reads as the grey of its BGR channels
        assert np.array_equal(_png_grey(px), _png_grey(bgr))


def test_each_constant_is_settled_by_its_probe():
    """The probes DESIGN 5.11 derives the formula from, replayed: single-channel ramps bound each weight to an interval, four
    colours pick one weight from each interval, and the rounding and scale follow."""
    ramp = np.arange(256, dtype=np.int64)
    admitted = {}
    for ch, name in enumerate("BGR"):
        px = np.zeros((1, 256, 3), np.uint8)
        px[0, :, ch] = ramp
        obs = _png_grey(px)[0].astype(np.int64)
        admitted[name] = [c for c in range(1 << 15) if np.array_equal((c * ramp) >> 15, obs)]
        if name == "R":                       # no integer weight fits at >> 13, so the scale is 2^14 or finer
            assert not any(np.array_equal((c * ramp) >> 13, obs) for c in range(1 << 13))
    assert admitted == {"B": [3737, 3738], "G": [19234, 19235, 19236], "R": [9797, 9798]}
    # one colour refutes each weight above the model's: cv2 gives one level less than it would
    for bgr, refuted in [((1, 21, 236), "B = 3738"), ((0, 19, 150), "G = 19235"), ((0, 3, 158), "G = 19236"), ((0, 2, 73), "R = 9798")]:
        px = np.array(bgr, np.uint8).reshape(1, 1, 3)
        b, g, r = (int(v) for v in bgr)
        name, c = refuted.split(" = ")
        w = {"B": G.COEF_B, "G": G.COEF_G, "R": G.COEF_R}
        w[name] = int(c)
        assert int(_png_grey(px)[0, 0]) == G.grey_from_bgr(px)[0, 0] == ((w["R"] * r + w["G"] * g + w["B"] * b) >> 15) - 1, refuted
    assert G.COEF_R + G.COEF_G + G.COEF_B == 1 << G.SHIFT and int(_png_grey(np.full((1, 1, 3), 255, np.uint8))[0, 0]) == 255
    assert int(_png_grey(np.array([[[0, 1, 0]]], np.uint8))[0, 0]) == 0      # 19234 / 32768 truncates: no rounding offset
    assert int(_png_grey(np.array([[[0, 0, 255]]], np.uint8))[0, 0]) == 76   # red is the third BGR byte: 9797 * 255 >> 15
    assert int(_png_grey(np.array([[[255, 0, 0]]], np.uint8))[0, 0]) == 29   # blue the first: 3737 * 255 >> 15


def test_normalised_is_numpys_float32_division():
    g = np.arange(256, dtype=np.uint8)
    img = g.astype(np.float32)
    img /= 255.                                                              # NormalizedDataset's statement
    assert np.array_equal(G.normalised(g), img) and G.normalised(g).dtype == np.float32
    assert np.array_equal(torch.from_numpy(g).float().numpy() / np.float32(255), img)


# ---- frames.grey_frames: argument checks that run without a GPU ----

def _bgr(*shape):
    return torch.zeros(*shape, dtype=torch.uint8)


BAD_ARGS = [
    ("dtype", lambda: frames.grey_frames(_bgr(2, 8, 8, 3).float()), "uint8"),
    ("not a tensor", lambda: frames.grey_frames(np.zeros((8, 8, 3), np.uint8)), "torch.Tensor"),
    ("rank", lambda: frames.grey_frames(_bgr(8, 8)), r"\[F, H, W, 3\]"),
    ("rank 5", lambda: frames.grey_frames(_bgr(1, 2, 8, 8, 3)), r"\[F, H, W, 3\]"),
    ("channels for bgr", lambda: frames.grey_frames(_bgr(2, 8, 8, 4)), r"\[F, H, W, 3\]"),
    ("channels for rgba", lambda: frames.grey_frames(_bgr(2, 8, 8, 3), order="rgba"), r"\[F, H, W, 4\]"),
    ("order", lambda: frames.grey_frames(_bgr(2, 8, 8, 3), order="yuv"), "order must be one of"),
    ("order case", lambda: frames.grey_frames(_bgr(2, 8, 8, 3), order="BGR"), "order must be one of"),
    ("empty", lambda: frames.grey_frames(_bgr(0, 8, 8, 3)), "1..65535 images"),
    ("too many frames", lambda: frames.grey_frames(_bgr(1, 8, 8, 3).expand(65536, 8, 8, 3)), "1..65535 images"),
    ("side", lambda: frames.grey_frames(_bgr(1, 1, 1, 3).expand(1, 1, 32768, 3)), "1..32767 pixels"),
    ("planar channels", lambda: frames.grey_frames(_bgr(2, 3, 8, 8).permute(0, 2, 3, 1)), "packed pixels"),
    ("pixel stride", lambda: frames.grey_frames(_bgr(2, 8, 16, 3)[:, :, ::2]), "packed pixels"),
    ("channel subset", lambda: frames.grey_frames(_bgr(2, 8, 8, 4)[..., :3]), "packed pixels"),
    ("rows overlap", lambda: frames.grey_frames(_bgr(400).as_strided((2, 8, 8, 3), (192, 12, 3, 1))), "packed pixels"),
    ("frames overlap", lambda: frames.grey_frames(_bgr(400).as_strided((2, 8, 8, 3), (100, 24, 3, 1))), "packed pixels"),
    ("out dtype", lambda: frames.grey_frames(_bgr(2, 8, 8, 3), out={"grey": torch.zeros(2, 8, 8)}), r"out\['grey'\]"),
    ("out shape", lambda: frames.grey_frames(_bgr(2, 8, 8, 3), out={"grey": _bgr(2, 8, 9)}), r"out\['grey'\]"),
    ("out image shape", lambda: frames.grey_frames(_bgr(2, 8, 8, 3), out={"image": torch.zeros(2, 8, 8)}, normalised=True),
     r"out\['image'\]"),
]


@pytest.mark.parametrize("what,call,msg", BAD_ARGS, ids=[b[0] for b in BAD_ARGS])
def test_grey_frames_argument_mistakes_raise_value_error(what, call, msg):
    with pytest.raises(ValueError, match=msg):
        call()


def test_grey_frames_accepts_what_the_checks_allow_then_needs_a_device():
    """Layouts the checks accept -- padded rows, a frame stride of 0, a single [H, W, C] frame, frames cut from a larger tensor --
    reach the device check, which a CPU tensor fails."""
    big = _bgr(4, 20, 30, 4)
    for ok, order in [(_bgr(8, 8, 3), "bgr"), (_bgr(1, 8, 8, 3).expand(5, 8, 8, 3), "rgb"), (big[1:3, 2:10, 3:20], "bgra"),
                      (_bgr(3, 8, 9, 4)[:, :, :7], "rgba"), (_bgr(2, 1, 1, 3), "bgr")]:
        with pytest.raises(RuntimeError, match="no CPU path"):
            frames.grey_frames(ok, order)


# ---- opb_grey_frames: refusals with a message, in tests/test_no_handle_errors_cpu.py's pattern ----

def _args(**kw):
    """The arguments of opb_grey_frames and the stream: two 8 x 8 BGR frames, packed, with the given ones replaced."""
    a = dict(frames=P, frame_pitch=192, row_pitch=24, F=2, H=8, W=8, order=0, grey=P, grey_frame_pitch=64, grey_row_pitch=8, image=None,
             stream=None)
    a.update(kw)
    return tuple(a.values())


REFUSALS = [
    (_args(frames=None), "frames && grey"),
    (_args(grey=None), "frames && grey"),
    (_args(F=0), "F > 0"),
    (_args(F=65536), "F <= opb::kMaxFrames"),
    (_args(H=0), "H > 0"),
    (_args(W=32768, row_pitch=32768 * 3, frame_pitch=0, grey_row_pitch=32768, grey_frame_pitch=8 * 32768), "W <= opb::kMaxSide"),
    (_args(H=32768, frame_pitch=0, grey_frame_pitch=32768 * 8), "H <= opb::kMaxSide"),
    (_args(order=-1), "order >= OPB_ORDER_BGR"),
    (_args(order=4), "order <= OPB_ORDER_RGBA"),
    (_args(row_pitch=23), "row_pitch >= (int64_t)W * C"),
    (_args(order=2, row_pitch=24, frame_pitch=256), "row_pitch >= (int64_t)W * C"),
    (_args(frame_pitch=191), "frame_pitch == 0 || frame_pitch >= (int64_t)H * row_pitch"),
    (_args(frame_pitch=-1), "frame_pitch == 0 || frame_pitch >= (int64_t)H * row_pitch"),
    (_args(grey_row_pitch=7), "grey_row_pitch >= W"),
    (_args(grey_frame_pitch=63), "grey_frame_pitch >= (int64_t)H * grey_row_pitch"),
    (_args(grey_frame_pitch=0), "grey_frame_pitch >= (int64_t)H * grey_row_pitch"),
]


@pytest.mark.parametrize("args,cond", REFUSALS, ids=[c for _, c in REFUSALS])
def test_a_refused_grey_frames_call_names_its_entry_point_and_condition(args, cond):
    lib = _lib.load()
    assert lib.opb_grey_frames(*args) == OPB_E_INVALID
    for msg in (lib.opb_last_error(None), lib.opb_sp_last_error(None)):
        assert msg.startswith(b"opb_grey_frames: "), msg
        assert cond.encode() in msg, (cond, msg)
