"""Colour camera frames to the reference's grey frames on the GPU (onepose_b200.frames / csrc/frames.cu) against the numpy model
of cv2's IMREAD_GRAYSCALE (tests/grey_reference.py, pinned against cv2 on every colour by tests/test_grey_reference_cpu.py):
every colour in every channel order, every layout the entry point takes, the frame consumers fed from it, and the caller's
streams and devices."""
import numpy as np
import pytest
import torch

from onepose_b200 import crop, detect, frames
from tests import crop_reference as cr
from tests import grey_reference as G
from tests.golden_util import GOLDEN_DIR

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SLEEP = 1 << 29              # device cycles of torch.cuda._sleep: about 0.25 s on an H100


def _colour(F, H, W, seed):
    """F BGR frames [F, H, W, 3] with structure and noise in every channel (integers only)."""
    return np.stack([np.stack([cr.synthetic_frame(H, W, 3 * (seed + f) + c) for c in range(3)], -1) for f in range(F)])


def _want(px, order):
    g = G.grey_from_bgr(G.to_bgr(px, order))
    return g, G.normalised(g)


def _check(dev_frames, order, want_grey, out=None):
    grey, image = frames.grey_frames(dev_frames, order, out=out, normalised=True)
    F = want_grey.shape[0]
    assert grey.dtype == torch.uint8 and tuple(grey.shape) == want_grey.shape
    assert image.dtype == torch.float32 and tuple(image.shape) == (F, 1, *want_grey.shape[1:]) and image.is_contiguous()
    assert np.array_equal(grey.cpu().numpy(), want_grey)
    assert np.array_equal(image.cpu().numpy()[:, 0], G.normalised(want_grey))
    # torch's true division on the CPU; on a CUDA tensor torch divides by a scalar as a multiply by its reciprocal, which
    # differs from numpy's `/ 255.` on 126 of the 256 levels
    assert torch.equal(image[:, 0].cpu(), grey.float().cpu() / 255)
    assert torch.equal(frames.grey_frames(dev_frames, order), grey)                 # without the fp32 output: the same grey
    return grey, image


# ---- every colour ----

@pytest.mark.parametrize("order", G.ORDERS)
def test_every_colour_in_every_order(order):
    bgr = G.every_colour_bgr()
    want = G.grey_from_bgr(bgr)[None]
    alpha = np.random.default_rng(1).integers(0, 256, bgr.shape[:2], dtype=np.uint8)
    px = torch.from_numpy(G.from_bgr(bgr, order, alpha)).to(DEV)
    _check(px[None], order, want)
    _check(px, order, want)                                                              # one [H, W, C] frame


def test_normalised_is_a_true_division_not_torchs_cuda_scalar_division():
    levels = torch.arange(256, dtype=torch.uint8, device=DEV).repeat_interleave(3).view(1, 1, 256, 3)   # grey v for (v, v, v)
    grey, image = frames.grey_frames(levels, normalised=True)
    assert torch.equal(grey[0, 0], levels[0, 0, :, 0])
    assert np.array_equal(image.cpu().numpy().reshape(-1), G.normalised(np.arange(256, dtype=np.uint8)))
    assert int((grey.float() / 255 != image[:, 0]).sum()) == 126


# ---- layouts ----

@pytest.mark.parametrize("order", G.ORDERS)
def test_padded_rows_and_misaligned_starts(order):
    """Row pitches above W * C, odd ones among them, and frames starting at every byte offset mod 16: the kernel's word and
    byte paths."""
    C = len(order)
    rng = np.random.default_rng(C)
    for F, H, W, pad, offset in [(3, 17, 29, 1, 0), (2, 9, 64, 16, 0), (2, 9, 64, 0, 1), (3, 11, 13, 5, 3), (1, 7, 4, 3, 2), (2, 5, 8, 0, 15),
                                 (4, 6, 1, 2, 7)]:
        row = W * C + pad
        buf = torch.from_numpy(rng.integers(0, 256, offset + F * H * row, dtype=np.uint8)).to(DEV)
        px = buf[offset:].as_strided((F, H, W, C), (H * row, row, C, 1))
        _check(px, order, _want(px.cpu().numpy(), order)[0])


def test_frame_pitch_zero_broadcasts_one_frame():
    one = _colour(1, 37, 53, 0)
    want = np.repeat(G.grey_from_bgr(one), 6, axis=0)
    _check(torch.from_numpy(one).to(DEV).expand(6, -1, -1, -1), "bgr", want)
    _check(torch.from_numpy(one[0]).to(DEV).expand(6, -1, -1, -1), "bgr", want)


def test_frames_cut_from_a_larger_tensor_into_caller_buffers():
    big = torch.from_numpy(np.random.default_rng(5).integers(0, 256, (5, 40, 50, 4), dtype=np.uint8)).to(DEV)
    px = big[1:4, 3:31, 7:44]                                                            # [3, 28, 37, 4], every stride foreign
    want = _want(px.cpu().numpy(), "rgba")[0]
    gbig = torch.full((4, 33, 45), 7, dtype=torch.uint8, device=DEV)
    out = {"grey": gbig[1:4, 2:30, 5:42], "image": torch.full((3, 1, 28, 37), -1.0, device=DEV)}
    grey, image = _check(px, "rgba", want, out=out)
    assert grey.data_ptr() == out["grey"].data_ptr() and image.data_ptr() == out["image"].data_ptr()
    outside = torch.ones_like(gbig, dtype=torch.bool)
    outside[1:4, 2:30, 5:42] = False
    assert bool((gbig[outside] == 7).all()), "a byte outside the caller's grey view was written"
    part = _colour(1, 28, 37, 9)
    frames.grey_frames(torch.from_numpy(part).to(DEV), out={"grey": gbig[0, :28, :37][None]})
    assert np.array_equal(gbig[0, :28, :37].cpu().numpy(), G.grey_from_bgr(part[0]))


@pytest.mark.parametrize("F", [1, 2, 3, 255, 4097, 65535])
def test_frame_counts_up_to_the_bound(F):
    rng = np.random.default_rng(F)
    H, W = (2, 3) if F > 4096 else (5, 6)
    for order in ("bgr", "rgba"):
        px = rng.integers(0, 256, (F, H, W, len(order)), dtype=np.uint8)
        _check(torch.from_numpy(px).to(DEV), order, _want(px, order)[0])


@pytest.mark.parametrize("H,W", [(32767, 7), (5, 32767), (32767, 1), (1, 32767)])
def test_the_largest_side(H, W):
    rng = np.random.default_rng(H + W)
    for order in ("rgb", "bgra"):
        px = rng.integers(0, 256, (2, H, W, len(order)), dtype=np.uint8)
        _check(torch.from_numpy(px).to(DEV), order, _want(px, order)[0])


def test_refusals_reach_python_with_their_message():
    px = torch.zeros(1, 8, 8, 3, dtype=torch.uint8, device=DEV)
    with pytest.raises(ValueError, match=r"out\['grey'\] must have packed pixels"):
        frames.grey_frames(px, out={"grey": torch.zeros(1, 8, 16, dtype=torch.uint8, device=DEV)[:, :, ::2]})
    with pytest.raises(ValueError, match=r"out\['image'\] must be contiguous"):
        frames.grey_frames(px, out={"image": torch.zeros(1, 1, 8, 16, device=DEV)[..., ::2]}, normalised=True)


# ---- the frame consumers, fed from colour frames ----

def test_previous_pose_detect_from_colour_frames_equals_host_grey_frames():
    B, H, W = 4, 480, 640
    bgr = _colour(B, H, W, 20)
    host = torch.from_numpy(G.grey_from_bgr(bgr)).to(DEV)
    dev = frames.grey_frames(torch.from_numpy(bgr).to(DEV))
    assert torch.equal(dev, host)
    K = torch.tensor([[500.0, 0, 320], [0, 500, 240], [0, 0, 1]], dtype=torch.float64, device=DEV)
    pose = torch.zeros(B, 3, 4, dtype=torch.float64, device=DEV)
    pose[:, :, :3] = torch.eye(3, dtype=torch.float64)
    pose[:, :, 3] = torch.tensor([[0.0, 0, 0.6], [0.05, -0.02, 0.5], [-0.08, 0.04, 0.9], [0.02, 0.03, 0.35]], dtype=torch.float64)
    corners = torch.tensor([[x, y, z] for x in (-0.06, 0.06) for y in (-0.05, 0.05) for z in (-0.04, 0.04)], dtype=torch.float64, device=DEV)
    a = crop.previous_pose_detect(dev, K, pose, corners)
    b = crop.previous_pose_detect(host, K, pose, corners)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    assert bool(a[1].any())
    rgb = torch.from_numpy(np.ascontiguousarray(bgr[..., ::-1])).to(DEV)            # the same colours as a camera API's RGB
    for x, y in zip(crop.previous_pose_detect(frames.grey_frames(rgb, "rgb"), K, pose, corners), b):
        assert torch.equal(x, y)


def test_detect_from_matches_from_colour_frames_equals_host_grey_frames():
    g = dict(np.load(f"{GOLDEN_DIR}/pnp_detect_cases.npz", allow_pickle=False))
    H, W, _ = (int(v) for v in g["s0_frame"])
    qs = [{k: g[f"s0_q{q}_{k}"] for k in ("keypoints", "matches0")} for q in range(int(g["s0_n_queries"]))]
    ref = {k: torch.from_numpy(g[f"s0_ref_{k}"]).to(DEV) for k in ("keypoints", "counts", "sizes")}
    cap = max(max(len(q["keypoints"]) for q in qs), 1)
    kp = np.zeros((len(qs), cap, 2), np.float32)
    for b, q in enumerate(qs):
        kp[b, :len(q["keypoints"])] = q["keypoints"]
    query = {"keypoints": torch.from_numpy(kp).to(DEV), "counts": torch.tensor([len(q["keypoints"]) for q in qs], dtype=torch.int32, device=DEV)}
    m0 = torch.from_numpy(np.stack([q["matches0"] for q in qs])).to(DEV, torch.int64)
    bgr = _colour(len(qs), H, W, 40)
    K = torch.from_numpy(g["s0_K"]).to(DEV)
    a = detect.detect_from_matches(frames.grey_frames(torch.from_numpy(bgr).to(DEV)), K, ref, query, m0, crop_size=256)
    b = detect.detect_from_matches(torch.from_numpy(G.grey_from_bgr(bgr)).to(DEV), K, ref, query, m0, crop_size=256)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    assert bool(a[1].any())


# ---- the caller's streams and devices (tests/test_streams_devices_gpu.py's conventions) ----

def test_runs_on_the_callers_stream_without_synchronising():
    """The stale-input pattern: on a fresh stream the input is first written with other frames, the stream sleeps, then the real
    frames are copied in and the call is made.  A launch on any other stream would read the stale frames; the stream must still
    be asleep when the call returns."""
    real, stale = (torch.from_numpy(_colour(3, 61, 83, s)).to(DEV) for s in (1, 2))
    want = frames.grey_frames(real, normalised=True)
    buf = torch.empty_like(real)
    torch.cuda.synchronize()
    s = torch.cuda.Stream(DEV)
    asleep = torch.cuda.Event()
    with torch.cuda.stream(s):
        buf.copy_(stale)
        torch.cuda._sleep(SLEEP)
        asleep.record(s)
        buf.copy_(real)
        out = frames.grey_frames(buf, normalised=True)
        busy = not asleep.query()
    torch.cuda.synchronize()
    assert busy, "grey_frames synchronised the host with the caller's stream"
    for x, y in zip(out, want):
        assert torch.equal(x, y)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two visible GPUs")
def test_on_the_second_device():
    torch.cuda.set_device(0)
    bgr = _colour(2, 45, 67, 3)
    want = frames.grey_frames(torch.from_numpy(bgr).to("cuda:0"), normalised=True)
    got = frames.grey_frames(torch.from_numpy(bgr).to("cuda:1"), normalised=True)
    assert torch.cuda.current_device() == 0
    assert all(t.device == torch.device("cuda:1") for t in got)
    for x, y in zip(got, want):
        assert torch.equal(x.cpu(), y.cpu())
    assert np.array_equal(got[0].cpu().numpy(), G.grey_from_bgr(bgr))
