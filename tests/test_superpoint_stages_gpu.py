"""Every stage of the SuperPoint extractor against its fp64 stage reference (tests/superpoint_stage_reference.py), on the
device's own input to that stage: the call is stopped after each encoder step (opb_sp_debug_set_stop) and the activation
read back (debug_read(4)); the heads, dense scores and NMS output are read after a full call, the key points, scores,
descriptors and counts come from forward_padded.  The references run in fp64 on the GPU.

Bars (R.check), from the operand formats; each measured error is printed as a multiple of its bar:
  conv1a                 2^-20 sum|w||x| + 2^-22 |ref| + 2^-30          (nine fp32 FMAs, output split)
  3x3 convolutions       (2^-21 + K 2^-26) sum|w||x| + 2^-22 |ref| + 2^-30   (operand split and dropped lo.lo, the truncating
                         accumulator over K = 9 C_in, output split); border and padding rows exactly 0
  convPb, convDb         (2^-21 + 256 x 2^-26) sum|w||x| + 2^-30
  pooling, NMS, selection, top-k, counts    bit-exact
  dense scores           2^-20 relative + 2^-30;   descriptors   2^-19 absolute
Besides: batch independence at the benchmarked shape, a poisoned workspace, one handle across shape changes, and the range
guard of the fp16-split operands (an activation past 1023 is reported, never turned into silent zeros)."""
import numpy as np
import pytest
import torch

from onepose_b200 import SuperPoint, _lib, synthetic
from oracle import superpoint_oracle as O
from tests import superpoint_stage_reference as R

pytestmark = pytest.mark.gpu

RELEASED = {"nms_radius": 3, "keypoint_threshold": 0.005, "max_keypoints": 4096, "remove_borders": 4}
SCORE_TOL, DESC_TOL = 2e-5, 1e-5


def _module(sd, conf, align_corners=True):
    m = SuperPoint(conf, align_corners=align_corners).eval()
    m.load_state_dict({k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in sd.items()}, strict=True)
    return m.cuda()


def _images(seeds, H, W):
    return torch.from_numpy(np.stack([synthetic.make_image(i, H, W) for i in seeds], 0)).cuda()


def _cfg(conf):
    return {**O.DEFAULT_CONFIG, **conf}


def device_result(m, img, cap, stages=True):
    """The extractor's result in the layout of R.check: per-step activations (stop hook), heads, scores, NMS, outputs."""
    B, _, H, W = img.shape
    act = []
    m.forward_padded(img, cap)                      # creates the handle and loads the weights
    if stages:
        for i in range(12):
            m.debug_stop_after(i)
            m.forward_padded(img, cap)
            _, _, P = R.stage(H, W, R.LEVEL[i])
            act.append(m.debug_read(4, B * P * R.CHANNELS[i]).reshape(B * P, R.CHANNELS[i]).clone())
        m.debug_stop_after(-1)
    out = m.forward_padded(img, cap)
    _, _, P3 = R.stage(H, W, 3)
    torch.cuda.synchronize()
    m.check_range()
    return {"image": img[:, 0], "act": act, "logits": m.debug_read(2, B * P3 * 128).reshape(B * P3, 128).clone(),
            "ddesc": m.debug_read(3, B * P3 * 256).reshape(B * P3, 256).clone(), "scores": m.debug_read(0, B * H * W).reshape(B, H, W).clone(),
            "nms": m.debug_read(1, B * H * W).reshape(B, H, W).clone(), "kpts": out["keypoints"], "kscores": out["scores"],
            "desc": out["descriptors"], "counts": out["counts"]}


def _check(m, img, sd, conf, cap, tag, align_corners=True, stages=None):
    dev = device_result(m, img, cap, stages is None)
    r = R.check(dev, R.params64(sd, "cuda"), _cfg(conf), align_corners, stages)
    print(R.table(r, tag))
    bad = {k: v for k, v in r.items() if not v <= 1}
    assert not bad, f"{tag}: stages over their bars: {bad}"
    return dev


def _same(a, b, tag):
    n = a["counts"].tolist()
    assert n == b["counts"].tolist(), (tag, n, b["counts"].tolist())
    for i, c in enumerate(n):
        assert torch.equal(a["keypoints"][i, :c], b["keypoints"][i, :c]), (tag, i)
        assert torch.equal(a["scores"][i, :c], b["scores"][i, :c]), (tag, i)
        assert torch.equal(a["descriptors"][i, :, :c], b["descriptors"][i, :, :c]), (tag, i)


# ----------------------------------------------------------------------------- stage by stage
@pytest.mark.parametrize("halo", [1, 0])
def test_bench_shape_stages(halo):
    """8 x 512 x 512, the benchmarked images and weights, released configuration: multi-tile 128-channel stages and heads, a
    rank over ~4 500 - 5 000 candidates per image; both ways of staging the 64-channel convolutions; both align_corners."""
    lib = _lib.load()
    sd = synthetic.make_superpoint_state_dict(0, 4.0)
    img = _images(range(100, 108), 512, 512)
    try:
        assert lib.opb_debug_set_conv_halo(halo) == 0
        dev = _check(_module(sd, RELEASED), img, sd, RELEASED, 4096, f"bench halo {halo}")
        assert min(dev["counts"].tolist()) == 4096                   # every image has more candidates than k
        _check(_module(sd, RELEASED, align_corners=False), img, sd, RELEASED, 4096, f"bench halo {halo} ac0", False, ["select", "sample"])
    finally:
        lib.opb_debug_set_conv_halo(1)


@pytest.mark.parametrize("k", [-1, 1000])
def test_vga_stages(k):
    """2 x 480 x 640, r 4, remove_borders 0: non-square, key points on the outermost pixels."""
    sd = synthetic.make_superpoint_state_dict(2, 4.0)
    conf = {"nms_radius": 4, "max_keypoints": k, "remove_borders": 0}
    dev = _check(_module(sd, conf), _images((30, 31), 480, 640), sd, conf, 20000 if k < 0 else k, f"vga k {k}")
    kp = torch.cat([dev["kpts"][b, :n] for b, n in enumerate(dev["counts"].tolist())])
    if k < 0:
        assert bool(((kp[:, 0] == 0) | (kp[:, 0] == 639) | (kp[:, 1] == 0) | (kp[:, 1] == 479)).any()), "no key point on the outermost pixels"


@pytest.mark.parametrize("shape", [(3, 8, 8), (2, 8, 1024), (2, 1024, 8)])
@pytest.mark.parametrize("r", [0, 6])
def test_thin_stages(shape, r):
    """Coarse grids of height or width 1."""
    B, H, W = shape
    sd = synthetic.make_superpoint_state_dict(1, 4.0)
    conf = {"nms_radius": r, "max_keypoints": -1, "remove_borders": 0, "keypoint_threshold": 0.001}
    _check(_module(sd, conf), _images(range(40, 40 + B), H, W), sd, conf, H * W, f"thin {shape} r {r}")


@pytest.mark.parametrize("r", [0, 1, 2, 5, 6])
def test_every_nms_radius(r):
    """2 x 200 x 264 (no multiple of the 32-pixel NMS tile); r 5 and 6 use 161 and 203 KB of shared memory."""
    sd = synthetic.make_superpoint_state_dict(0, 4.0)
    conf = {"nms_radius": r, "max_keypoints": -1}
    _check(_module(sd, conf), _images((50, 51), 200, 264), sd, conf, 200 * 264, f"radius {r}",
           stages=["scores", "nms", "select", "sample"] if r not in (0, 6) else None)


def test_tied_scores_across_ranks_and_tiles():
    """Images of constant regions (one grey level, and three): cells farther than the receptive field from every edge see the
    same input and give exactly tied scores, on plateaus that cross NMS tiles.  Threshold 0, and k at every boundary of the
    rank's 1 024-key tiles and of the candidate count; a capacity below k."""
    sd = synthetic.make_superpoint_state_dict(0, 4.0)
    img = torch.full((2, 1, 256, 320), 0.5, device="cuda")
    img[1, :, :128, :160] = 0.2
    img[1, :, 128:, 160:] = 0.8
    base = {"nms_radius": 3, "keypoint_threshold": 0.0, "max_keypoints": -1}
    dev = _check(_module(sd, base), img, sd, base, 256 * 320, "ties k -1")
    nms = dev["nms"].cpu().numpy()
    totals = dev["counts"].tolist()
    cand = nms[0][nms[0] > 0]
    assert len(cand) - len(np.unique(cand)) > 100, "the quantised image must tie candidates"
    t = min(totals)
    for k in sorted({1, 1023, 1024, 1025, t - 1, t, t + 1, 2049, 3073}):
        conf = {**base, "max_keypoints": k}
        m = _module(sd, conf)
        for cap in (k, max(k // 2, 1)):
            _check(m, img, sd, conf, cap, f"ties k {k} cap {cap}", stages=["nms", "select", "sample"])


def test_stress_activations():
    """conv1a scaled so that the largest activation is in [300, 900]: the accumulator term at large values, and the
    end-to-end comparison with the oracle.  The end-to-end bars are those of O(1) activations scaled by the factor a: both
    the fp32 oracle's and the device's errors grow with the activations (measured: score error 3.9e-4 at a = 146)."""
    sd = dict(synthetic.make_superpoint_state_dict(0, 4.0))
    img = _images((70, 71), 256, 320)
    m = _module(sd, RELEASED)
    base = device_result(m, img, 4096)
    peak = max(float(a.abs().max()) for a in base["act"])
    a = np.float32(600.0 / peak)
    sd["conv1a.weight"] = sd["conv1a.weight"] * a
    sd["conv1a.bias"] = sd["conv1a.bias"] * a
    m = _module(sd, RELEASED)
    dev = _check(m, img, sd, RELEASED, 4096, f"stress x{a:.0f}")
    peak = max(float(x.abs().max()) for x in dev["act"])
    assert 300 <= peak <= 900, peak
    ref = O.forward(O.params_from_numpy(sd), img.cpu().numpy(), RELEASED)
    for b in range(2):
        n = int(dev["counts"][b])
        d = O.compare_keypoints(dev["kpts"][b, :n].cpu().numpy(), dev["kscores"][b, :n].cpu().numpy(), ref["keypoints"][b].numpy(),
                                ref["scores"][b].numpy(), SCORE_TOL * float(a), RELEASED["max_keypoints"])
        same = (dev["kpts"][b, :n].cpu() == ref["keypoints"][b]).all(1)
        err = float((dev["desc"][b, :, :n].cpu() - ref["descriptors"][b])[:, same].abs().max())
        print(f"stress[{b}] peak {peak:.0f}: {d}, descriptor error {err:.2e}")
        assert err <= DESC_TOL * float(a)


# ----------------------------------------------------------------------------- whole calls
def test_bench_shape_batch_independence():
    sd = synthetic.make_superpoint_state_dict(0, 4.0)
    img = _images(range(100, 108), 512, 512)
    m = _module(sd, RELEASED)
    both = {k: v.clone() for k, v in m.forward_padded(img).items()}
    for b in range(8):
        solo = m.forward_padded(img[b:b + 1])
        _same({k: v[b:b + 1] for k, v in both.items()}, solo, f"image {b}")


def test_poisoned_workspace_changes_nothing():
    lib = _lib.load()
    sd = synthetic.make_superpoint_state_dict(0, 4.0)
    thin = {"nms_radius": 6, "max_keypoints": -1, "remove_borders": 0, "keypoint_threshold": 0.001}
    runs = []
    try:
        for fill in (-1, 0xFF):
            assert lib.opb_debug_set_ws_fill(fill) == 0
            runs.append([{k: v.clone() for k, v in _module(sd, RELEASED).forward_padded(_images(range(100, 108), 512, 512)).items()},
                         {k: v.clone() for k, v in _module(sd, thin).forward_padded(_images((40, 41), 8, 1024), 8 * 1024).items()},
                         {k: v.clone() for k, v in _module(sd, thin).forward_padded(_images((40, 41, 42), 8, 8), 64).items()}])
    finally:
        lib.opb_debug_set_ws_fill(-1)
    for a, b, tag in zip(runs[0], runs[1], ("bench", "8 x 1024", "8 x 8")):
        _same(a, b, tag)


def test_one_handle_across_shape_changes():
    sd = synthetic.make_superpoint_state_dict(0, 4.0)
    seq = [_images(range(100, 108), 512, 512), _images((40, 41, 42), 8, 8), _images((30, 31), 480, 640), _images(range(100, 108), 512, 512)]
    m = _module(sd, RELEASED)
    for i, img in enumerate(seq):
        got = {k: v.clone() for k, v in m.forward_padded(img).items()}
        _same(got, _module(sd, RELEASED).forward_padded(img), f"call {i} {tuple(img.shape)}")


# ----------------------------------------------------------------------------- operand range guard
@pytest.mark.parametrize("layer", ["conv1a", "conv3a"])
def test_activation_past_the_operand_range_is_reported(layer):
    """A layer whose output passes 1023 (64 x >= 65 520 overflows the fp16 hi plane) must not turn into a block of zeros and
    finite key points: the call reports count 0 for every image and OPB_E_RANGE reaches the host."""
    sd = dict(synthetic.make_superpoint_state_dict(0, 4.0))
    gain = np.float32(5000 if layer == "conv1a" else 900)      # conv3a's largest weight stays below 1023 (a refused weight)
    sd[layer + ".weight"] = sd[layer + ".weight"] * gain
    sd[layer + ".bias"] = sd[layer + ".bias"] * gain
    img = _images((1, 2), 96, 128)
    m = _module(sd, RELEASED)
    out = m.forward_padded(img)
    assert out["counts"].tolist() == [0, 0]
    with pytest.raises(_lib.OpbError, match="OPB_E_RANGE"):
        m.check_range()
    m.check_range()                                                      # reporting cleared it
    with pytest.raises(_lib.OpbError, match="OPB_E_RANGE"):              # forward() synchronises for the counts: raises at once
        m(img)
    m.forward_padded(img)
    torch.cuda.synchronize()
    with pytest.raises(_lib.OpbError, match="OPB_E_RANGE"):              # a finished earlier call: reported by the next one
        m.forward_padded(img)
    m.check_range()
    # the same handle with sane weights: key points again, no error
    sane = synthetic.make_superpoint_state_dict(0, 4.0)
    m.load_state_dict({k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in sane.items()})
    out = m.forward_padded(img)
    m.check_range()
    assert min(out["counts"].tolist()) > 0


def test_weights_outside_the_operand_range_are_refused():
    """The range guard's premise: finite weights and biases, and weights that split (|w| < 1023)."""
    for name, value in (("conv2a.weight", 2000.0), ("convDb.weight", np.inf), ("conv4b.bias", np.nan), ("conv1a.weight", np.nan)):
        sd = dict(synthetic.make_superpoint_state_dict(0, 4.0))
        sd[name] = sd[name].copy()
        sd[name].flat[3] = value
        m = _module(sd, RELEASED)
        with pytest.raises(_lib.OpbError, match="OPB_E_RANGE"):
            m.forward_padded(_images((1,), 64, 64))
