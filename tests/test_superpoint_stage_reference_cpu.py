"""The extractor's fp64 stage references (tests/superpoint_stage_reference.py) without a GPU:
  * chained, the stages are the oracle's forward run in fp64;
  * the selection reference is the device's rule (tests/sp_emulation.py), and the oracle's wherever scores do not tie;
  * each planted defect moves its own stage by at least 10x that stage's bar, and the table records which of them the
    end-to-end bars (key points exact, scores within 2e-5, descriptors within 1e-5) would miss."""
import numpy as np
import pytest
import torch

from onepose_b200 import synthetic
from oracle import superpoint_oracle as O
from tests import sp_emulation as E
from tests import superpoint_stage_reference as R
from tests.golden_util import load_superpoint_case

SCORE_TOL, DESC_TOL = 2e-5, 1e-5


def _oracle64(p, image, cfg, align_corners):
    """The oracle's forward (superpoint_oracle.forward) in fp64; image [B, 1, H, W]."""
    x = torch.as_tensor(image, dtype=torch.float64)
    feat = O.encoder(p, x)
    scores = O.dense_scores(p, feat)
    nms = O.simple_nms(scores, cfg["nms_radius"])
    dd = O.dense_descriptors(p, feat)
    out = []
    for b in range(x.shape[0]):
        k, s = O.select_keypoints(nms[b], cfg)
        out.append((k, s, O.sample_descriptors(k.double(), dd[b], 8, align_corners)))
    return scores, out


def _err(a, b):
    d = (a - b).abs()
    return float(d.max()) if d.numel() else 0.0


def _synthetic(seeds, H, W):
    return np.stack([synthetic.make_image(i, H, W)[0] for i in seeds], 0)


CASES = {
    "golden_all_64x64": lambda: load_superpoint_case("superpoint_all_64x64"),
    "golden_topk_96x128": lambda: load_superpoint_case("superpoint_topk_96x128"),
    "synthetic_64x80": lambda: (None, synthetic.make_superpoint_state_dict(0, 4.0), {"nms_radius": 3}, _synthetic((1, 2), 64, 80)[:, None]),
    "synthetic_8x8": lambda: (None, synthetic.make_superpoint_state_dict(1, 4.0), {"nms_radius": 0, "remove_borders": 0, "keypoint_threshold": 0.0},
                              _synthetic((3, 4, 5), 8, 8)[:, None]),
}


@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("align_corners", [True, False])
def test_chained_stages_equal_the_fp64_oracle(case, align_corners):
    _, sd, conf, img = CASES[case]()
    cfg = {**O.DEFAULT_CONFIG, **conf}
    p = R.params64(sd)
    image = torch.from_numpy(img[:, 0])
    H, W = image.shape[1:]
    dev = R.chain(p, image, cfg, cap=H * W, align_corners=align_corners)
    scores, ref = _oracle64(p, img, cfg, align_corners)
    assert float((dev["scores"] - scores).abs().max()) < 1e-10
    total = 0
    for b, (k, s, d) in enumerate(ref):
        n = int(dev["counts"][b])
        assert n == len(k), (b, n, len(k))
        assert torch.equal(dev["kpts"][b, :n], k.float()), f"image {b}: key points differ"
        assert _err(dev["kscores"][b, :n], s) < 1e-10
        assert _err(dev["desc"][b, :, :n], d) < 1e-10
        total += n
    assert total > 0
    # every stage of the chain against itself: zero error, and zero border rows
    r = R.check(dev, p, cfg, align_corners, positions=np.float64)
    assert all(v == 0.0 for v in r.values()), r


def test_selection_reference_is_the_device_rule():
    """select == sp_emulation.select (score descending, pixel ascending) everywhere, == oracle.select_keypoints (torch.topk)
    on images without tied candidates; a constant image ties whole plateaus, where only the device rule decides."""
    sd = synthetic.make_superpoint_state_dict(0, 4.0)
    p = R.params64(sd)
    imgs = np.concatenate([_synthetic((1, 2), 96, 128), np.full((1, 96, 128), 0.5, np.float32)], 0)
    cfg = {**O.DEFAULT_CONFIG, "nms_radius": 3}
    dev = R.chain(p, torch.from_numpy(imgs), cfg, cap=1)
    nms32 = dev["nms"].float().numpy()
    tied = 0
    for b in range(3):
        cand = nms32[b][nms32[b] > np.float32(cfg["keypoint_threshold"])]
        ties = len(cand) - len(np.unique(cand))
        for k in (1, 7, 50, 300, -1):
            kp, s, n = R.select(nms32[b], cfg["keypoint_threshold"], cfg["remove_borders"], k, cap=10 ** 6)
            ek, es = E.select(nms32[b], cfg["keypoint_threshold"], cfg["remove_borders"], k)
            assert np.array_equal(kp, ek) and np.array_equal(s, es), (b, k)
            if ties == 0:
                ok, os_ = O.select_keypoints(torch.from_numpy(nms32[b]), {**cfg, "max_keypoints": k})
                assert np.array_equal(kp, ok.numpy()) and np.array_equal(s, os_.numpy()), (b, k)
            # cap truncates the same order
            kc, sc, nc = R.select(nms32[b], cfg["keypoint_threshold"], cfg["remove_borders"], k, cap=3)
            assert nc == min(n, 3) and np.array_equal(kc, kp[:nc])
        tied += ties > 0
    assert tied >= 1, "the constant image must tie candidates"


# ----------------------------------------------------------------------------- planted defects
STAGES_OF = {
    "tap_offset": ["conv1b", "conv2a", "conv2b", "conv3a", "conv3b", "conv4a", "conv4b", "convPa|convDa"],
    "border_last_tile": ["conv1b", "conv2a", "conv2b", "conv3a", "conv3b", "conv4a", "conv4b", "convPa|convDa"],
    "pool_hi_only": ["pool1", "pool2", "pool3"],
    "topk_ties_high": ["select"],
    "align_corners_edge": ["sample"],
    "sample_skip_norm": ["sample"],
}
# which defects the end-to-end bars let through on this case (measured by the test below and pinned): pooling by hi moves
# activations by a lo-plane amount only, and compare_keypoints accepts any order among tied scores
E2E_MISSES = {"pool_hi_only", "topk_ties_high"}


def _end_to_end_catches(dev, ref, max_keypoints):
    """The end-to-end bars of tests/test_superpoint_gpu.py: key points by oracle.compare_keypoints (exact, or under top-k
    exact up to ties within the score tolerance), scores within 2e-5, descriptors within 1e-5 where the key points agree."""
    for b in range(len(ref["counts"])):
        n, nr = int(dev["counts"][b]), int(ref["counts"][b])
        try:
            O.compare_keypoints(dev["kpts"][b, :n].numpy(), dev["kscores"][b, :n].numpy(), ref["kpts"][b, :nr].numpy(),
                                ref["kscores"][b, :nr].numpy(), SCORE_TOL, max_keypoints)
        except AssertionError:
            return True
        same = (dev["kpts"][b, :n] == ref["kpts"][b, :nr]).all(1)
        if _err(dev["desc"][b, :, :n][:, same], ref["desc"][b, :, :nr][:, same]) > DESC_TOL:
            return True
    return False


def test_planted_defects_move_their_stage():
    sd = synthetic.make_superpoint_state_dict(0, 4.0)
    p = R.params64(sd)
    imgs = _synthetic((1, 2), 64, 80)
    image = torch.from_numpy(imgs)
    cfg = {**O.DEFAULT_CONFIG, "nms_radius": 3, "max_keypoints": 40}
    cap = 40
    # dense scores in fp32 (as the device stores them) on a grid of 2^-7: exactly tied candidates across the top-k cut
    kw = dict(positions=np.float32, score_dtype=torch.float32, quantum=2.0 ** -7)
    clean = R.chain(p, image, cfg, cap, **kw)
    assert all(int(c) > cap for c in [len(R.select(clean["nms"][b].numpy(), cfg["keypoint_threshold"], cfg["remove_borders"], -1, 10 ** 6)[0])
                                     for b in range(2)]), "both images need more candidates than k"
    lines, misses = [], set()
    for defect in R.DEFECTS:
        dev = R.chain(p, image, cfg, cap, defect=defect, **kw)
        r = R.check(dev, p, cfg, stages=STAGES_OF[defect])
        worst = max(r[s] for s in STAGES_OF[defect])
        caught = _end_to_end_catches(dev, clean, cfg["max_keypoints"])
        if not caught:
            misses.add(defect)
        lines.append(f"{defect:20s} stage x bar {worst:9.3g}   end-to-end bars {'catch it' if caught else 'MISS it'}")
        assert worst >= 10, f"{defect}: its stage moves by only {worst:.3g} x its bar ({R.table(r)})"
    print("\n".join(["planted defect       own stage           end to end"] + lines))
    assert misses == E2E_MISSES, misses
