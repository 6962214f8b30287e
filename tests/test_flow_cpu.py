"""Argument checks of the flow step that run before any device work, and the keyframe-state shapes."""
import pytest
import torch

from onepose_b200 import flow


def test_params_checks():
    ok = ((15, 15), 2, (3, 10, 0.03), 1e-4)
    assert flow._params(*ok) == (15, 15, 2, 3, 10, 0.03, 1e-4)
    for win in [(2, 3), (4, 5), (33, 33), (15, 14)]:
        with pytest.raises(ValueError):
            flow._params(win, *ok[1:])
    for lev in [-1, 5]:
        with pytest.raises(ValueError):
            flow._params(ok[0], lev, *ok[2:])
    for crit in [(0, 10, 0.1), (4, 10, 0.1), (1, 0, 0.1), (1, 101, 0.1), (2, 0, -0.5), (3, 10, float("nan"))]:
        with pytest.raises(ValueError):
            flow._params(ok[0], ok[1], crit, ok[3])
    assert flow._params(ok[0], ok[1], (2, 0, 0.5), ok[3])[3:6] == (2, 0, 0.5)      # count is not read without COUNT
    with pytest.raises(ValueError):
        flow._params(*ok, flags=flow.OPTFLOW_LK_GET_MIN_EIGENVALS)
    with pytest.raises(ValueError):
        flow._params(*ok[:3], -1.0)


def test_cpu_tensors_refused():
    img = torch.zeros(1, 32, 32, dtype=torch.uint8)
    with pytest.raises(RuntimeError, match="CUDA"):
        flow.lk_batch(img, img, torch.zeros(1, 2), torch.tensor([0, 1], dtype=torch.int32))


def test_keyframe_state_checks():
    B, cap, S = 3, 8, 16
    kf = {"image": torch.zeros(B, S, S, dtype=torch.uint8), "pts2d": torch.zeros(B, cap, 2), "pts3d": torch.zeros(B, cap, 3),
          "counts": torch.zeros(B, dtype=torch.int32)}
    with pytest.raises(RuntimeError, match="CUDA"):
        flow._check_kf(kf)
    bad = dict(kf)
    del bad["counts"]
    with pytest.raises(ValueError, match="counts"):
        flow._check_kf(bad)


def test_u8_crops():
    u8 = torch.randint(0, 256, (2, 8, 8), dtype=torch.uint8)
    assert torch.equal(flow._u8_crops(u8, "x"), u8)
    assert torch.equal(flow._u8_crops((u8.float() / 255)[:, None], "x"), u8)
    with pytest.raises(ValueError):
        flow._u8_crops(torch.zeros(2, 8, 8), "x")


def test_last_level_matches_model():
    from tests import lk_reference as L
    for h, w in [(10, 10), (37, 50), (64, 64), (512, 512), (100, 31)]:
        for win in [(3, 3), (15, 15), (31, 31), (7, 21)]:
            for lev in range(5):
                assert flow._last_level(h, w, win, lev) == L.n_levels(h, w, win, lev)


def test_keyframe_state_without_rows_refused():
    """A keyframe state of cap = 0 (from a result of N = 0 pairs per frame) has nothing to track: refused before any work."""
    kf = {"image": torch.zeros(2, 16, 16, dtype=torch.uint8), "pts2d": torch.zeros(2, 0, 2), "pts3d": torch.zeros(2, 0, 3),
          "counts": torch.zeros(2, dtype=torch.int32)}
    with pytest.raises(ValueError, match="cap = 0"):
        flow.flow_track(kf, kf["image"], torch.eye(3), torch.eye(4).expand(2, 4, 4))
