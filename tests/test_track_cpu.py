"""Argument checks of onepose_b200.track that run before any device work."""
import pytest
import torch

from onepose_b200 import track


def test_init_state_checks():
    for args in [(0, 8, 16), (2, 0, 16), (2, 8, 0)]:
        with pytest.raises(ValueError):
            track.init_state(*args, "cpu")
    with pytest.raises(RuntimeError, match="no CPU path"):
        track.init_state(2, 8, 16, "cpu")


def test_reset_mask_checks():
    state = {"frame": torch.zeros(3, dtype=torch.int64)}
    with pytest.raises(ValueError, match="bool"):
        track.reset(state, torch.zeros(3, dtype=torch.int32))
    with pytest.raises(ValueError, match="bool"):
        track.reset(state, torch.zeros(2, dtype=torch.bool))


def test_state_checks():
    with pytest.raises(ValueError, match="init_state"):
        track.step({"frame": torch.zeros(1)}, {}, torch.zeros(1, 8, 8, dtype=torch.uint8), torch.eye(3))
