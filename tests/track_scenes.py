"""The rendered scenes of the flow-only tracking goldens (tests/golden/make_track.py), free of side effects on import.

The golden keeps each frame's planted pose, the object's seed and a CRC-32 of the crop the reference tracked, not the crops:
``crop`` renders them again from those (numpy, fp64, then uint8) and the tests check every CRC before using one.
"""
from __future__ import annotations

import zlib

import numpy as np

from tests.flow_scenes import blob_object, pose_at, render_blobs, rodrigues

S = 160
K = np.array([[380.0, 0, S / 2], [0, 380.0, S / 2], [0, 0, 1]])
N = 80                    # pairs per frame (the device result's cap) and blobs per object

# (name, frames, object seed, per-frame matcher offset: {frame: (d rotvec, d translation)}, frames whose crop is turned by
# 180 degrees (the keyframe points are lost), frames with 3 matches)
SCENES = [
    ("smooth", 28, 31, {}, (), ()),
    ("reject", 26, 32, {10: ([0.0, 0.0, 0.0], [0.12, 0.0, 0.0])}, (), ()),
    ("lost", 27, 37, {}, (12, 13), ()),
    ("band", 25, 34, {f: ([0.0, 0.0, 0.0], [0.15, 0.0, 0.0]) for f in (1, 2, 3)}, (), ()),
    ("far", 25, 35, {f: ([0.0, 0.0, 0.0], [0.25, 0.0, 0.0]) for f in (1, 2, 3)}, (), ()),
    ("no_inliers", 30, 36, {}, (), (7, 8)),
]


def truth(seed: int, f: int) -> np.ndarray:
    """The planted pose [3,4] of frame f of the scene with object seed ``seed``: a seeded start and constant motion."""
    rs = np.random.RandomState(seed)
    p0 = np.concatenate([rodrigues(rs.uniform(-0.2, 0.2, 3)), [[rs.uniform(-0.01, 0.01)], [rs.uniform(-0.01, 0.01)], [0.45]]], 1)
    dw, dt = rs.uniform(-0.004, 0.004, 3), rs.uniform(-0.001, 0.001, 3)
    return pose_at(p0, f * dw, f * dt)


def crop(seed: int, pose, turned: bool) -> np.ndarray:
    """uint8 [S,S]: the scene's object seen from ``pose`` ([3,4] or [4,4]), turned by 180 degrees if ``turned``."""
    X, amp = blob_object(seed, N)
    image = render_blobs(K, np.asarray(pose)[:3], X, amp, S)
    return np.ascontiguousarray(image[::-1, ::-1]) if turned else image


def crc(image: np.ndarray) -> int:
    return zlib.crc32(np.ascontiguousarray(image, np.uint8).tobytes())
