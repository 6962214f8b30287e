"""The numpy model of the tracker's flow-only state machine (tests/track_reference.py): its Euler-angle code against scipy,
its cm / degree distance against pnp.pose_errors (to rounding: torch's CPU
kernels may fuse), and its run of the golden sequences against the reference's BATracker."""
import os

import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

from onepose_b200 import pnp
from tests import track_reference as TR
from tests import track_scenes as TS

Z = np.load(os.path.join(os.path.dirname(__file__), "golden", "pnp_track_cases.npz"))


def test_euler_against_scipy():
    """transforms3d's 'sxyz' is scipy's extrinsic 'xyz', away from gimbal lock."""
    rs = np.random.RandomState(0)
    for _ in range(500):
        a = rs.uniform([-np.pi, -1.5, -np.pi], [np.pi, 1.5, np.pi])
        M = TR.euler2mat(*a)
        np.testing.assert_allclose(M, Rotation.from_euler("xyz", a).as_matrix(), atol=1e-14)
        np.testing.assert_allclose(TR.mat2euler(M), a, atol=1e-12)
        R = Rotation.random(random_state=rs)
        e = R.as_euler("xyz")
        if abs(abs(e[1]) - np.pi / 2) > 1e-3:
            np.testing.assert_allclose(TR.mat2euler(R.as_matrix()), e, atol=1e-10)


@pytest.mark.parametrize("pitch", [np.pi / 2, -np.pi / 2])
def test_gimbal_lock_branch(pitch):
    """At a pitch of exactly +-90 degrees cy <= 4 eps: the yaw is 0 and the roll absorbs it, the matrix is kept."""
    rs = np.random.RandomState(1)
    for _ in range(50):
        M = TR.euler2mat(rs.uniform(-3, 3), pitch, rs.uniform(-3, 3))
        assert np.hypot(M[0, 0], M[1, 0]) <= TR.EPS4
        e = TR.mat2euler(M)
        assert e[2] == 0.0 and abs(e[1] - pitch) < 1e-7
        np.testing.assert_allclose(TR.euler2mat(*e), M, atol=1e-7)


def test_cm_degree_is_pose_errors():
    rs = np.random.RandomState(2)
    for _ in range(300):
        a = np.eye(4)
        b = np.eye(4)
        a[:3, :3], b[:3, :3] = Rotation.random(random_state=rs).as_matrix(), Rotation.random(random_state=rs).as_matrix()
        a[:3, 3], b[:3, 3] = rs.randn(3), rs.randn(3)
        cm, deg = TR.cm_degree(a, b)
        rot, trans = pnp.pose_errors(torch.from_numpy(a[None]), torch.from_numpy(b[None]))
        assert abs(cm - float(trans)) <= 1e-15 * cm and abs(deg - float(rot)) <= 1e-12 * max(deg, 1.0)


def test_motion_prediction_slip():
    """rot_t is mat2euler of pose_list[-2]: the rotation extrapolates half a step from the middle pose."""
    p = [np.eye(4) for _ in range(3)]
    for k in range(3):
        p[k][:3, :3] = TR.euler2mat(0.1 * k, 0.0, 0.0)
        p[k][:3, 3] = [0.01 * k, 0.0, 0.5]
    out = TR.motion_prediction(*p)
    np.testing.assert_allclose(TR.mat2euler(out), [0.15, 0.0, 0.0], atol=1e-15)
    np.testing.assert_allclose(out[:3, 3], [0.03, 0.0, 0.5], atol=1e-15)


def test_model_on_goldens():
    """The model fed the reference's own flow poses and kpt_dist reproduces its gate, branch, counters and reported poses;
    motion poses bit for bit (the golden's motion_prediction ran on this model's Euler code)."""
    for s, name in enumerate(Z["names"]):
        st = TR.init_state(1)
        for i in range(len(Z[f"s{s}_n"])):
            pp = Z[f"s{s}_pose_pred"][i][None]
            g = TR.gate(st, pp)
            pose, br = TR.select(st, pp, Z[f"s{s}_flow_pose"][i][None], Z[f"s{s}_kpt_dist"][i:i + 1])
            at = f"{name}[{i}]"
            assert g[0] == Z[f"s{s}_gate"][i] and br[0] == Z[f"s{s}_branch"][i], at
            assert st["use_motion_cnt"][0] == Z[f"s{s}_umc"][i] and st["init_cnt"][0] == Z[f"s{s}_init_cnt"][i], at
            np.testing.assert_array_equal(pose[0], Z[f"s{s}_pose"][i], err_msg=at)


def test_golden_crops_render():
    """The golden keeps CRC-32s, not crops: every frame's crop renders again to the crop the reference tracked."""
    for s, name in enumerate(Z["names"]):
        for i in range(len(Z[f"s{s}_n"])):
            im = TS.crop(int(Z[f"s{s}_seed"]), Z[f"s{s}_truth"][i], bool(Z[f"s{s}_turned"][i]))
            assert im.shape == (TS.S, TS.S) and TS.crc(im) == int(Z[f"s{s}_crc"][i]), f"{name}[{i}]"
    assert np.array_equal(Z["K"], TS.K) and int(Z["cap"]) == TS.N
