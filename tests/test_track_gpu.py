"""The tracker's flow-only state machine on the device (csrc/track.cu, onepose_b200/track.py) against the numpy model
(tests/track_reference.py) and the reference's BATracker (tests/golden/make_track.py)."""
import os

import numpy as np
import pytest
import torch

from onepose_b200 import _lib, pnp, track
from tests import flow_scenes as FS
from tests import track_reference as TR
from tests import track_scenes as TS

pytestmark = pytest.mark.gpu
DEV = "cuda"
Z = np.load(os.path.join(os.path.dirname(__file__), "golden", "pnp_track_cases.npz"))
ROT_TOL = 1e-12          # motion-predicted rotation entries: CUDA's atan2 / sin / cos against glibc's


def _rot(rs, scale=1.0):
    return FS.rodrigues(rs.uniform(-scale, scale, 3))


def _pose(R, t):
    P = np.eye(4)
    P[:3, :3], P[:3, 3] = R, t
    return P


def _dev_state(s):
    return {k: torch.from_numpy(np.ascontiguousarray(v)).to(DEV) for k, v in s.items()}


def _run_kernels(state, pose_pred, pose_flow, kpt_dist):
    d = _dev_state(state)
    B = len(state["frame"])
    pp, pf = torch.from_numpy(pose_pred).to(DEV), torch.from_numpy(pose_flow).to(DEV)
    gate = torch.empty(B, dtype=torch.int32, device=DEV)
    _lib.call(pp.device, "opb_track_gate", pp, B, d["frame"], d["hist"], d["hist_len"], gate)
    out = torch.empty(B, 4, 4, dtype=torch.float64, device=DEV)
    branch = torch.empty(B, dtype=torch.int32, device=DEV)
    _lib.call(pp.device, "opb_track_select", pp, pf, torch.from_numpy(kpt_dist).to(DEV), B, d["frame"], d["hist"], d["hist_len"], d["init_cnt"],
              d["use_motion_cnt"], out, branch)
    return gate.cpu().numpy(), out.cpu().numpy(), branch.cpu().numpy(), {k: v.cpu().numpy() for k, v in d.items()}


def _constructed(B, seed):
    """B tracks on constructed states: histories of 0-3 poses, every counter value, flow poses near and far (translation-only
    deltas of exactly 10 and 20 cm among them), NaN kpt_dist and gimbal-lock poses."""
    rs = np.random.RandomState(seed)
    st = TR.init_state(B)
    pose_pred, pose_flow, kpt = np.zeros((B, 4, 4)), np.zeros((B, 4, 4)), np.zeros(B)
    for b in range(B):
        n = b % 4
        st["hist_len"][b] = n
        st["frame"][b] = 0 if n == 0 else [1, 2, 4, 5, 10, 7][(b // 4) % 6]
        st["init_cnt"][b] = (b // 24) % 5 - 1            # -1 .. 3
        st["use_motion_cnt"][b] = (b // 120) % 6          # 0 .. 5
        base = _pose(_rot(rs), rs.uniform(-0.1, 0.1, 3) + [0, 0, 0.5])
        kind = (b // 7) % 5
        for k in range(n):
            R = base[:3, :3] @ _rot(rs, 0.05 * k)
            if kind == 4:                                  # gimbal lock: pitch of exactly +-90 degrees
                R = TR.euler2mat(rs.uniform(-1, 1), np.pi / 2 * (1 if k % 2 else -1), rs.uniform(-1, 1))
            st["hist"][b, k] = _pose(R, base[:3, 3] + 0.01 * k * rs.randn(3))
        last = st["hist"][b, max(n - 1, 0)] if n else base
        pose_pred[b] = _pose(last[:3, :3] @ _rot(rs, 0.3 * rs.rand()), last[:3, 3] + rs.uniform(-0.2, 0.2, 3) * rs.rand())
        if kind == 0:                                     # a translation-only delta of exactly 10 or 20 cm
            pose_flow[b] = last.copy()
            pose_flow[b, 0, 3] = last[0, 3] + (0.1 if b % 2 else 0.2)
            pose_flow[b, 1:3, 3] = last[1:3, 3]
            if b % 3 == 0:
                pose_pred[b] = pose_flow[b]
        else:
            pose_flow[b] = _pose(last[:3, :3] @ _rot(rs, 0.4 * rs.rand()), last[:3, 3] + rs.uniform(-0.25, 0.25, 3) * rs.rand())
        kpt[b] = [np.nan, 0.5, 9.0, 10.0, 11.0, 100.0][b % 6]
    return st, pose_pred, pose_flow, kpt


@pytest.mark.parametrize("B", [1, 7, 130, 1000])
def test_kernels_against_model(B):
    st, pp, pf, kd = _constructed(B, B)
    gate, pose, branch, dst = _run_kernels(st, pp, pf, kd)
    want_gate = TR.gate(st, pp)
    want_pose, want_branch = TR.select(st, pp, pf, kd)
    np.testing.assert_array_equal(gate, want_gate)
    np.testing.assert_array_equal(branch, want_branch)
    for k in ("frame", "hist_len", "init_cnt", "use_motion_cnt"):
        np.testing.assert_array_equal(dst[k], st[k], err_msg=k)
    copied = branch != TR.MOTION
    np.testing.assert_array_equal(pose[copied], want_pose[copied])
    mo = ~copied
    if mo.any():                # translation bit for bit, rotation to ROT_TOL
        np.testing.assert_array_equal(pose[mo][:, :, 3], want_pose[mo][:, :, 3])
        assert np.abs(pose[mo][:, :3, :3] - want_pose[mo][:, :3, :3]).max() <= ROT_TOL
    np.testing.assert_array_equal(dst["hist"][copied], st["hist"][copied])
    if B >= 130:
        assert set(np.unique(branch)) == {0, 1, 2, 3, 4} and set(np.unique(gate)) == {0, 1, 2, 3}


def test_exact_thresholds():
    """Translation-only deltas of exactly 10 and 20 cm: the model's distance is 10.0 / 20.0 and the device decides the same."""
    last = _pose(np.eye(3), [0.0, 0.0, 0.5])
    cases = []
    for dx in (0.1, 0.2):
        f = last.copy()
        f[0, 3] = dx
        cm, deg = TR.cm_degree(last, f)
        assert cm == (10.0 if dx == 0.1 else 20.0) and deg == 0.0
        cases.append(f)
    B = 2 * 4
    st = TR.init_state(B)
    pf = np.zeros((B, 4, 4))
    for b in range(B):
        st["frame"][b], st["hist_len"][b], st["init_cnt"][b], st["use_motion_cnt"][b] = 5, 3, 0, [0, 3, 0, 3][b % 4]
        st["hist"][b] = last
        pf[b] = cases[b // 4]
    pp = np.stack([cases[b // 4] if b % 4 >= 2 else last for b in range(B)])
    gate, pose, branch, dst = _run_kernels(st, pp, pf, np.zeros(B))
    np.testing.assert_array_equal(gate, TR.gate(st, pp))
    _, wb = TR.select(st, pp, pf, np.zeros(B))
    np.testing.assert_array_equal(branch, wb)
    np.testing.assert_array_equal(dst["use_motion_cnt"], st["use_motion_cnt"])
    print("branches at 10 / 20 cm:", branch.tolist())


_CROPS = {}


def _crop(s, i):
    """Frame i of scene s as the reference tracked it: rendered again, its CRC-32 checked against the golden's."""
    if (s, i) not in _CROPS:
        im = TS.crop(int(Z[f"s{s}_seed"]), Z[f"s{s}_truth"][i], bool(Z[f"s{s}_turned"][i]))
        assert TS.crc(im) == int(Z[f"s{s}_crc"][i]), f"the crop of scene {s} frame {i} does not render as the golden's"
        _CROPS[(s, i)] = im
    return _CROPS[(s, i)]


def _golden_results(fi, scenes):
    """Frame fi[b] of each scene as a poses_from_matches result (the reference's own matcher poses and inliers) and its crops."""
    N = int(Z["cap"])
    B = len(scenes)
    n = np.array([int(Z[f"s{s}_n"][i]) for s, i in zip(scenes, fi)])
    off = np.concatenate([[0], np.cumsum(n)]).astype(np.int32)
    p2, p3, mask = np.zeros((B * N, 2)), np.zeros((B * N, 3)), np.zeros(B * N, bool)
    for b, (s, i) in enumerate(zip(scenes, fi)):
        p2[off[b]:off[b + 1]] = Z[f"s{s}_m2d"][i][:n[b]]
        p3[off[b]:off[b + 1]] = Z[f"s{s}_m3d"][i][:n[b]]
        mask[off[b]:off[b + 1]] = Z[f"s{s}_mask"][i][:n[b]]
    res = {"offsets": torch.from_numpy(off).to(DEV), "inlier_mask": torch.from_numpy(mask).to(DEV), "pts2d": torch.from_numpy(p2).to(DEV),
           "pts3d": torch.from_numpy(p3).to(DEV), "pose_homo": torch.from_numpy(np.stack([Z[f"s{s}_pose_pred"][i] for s, i in zip(scenes, fi)])).to(DEV)}
    crops = torch.from_numpy(np.stack([_crop(s, i) for s, i in zip(scenes, fi)])).to(DEV)
    return res, crops


def _run_golden(scenes, frames, start=None):
    """The scenes through track.step, track b from step start[b] on (it is reset there; before, it runs its frame 0)."""
    B = len(scenes)
    start = start or [0] * B
    state = track.init_state(B, int(Z["cap"]), TS.S, DEV)
    K = torch.from_numpy(Z["K"]).to(DEV)
    outs = []
    for t in range(frames):
        if any(t == s0 > 0 for s0 in start):
            track.reset(state, torch.tensor([t == s0 for s0 in start], device=DEV))
        fi = [min(max(t - s0, 0), len(Z[f"s{s}_n"]) - 1) for s, s0 in zip(scenes, start)]
        res, crops = _golden_results(fi, scenes)
        o = track.step(state, res, crops, K)
        outs.append({"pose": o["pose"].cpu().numpy(), "branch": o["branch"].cpu().numpy(), "gate": o["gate"].cpu().numpy(),
                     "accept": o["flow"]["accept"].cpu().numpy(), "umc": state["use_motion_cnt"].cpu().numpy().copy(),
                     "init_cnt": state["init_cnt"].cpu().numpy().copy(), "hist": state["hist"].cpu().numpy().copy(),
                     "hist_len": state["hist_len"].cpu().numpy().copy()})
    return outs


def test_golden_sequences():
    """Every scene's frames through track.step against the reference's BATracker: gate outcomes, branch codes, counters and
    flow_track accepts equal on every frame; init / keyframe frames bit-equal to the reference's pose; flow frames within
    test_flow_gpu's tolerances; motion frames within ROT_TOL of the model on the device's own history."""
    names = list(Z["names"])
    scenes = list(range(len(names)))
    frames = max(len(Z[f"s{s}_n"]) for s in scenes)
    outs = _run_golden(scenes, frames)
    worst = {}
    for b, s in enumerate(scenes):
        name = names[s]
        for i in range(len(Z[f"s{s}_n"])):
            o = outs[i]
            at = f"{name}[{i}]"
            assert o["gate"][b] == Z[f"s{s}_gate"][i], at
            assert o["branch"][b] == Z[f"s{s}_branch"][i], (at, o["branch"][b], Z[f"s{s}_branch"][i])
            assert o["umc"][b] == Z[f"s{s}_umc"][i] and o["init_cnt"][b] == Z[f"s{s}_init_cnt"][i], at
            if i > 0:
                assert bool(o["accept"][b]) == bool(Z[f"s{s}_accept"][i]), at
            code = int(o["branch"][b])
            ref = Z[f"s{s}_pose"][i]
            if code in (TR.INIT, TR.KEYFRAME, TR.PRED):
                np.testing.assert_array_equal(o["pose"][b], ref, err_msg=at)
            elif code == TR.FLOW:
                rot, trans = pnp.pose_errors(torch.from_numpy(o["pose"][b:b + 1]), torch.from_numpy(ref[None]))
                assert float(rot) <= 1.0 and float(trans) <= 1.0, (at, float(rot), float(trans))
                worst["flow"] = max(worst.get("flow", (0, 0)), (float(rot), float(trans)))
            else:
                h = outs[i - 1]["hist"][b]
                want = TR.motion_prediction(h[0], h[1], h[2])
                np.testing.assert_array_equal(o["pose"][b][:, 3], want[:, 3], err_msg=at)
                err = np.abs(o["pose"][b][:3, :3] - want[:3, :3]).max()
                assert err <= ROT_TOL, (at, err)
                worst["motion"] = max(worst.get("motion", 0.0), err)
                rot, trans = pnp.pose_errors(torch.from_numpy(o["pose"][b:b + 1]), torch.from_numpy(ref[None]))
                worst["motion_vs_ref"] = max(worst.get("motion_vs_ref", (0, 0)), (float(rot), float(trans)))
    print("worst:", worst)


def test_tracks_at_different_frames():
    """Tracks started at different steps in one call equal each track run alone, bit for bit; reset on a subset."""
    scenes = [0, 3, 5]
    start = [0, 4, 9]
    frames = 20
    together = _run_golden(scenes, frames, start)
    for b, s in enumerate(scenes):
        alone = _run_golden([s], frames - start[b])
        for t in range(start[b], frames):
            a, o = alone[t - start[b]], together[t]
            np.testing.assert_array_equal(o["pose"][b], a["pose"][0])
            for k in ("branch", "gate", "umc", "init_cnt", "hist_len"):
                assert o[k][b] == a[k][0], (s, t, k)


def test_reset_subset():
    B = 4
    st = track.init_state(B, 8, 16, DEV)
    st["frame"].fill_(7)
    st["hist_len"].fill_(3)
    st["init_cnt"].fill_(0)
    st["use_motion_cnt"].fill_(2)
    track.reset(st, torch.tensor([True, False, True, False], device=DEV))
    assert st["frame"].tolist() == [0, 7, 0, 7] and st["hist_len"].tolist() == [0, 3, 0, 3]
    assert st["init_cnt"].tolist() == [3, 0, 3, 0] and st["use_motion_cnt"].tolist() == [0, 2, 0, 2]


def test_side_stream_sentinels():
    """The entry points on a side stream write every output element: they start as NaN / -7 sentinels."""
    st, pp, pf, kd = _constructed(64, 3)
    want_gate = TR.gate({k: v.copy() for k, v in st.items()}, pp)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        d = _dev_state(st)
        ppd, pfd, kdd = (torch.from_numpy(x).to(DEV) for x in (pp, pf, kd))
        gate = torch.full((64,), -7, dtype=torch.int32, device=DEV)
        out = torch.full((64, 4, 4), float("nan"), dtype=torch.float64, device=DEV)
        branch = torch.full((64,), -7, dtype=torch.int32, device=DEV)
        _lib.call(ppd.device, "opb_track_gate", ppd, 64, d["frame"], d["hist"], d["hist_len"], gate)
        _lib.call(ppd.device, "opb_track_select", ppd, pfd, kdd, 64, d["frame"], d["hist"], d["hist_len"], d["init_cnt"], d["use_motion_cnt"], out, branch)
    s.synchronize()
    assert torch.isfinite(out).all() and (branch >= 0).all()
    np.testing.assert_array_equal(gate.cpu().numpy(), want_gate)


def test_argument_errors():
    lib = _lib.load()
    x = torch.zeros(16, dtype=torch.float64, device=DEV)
    rc = lib.opb_track_gate(x.data_ptr(), 0, x.data_ptr(), x.data_ptr(), x.data_ptr(), x.data_ptr(), None)
    assert rc == -1 and b"B > 0" in lib.opb_last_error(None)
    rc = lib.opb_track_select(x.data_ptr(), None, x.data_ptr(), 1, x.data_ptr(), x.data_ptr(), x.data_ptr(), x.data_ptr(), x.data_ptr(), x.data_ptr(),
                              x.data_ptr(), None)
    assert rc == -1 and b"pose_flow" in lib.opb_last_error(None)
    st = track.init_state(2, 8, 16, DEV)
    res = {"pose_homo": torch.zeros(2, 4, 4, dtype=torch.float64, device=DEV), "inlier_mask": torch.zeros(2 * 9, dtype=torch.bool, device=DEV)}
    with pytest.raises(ValueError, match="pairs per frame"):
        track.step(st, res, torch.zeros(2, 16, 16, dtype=torch.uint8, device=DEV), torch.eye(3, device=DEV))
    res["pose_homo"] = torch.zeros(2, 3, 4, dtype=torch.float64, device=DEV)
    with pytest.raises(ValueError, match="pose_homo"):
        track.step(st, res, torch.zeros(2, 16, 16, dtype=torch.uint8, device=DEV), torch.eye(3, device=DEV))


def test_closed_loop():
    """3 objects over 30 frames of planted motion, through poses_from_matches_objects on planted matches and track.step:
    every reported pose within 1 cm / 1 degree of the planted one."""
    S = 192
    K = np.array([[450.0, 0, S / 2], [0, 450.0, S / 2], [0, 0, 1]])
    objs = [FS.blob_object(21, 80), FS.blob_object(22, 70), FS.blob_object(23, 75)]
    pose0 = [np.concatenate([FS.rodrigues([0.1, 0.2, -0.05]), [[0.01], [-0.01], [0.45]]], 1),
             np.concatenate([FS.rodrigues([-0.2, 0.05, 0.1]), [[-0.01], [0.0], [0.5]]], 1),
             np.concatenate([FS.rodrigues([0.05, -0.15, 0.2]), [[0.0], [0.01], [0.48]]], 1)]
    steps = [(np.array([0.004, -0.003, 0.002]), np.array([0.0008, -0.0006, 0.0012])),
             (np.array([-0.003, 0.004, -0.002]), np.array([-0.0006, 0.0009, -0.001])),
             (np.array([0.002, 0.002, -0.003]), np.array([0.0005, 0.0005, 0.0008]))]
    B, N = 3, 80
    Kd = torch.from_numpy(K).to(DEV)
    kp3 = {k: torch.from_numpy(objs[k][0]).to(DEV) for k in range(B)}
    rs = np.random.RandomState(5)
    state = track.init_state(B, N, S, DEV)
    worst, seen = (0.0, 0.0), set()
    for f in range(30):
        truth = [FS.pose_at(pose0[k], f * steps[k][0], f * steps[k][1]) for k in range(B)]
        imgs = torch.from_numpy(np.stack([FS.render_blobs(K, truth[k], *objs[k], S) for k in range(B)])).to(DEV)
        kp2 = np.zeros((B, N, 2), np.float32)
        m0 = np.full((B, N), -1, np.int64)
        for k in range(B):
            M = len(objs[k][0])
            kp2[k, :M] = FS.project(K, truth[k], objs[k][0]) + 0.2 * rs.randn(M, 2)
            m0[k, :M] = np.arange(M)
        res = pnp.poses_from_matches_objects(Kd, torch.from_numpy(kp2).to(DEV), kp3, [0, 1, 2], torch.from_numpy(m0).to(DEV), scale=1000,
                                             method="epnp", confidence=0.99)
        out = track.step(state, res, imgs, Kd)
        ref = torch.from_numpy(np.stack([np.concatenate([t, [[0, 0, 0, 1.0]]]) for t in truth])).to(DEV)
        rot, trans = pnp.pose_errors(out["pose"], ref)
        assert (rot < 1.0).all() and (trans < 1.0).all(), (f, rot.tolist(), trans.tolist(), out["branch"].tolist())
        worst = (max(worst[0], float(rot.max())), max(worst[1], float(trans.max())))
        seen |= set(out["branch"].tolist())
    assert TR.FLOW in seen and TR.INIT in seen
    print(f"closed loop: worst reported pose {worst[0]:.3f} deg / {worst[1]:.3f} cm from the planted poses; branches {sorted(seen)}")
