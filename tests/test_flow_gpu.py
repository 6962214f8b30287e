"""The tracker's flow step on the GPU against cv2 4.13 and the reference's BATracker.flow_track, through the goldens of
tests/golden/make_flow.py (the GPU machines need neither cv2 nor the reference)."""
import os

import numpy as np
import pytest
import torch

from onepose_b200 import _lib, crop, flow, pnp
from tests import flow_scenes as FS
from tests import lk_reference as L

pytestmark = pytest.mark.gpu
DEV = "cuda"
Z = np.load(os.path.join(os.path.dirname(__file__), "golden", "pnp_flow_cases.npz"))
LK = range(6)


def _scene(i):
    p = Z[f"lk{i}_params"]
    return (Z[f"lk{i}_prev"], Z[f"lk{i}_next"], Z[f"lk{i}_pts"], (int(p[0]), int(p[1])), int(p[2]), (int(p[3]), int(p[4]), float(p[5])))


def _run(prev, nxt, pts, offsets, win, lev, crit, **kw):
    return flow.lk_batch(prev, nxt, pts, offsets, win, lev, crit, **kw)


def _compare(i, pts, st, err, label=""):
    cs, cp, ce = Z[f"lk{i}_status"], Z[f"lk{i}_next_pts"], Z[f"lk{i}_err"]
    st, pts, err = st.cpu().numpy(), pts.cpu().numpy(), err.cpu().numpy()
    np.testing.assert_array_equal(st, cs)
    m = cs == 1
    d = np.abs(pts[m] - cp[m]).max()
    print(f"scene {i}{label}: {int((pts[m] == cp[m]).all(1).sum())} of {int(m.sum())} status-1 points bit-equal, max |dpt| {d:.3g}, "
          f"{int((err[m] == ce[m]).sum())} err bit-equal")
    assert d <= 1e-3
    np.testing.assert_allclose(err[m], ce[m], rtol=1e-4, atol=0)
    assert np.all(err[~m] == 0)


@pytest.mark.parametrize("i", LK)
def test_lk_goldens(i):
    prev, nxt, pts, win, lev, crit = _scene(i)
    H, W = prev.shape
    ws = torch.full((flow.workspace_bytes(1, H, W, lev),), 0xAB, dtype=torch.uint8, device=DEV)
    p, s, e = _run(torch.from_numpy(prev)[None].to(DEV), torch.from_numpy(nxt)[None].to(DEV), torch.from_numpy(pts).to(DEV),
                   torch.tensor([0, len(pts)], dtype=torch.int32, device=DEV), win, lev, crit, workspace=ws)
    _compare(i, p, s, e)
    levels = flow.pyramid_views(ws, 1, H, W, lev, win, 0)
    assert len(levels) == int(Z[f"lk{i}_levels"]) + 1
    for level, (ip, inx, der) in enumerate(levels):
        np.testing.assert_array_equal(der.cpu().numpy(), Z[f"lk{i}_pyr_der{level}"])
        if level:
            np.testing.assert_array_equal(ip.cpu().numpy(), Z[f"lk{i}_pyr_prev{level}"])
            np.testing.assert_array_equal(inx.cpu().numpy(), Z[f"lk{i}_pyr_next{level}"])


@pytest.mark.parametrize("B", [1, 7, 64])
def test_batched_sizes_ragged_strided(B):
    """B pairs of different sizes in one call -- crops of golden scene 1 from 40 x 50 to its full 120 x 160, in padded slots
    with a row stride past the width -- with ragged and empty point sets, against the numpy model on each pair alone."""
    prev, nxt, pts, win, lev, crit = _scene(1)
    rs = np.random.RandomState(B)
    H, W = prev.shape
    big_p = torch.zeros(B, H, W + 9, dtype=torch.uint8, device=DEV)
    big_n = torch.zeros(B, H, W + 9, dtype=torch.uint8, device=DEV)
    sizes, plist, offs = [], [], [0]
    for b in range(B):
        h, w = (H, W) if b == 0 else (int(rs.randint(40, H + 1)), int(rs.randint(50, W + 1)))
        big_p[b, :h, :w] = torch.from_numpy(prev[:h, :w])
        big_n[b, :h, :w] = torch.from_numpy(nxt[:h, :w])
        sizes.append((h, w))
        n = 0 if b % 5 == 3 else int(rs.randint(1, 60))
        plist.append(np.stack([rs.uniform(-10, w + 10, n), rs.uniform(-10, h + 10, n)], 1).astype(np.float32))
        offs.append(offs[-1] + n)
    p, s, e = _run(big_p[:, :, :W], big_n[:, :, :W], torch.from_numpy(np.concatenate(plist)).to(DEV),
                   torch.tensor(offs, dtype=torch.int32, device=DEV), win, lev, crit, sizes=torch.tensor(sizes, dtype=torch.int32, device=DEV))
    p, s, e = p.cpu().numpy(), s.cpu().numpy(), e.cpu().numpy()
    for b in range(B):
        h, w = sizes[b]
        rp, rst, rerr = L.calc_optical_flow_pyr_lk(prev[:h, :w], nxt[:h, :w], plist[b], win, lev, crit)
        sl = slice(offs[b], offs[b + 1])
        np.testing.assert_array_equal(s[sl], rst)
        m = rst == 1
        np.testing.assert_array_equal(p[sl][m], rp[m])
        np.testing.assert_array_equal(e[sl][m], rerr[m])


def test_side_stream_and_fully_written():
    """The C entry point on a side stream writes every element of its outputs: they start as NaN / 0xAB sentinels."""
    prev, nxt, pts, win, lev, crit = _scene(1)
    a, b = torch.from_numpy(prev)[None].to(DEV), torch.from_numpy(nxt)[None].to(DEV)
    t = torch.from_numpy(pts).to(DEV)
    n = len(pts)
    off = torch.tensor([0, n], dtype=torch.int32, device=DEV)
    nbytes = flow.workspace_bytes(1, *prev.shape, lev)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ws = torch.full((nbytes,), 0x7F, dtype=torch.uint8, device=DEV)
        nxt_pts = torch.full((n, 2), float("nan"), device=DEV)
        st = torch.full((n,), 0xAB, dtype=torch.uint8, device=DEV)
        err = torch.full((n,), float("nan"), device=DEV)
        _lib.call(a.device, "opb_calc_optical_flow_pyr_lk", a, a.stride(0), a.stride(1), b, b.stride(0), b.stride(1), 1, *prev.shape, None, t, off, n,
                  win[0], win[1], lev, crit[0], crit[1], crit[2], 1e-4, 0, ws, nbytes, nxt_pts, st, err)
    s.synchronize()
    assert torch.isfinite(nxt_pts).all() and torch.isfinite(err).all() and bool(((st == 0) | (st == 1)).all())
    _compare(1, nxt_pts, st, err, " (side stream)")


def test_numpy_drop_in():
    prev, nxt, pts, win, lev, crit = _scene(2)
    p, s, e = flow.calc_optical_flow_pyr_lk(prev, nxt, pts[:, None], None, winSize=win, maxLevel=lev, criteria=crit)
    assert p.shape == (len(pts), 1, 2) and s.shape == (len(pts), 1) and e.shape == (len(pts), 1)
    assert p.dtype == np.float32 and s.dtype == np.uint8 and e.dtype == np.float32
    _compare(2, torch.from_numpy(p[:, 0]), torch.from_numpy(s[:, 0]), torch.from_numpy(e[:, 0]), " (drop-in)")
    with pytest.raises(ValueError):
        flow.calc_optical_flow_pyr_lk(prev, nxt, pts, flags=flow.OPTFLOW_USE_INITIAL_FLOW)


def test_argument_errors():
    img = torch.zeros(1, 64, 64, dtype=torch.uint8, device=DEV)
    pts = torch.zeros(4, 2, device=DEV)
    off = torch.tensor([0, 4], dtype=torch.int32, device=DEV)
    for kw in [dict(win_size=(4, 5)), dict(win_size=(33, 33)), dict(max_level=5), dict(criteria=(0, 10, 0.1)), dict(criteria=(1, 0, 0.1)),
               dict(criteria=(2, 10, -1.0)), dict(min_eig_threshold=-1.0)]:
        with pytest.raises(ValueError):
            flow.lk_batch(img, img, pts, off, **kw)
    with pytest.raises(ValueError):
        flow.lk_batch(img, img[:, :32], pts, off)
    with pytest.raises(ValueError):
        flow.lk_batch(img, img, pts, off, workspace=torch.empty(10, dtype=torch.uint8, device=DEV))
    lib = _lib.load()
    rc = lib.opb_calc_optical_flow_pyr_lk(img.data_ptr(), 4096, 64, img.data_ptr(), 4096, 64, 1, 64, 64, None, pts.data_ptr(), off.data_ptr(), 4,
                                          15, 15, 2, 3, 10, 0.03, 1e-4, 4, img.data_ptr(), 1 << 30, pts.data_ptr(), img.data_ptr(), pts.data_ptr(), None)
    assert rc == -1 and b"flags == 0" in lib.opb_last_error(None)


def _ft_batch(cases):
    cap = int(Z["ft_cap"])
    B = len(cases)
    kf = {"image": torch.from_numpy(np.stack([Z["ft_kf_image"]] * B)).to(DEV),
          "pts2d": torch.from_numpy(np.stack([Z[f"ft{c}_pts2d"] for c in cases])).to(DEV),
          "pts3d": torch.from_numpy(np.stack([Z[f"ft{c}_pts3d"] for c in cases])).to(DEV),
          "counts": torch.tensor([int(Z[f"ft{c}_count"]) for c in cases], dtype=torch.int32, device=DEV)}
    query = torch.from_numpy(np.stack([Z[f"ft{c}_query"] for c in cases])).to(DEV)
    ref = torch.from_numpy(np.stack([Z[f"ft{c}_pose_ref"] for c in cases])).to(DEV)
    return kf, query, ref, cap


def test_flow_track_goldens():
    """flow_track against the reference's BATracker.flow_track on a non-planar object: the tracked points bit for bit, n_tracked,
    n_inliers and accept equal, the pose within 0.1 degree / 0.25 cm (test_epnp_cv_gpu.py's bar), kpt_dist (see below), and
    the accepted keyframe state equal to the reference's last_kf_info."""
    cases = list(range(len(Z["ft_names"])))
    kf, query, ref, cap = _ft_batch(cases)
    K = torch.from_numpy(Z["ft_K"]).to(DEV)
    tracked, status, _ = flow.lk_batch(kf["image"], query, kf["pts2d"].reshape(-1, 2), torch.arange(0, (len(cases) + 1) * cap, cap, dtype=torch.int32,
                                                                                                       device=DEV))
    out = flow.flow_track(kf, query, K, ref)
    torch.cuda.synchronize()
    for b, c in enumerate(cases):
        name = str(Z["ft_names"][c])
        n = int(Z[f"ft{c}_count"])
        rows = slice(b * cap, b * cap + n)
        np.testing.assert_array_equal(status[rows].cpu().numpy(), Z[f"ft{c}_status"], err_msg=name)
        m = Z[f"ft{c}_status"] == 1
        np.testing.assert_array_equal(tracked[rows].cpu().numpy()[m], Z[f"ft{c}_tracked"][m], err_msg=name)
        assert int(out["n_tracked"][b]) == int(Z[f"ft{c}_n_tracked"]), name
        assert int(out["n_inliers"][b]) == int(Z[f"ft{c}_n_inliers"]), name
        assert bool(out["accept"][b]) == bool(Z[f"ft{c}_accept"]), name
        # The pose: test_epnp_cv_gpu.py's 0.1 degree / 0.25 cm for a clean track (every tracked point an inlier).  "large" keeps
        # 29 inliers of 80 mis-tracked points, several px off; EPnP's refit on them is ill-conditioned, and its pose is
        # held to 1 degree / 1 cm.  In both, the isolated solve below shows the gap is the solver's, not the flow step's.
        rot, trans = pnp.pose_errors(out["pose_init_homo"][b:b + 1], torch.from_numpy(Z[f"ft{c}_pose"][None]).to(DEV))
        clean = int(Z[f"ft{c}_n_inliers"]) == int(Z[f"ft{c}_n_tracked"])
        assert float(rot) <= (0.1 if clean else 1.0) and float(trans) <= (0.25 if clean else 1.0), (name, float(rot), float(trans))
        kd, rk = float(out["kpt_dist"][b]), float(Z[f"ft{c}_kpt_dist"])
        k = int(Z[f"ft{c}_n_tracked"])
        if k < 4:                               # cv2.error branch: the identity pose on both sides, the same arithmetic
            assert (np.isnan(kd) and np.isnan(rk)) or abs(kd - rk) <= 1e-9 * abs(rk), (name, kd, rk)
        else:
            # The solve in isolation: EPnP-RANSAC on the reference's own tracked points gives flow_track's pose bit for bit, so
            # flow_track feeds the solver exactly what the reference's ransac_PnP received; what remains is the solver's own
            # parity with cv2.solvePnPRansac on noisy points (0.1 degree / 0.25 cm, test_epnp_cv_gpu.py).
            p2 = torch.from_numpy(Z[f"ft{c}_tracked"][m].astype(np.float64)).to(DEV)
            p3 = torch.from_numpy(Z[f"ft{c}_pts3d"][:n][m].astype(np.float64)).to(DEV)
            iso, _, iso_n = pnp.ransac_pnp_batch(K[None], p2, p3, torch.tensor([0, k], dtype=torch.int32, device=DEV), reproj_error=5.0,
                                                 hypotheses=10000, method="epnp", confidence=0.99)
            assert torch.equal(iso[0], out["pose_init_homo"][b, :3]) and int(iso_n[0]) == int(out["n_inliers"][b]), name
            # kpt_dist is tracking_utils.project's mean distance on the device's pose, to 1e-9 ...
            P = out["pose_init_homo"][b, :3].cpu().numpy()
            X = Z[f"ft{c}_pts3d"][:n][m].astype(np.float64) @ P[:, :3].T + P[:, 3]
            X = X @ Z["ft_K"].T
            want = np.mean(np.linalg.norm(X[:, :2] / X[:, 2:] - Z[f"ft{c}_tracked"][m].astype(np.float64), axis=1))
            assert abs(kd - want) <= 1e-9 * want, (name, kd, want)
            # ... and moves with the pose: within 0.1 degree / 0.25 cm of cv2's pose it stays within 5 % of the reference's
            assert abs(kd - rk) <= 0.05 * rk, (name, kd, rk)
        nk = out["kf"]
        if bool(Z[f"ft{c}_accept"]):
            assert int(nk["counts"][b]) == k
            np.testing.assert_array_equal(nk["image"][b].cpu().numpy(), Z[f"ft{c}_query"])
            np.testing.assert_array_equal(nk["pts3d"][b, :k].cpu().numpy(), Z[f"ft{c}_kf_pts3d"])
            np.testing.assert_array_equal(nk["pts2d"][b, :k].cpu().numpy(), Z[f"ft{c}_kf_pts2d"])
            assert not nk["pts2d"][b, k:].any()
        else:
            assert torch.equal(nk["image"][b], kf["image"][b]) and torch.equal(nk["pts2d"][b], kf["pts2d"][b])
            assert int(nk["counts"][b]) == int(kf["counts"][b])
        print(f"{name}: n_tracked {int(out['n_tracked'][b])}, n_inliers {int(out['n_inliers'][b])}, kpt_dist {kd} (reference {rk}), "
              f"pose vs reference {float(rot):.2e} deg / {float(trans):.2e} cm, accept {bool(out['accept'][b])}")


def test_flow_track_multi_object_rows():
    """K tracks over shared frames: each object's query crop cut by crop_frames(frame_index=...) from one frame tensor."""
    cases = [0, 1, 3]
    kf, query, ref, cap = _ft_batch(cases)
    frames = query[[0, 1]]
    frame_index = torch.tensor([0, 1, 0], dtype=torch.int32, device=DEV)
    S = frames.shape[-1]
    boxes = torch.tensor([[0, 0, S, S]] * 3, dtype=torch.int32, device=DEV)
    K = torch.from_numpy(Z["ft_K"]).to(DEV)
    c = crop.crop_frames(frames, boxes, K, S, frame_index=frame_index)
    q = flow._u8_crops(c["image"], "q")
    assert torch.equal(q[0], query[0]) and torch.equal(q[1], query[1])
    out = flow.flow_track(kf, c["image"], c["K_crop"], ref)
    solo = flow.flow_track({k: v[:2] for k, v in kf.items()}, query[:2], K, ref[:2])
    for k in ("n_tracked", "n_inliers", "accept"):
        assert torch.equal(out[k][:2], solo[k])
    assert torch.equal(out["pose_init_homo"][:2], solo["pose_init_homo"])


def test_keyframes_from_poses():
    """The inlier pairs of each frame in pair order, as mkpts2d[inliers.flatten()] of inference_demo.py:266-267."""
    rs = np.random.RandomState(3)
    B, N = 4, 50
    lens = [50, 0, 17, 33]
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    p2 = rs.rand(B * N, 2).astype(np.float32).astype(np.float64)
    p3 = rs.rand(B * N, 3).astype(np.float32).astype(np.float64)
    mask = rs.rand(B * N) < 0.6
    res = {"offsets": torch.from_numpy(off).to(DEV), "inlier_mask": torch.from_numpy(mask).to(DEV), "pts2d": torch.from_numpy(p2).to(DEV),
           "pts3d": torch.from_numpy(p3).to(DEV)}
    crops = torch.randint(0, 255, (B, 32, 32), dtype=torch.uint8, device=DEV)
    kf = flow.keyframes_from_poses(res, crops)
    assert kf["pts2d"].shape == (B, N, 2) and kf["pts3d"].shape == (B, N, 3) and kf["counts"].dtype == torch.int32
    for b in range(B):
        rows = np.arange(off[b], off[b + 1])
        rows = rows[mask[rows]]
        n = len(rows)
        assert int(kf["counts"][b]) == n
        np.testing.assert_array_equal(kf["pts2d"][b, :n].cpu().numpy(), p2[rows].astype(np.float32))
        np.testing.assert_array_equal(kf["pts3d"][b, :n].cpu().numpy(), p3[rows].astype(np.float32))
        assert not kf["pts2d"][b, n:].any()
    assert torch.equal(kf["image"], crops)


def test_closed_loop():
    """20 frames of planted motion of two non-planar objects seen by their own crops: every 5th frame the keyframes come from
    poses_from_matches on planted matches (keyframes_from_poses), the other frames go through flow_track from the last
    keyframe.  Every flow pose is accepted and within 1 cm / 1 degree of the planted pose."""
    S = 192
    K = np.array([[450.0, 0, S / 2], [0, 450.0, S / 2], [0, 0, 1]])
    objs = [FS.blob_object(21, 80), FS.blob_object(22, 70)]
    pose0 = [np.concatenate([FS.rodrigues([0.1, 0.2, -0.05]), [[0.01], [-0.01], [0.45]]], 1),
             np.concatenate([FS.rodrigues([-0.2, 0.05, 0.1]), [[-0.01], [0.0], [0.5]]], 1)]
    steps = [(np.array([0.004, -0.003, 0.002]), np.array([0.0008, -0.0006, 0.0012])),
             (np.array([-0.003, 0.004, -0.002]), np.array([-0.0006, 0.0009, -0.001]))]
    B, N = 2, 80
    Kd = torch.from_numpy(K).to(DEV)
    kp3 = {k: torch.from_numpy(objs[k][0]).to(DEV) for k in range(B)}
    rs = np.random.RandomState(5)
    kf, worst = None, (0.0, 0.0)
    for f in range(20):
        truth = [FS.pose_at(pose0[k], f * steps[k][0], f * steps[k][1]) for k in range(B)]
        imgs = torch.from_numpy(np.stack([FS.render_blobs(K, truth[k], *objs[k], S) for k in range(B)])).to(DEV)
        if f % 5 == 0:
            kp2 = np.zeros((B, N, 2), np.float32)
            m0 = np.full((B, N), -1, np.int64)
            for k in range(B):
                M = len(objs[k][0])
                kp2[k, :M] = FS.project(K, truth[k], objs[k][0]) + 0.2 * rs.randn(M, 2)
                m0[k, :M] = np.arange(M)
            res = pnp.poses_from_matches_objects(Kd, torch.from_numpy(kp2).to(DEV), kp3, [0, 1], torch.from_numpy(m0).to(DEV), scale=1000,
                                                 method="epnp", confidence=0.99)
            kf = flow.keyframes_from_poses(res, imgs)
            assert kf["counts"].tolist() == res["n_inliers"].tolist()
            continue
        ref = torch.from_numpy(np.stack([np.concatenate([t, [[0, 0, 0, 1.0]]]) for t in truth])).to(DEV)
        out = flow.flow_track(kf, imgs, Kd, ref)
        rot, trans = pnp.pose_errors(out["pose_init_homo"], ref)
        assert out["accept"].all(), (f, out["kpt_dist"].tolist(), rot.tolist(), trans.tolist())
        assert (rot < 1.0).all() and (trans < 1.0).all(), (f, rot.tolist(), trans.tolist())
        worst = (max(worst[0], float(rot.max())), max(worst[1], float(trans.max())))
        kf = out["kf"]
    print(f"closed loop: worst flow pose {worst[0]:.3f} deg / {worst[1]:.3f} cm from the planted poses")
