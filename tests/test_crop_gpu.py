"""The pose-guided crop on the GPU (onepose_b200.crop / csrc/crop.cu) against the reference's own results
(tests/golden/pnp_crop_cases.npz, made by tests/golden/make_crop.py with OpenCV): pixels and transforms bit for bit."""
import os

import numpy as np
import pytest
import torch

from onepose_b200 import crop, pnp
from tests import crop_reference as cr
from tests.golden_util import GOLDEN_DIR

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def golden():
    g = dict(np.load(os.path.join(GOLDEN_DIR, "pnp_crop_cases.npz"), allow_pickle=False))
    g["frame_images"] = [cr.synthetic_frame(*(int(v) for v in f)) for f in g["frames"]]
    g["frame_tensors"] = [torch.from_numpy(f).to(DEV) for f in g["frame_images"]]
    return g


def _groups(g):
    """Case indices that one crop_frames call can take: the same frame and crop size."""
    keys = sorted({(int(f), int(s)) for f, s in zip(g["case_frame"], g["crop_size"])})
    return [(f, s, [i for i in range(len(g["box"])) if g["case_frame"][i] == f and g["crop_size"][i] == s]) for f, s in keys]


def _crop(g, f, S, idx):
    frames = g["frame_tensors"][f][None].expand(len(idx), -1, -1)          # frame stride 0: every case reads the one frame
    return crop.crop_frames(frames, torch.from_numpy(g["box"][idx]).to(DEV), torch.from_numpy(g["K"][idx]).to(DEV), S)


def test_crop_frames_equals_the_reference_bit_for_bit(golden):
    g = golden
    for f, S, idx in _groups(g):
        out = _crop(g, f, S, idx)
        assert out["image"].dtype == torch.float32 and tuple(out["image"].shape) == (len(idx), 1, S, S)
        img = out["image"].cpu().numpy()
        for k, i in enumerate(idx):
            ref = g[f"stage2_{i}"]
            assert np.array_equal(img[k, 0] * 255, ref), i
            assert np.array_equal(img[k, 0], ref.astype(np.float32) / 255), i                  # numpy's float32 division itself
            np.testing.assert_allclose(out["K_crop"][k].cpu().numpy(), g["K_crop"][i], rtol=1e-12, atol=0)
            assert np.array_equal(out["trans"][k].cpu().numpy(), np.stack([g["T1"][i], g["T2"][i]])), i
        assert out["status"].tolist() == [1] * len(idx)


def test_one_stage_drop_ins_equal_the_reference(golden):
    g = golden
    for i in range(len(g["box"])):
        x0, y0, x1, y1 = (int(v) for v in g["box"][i])
        S = int(g["crop_size"][i])
        im1, T1 = crop.get_image_crop_resize(g["frame_images"][g["case_frame"][i]], g["box"][i], [y1 - y0, x1 - x0])
        assert im1.dtype == np.uint8 and np.array_equal(im1, g[f"stage1_{i}"]), i
        assert T1.dtype == np.float64 and T1.shape == (3, 3) and np.array_equal(T1[:2], g["T1"][i]) and T1[2].tolist() == [0, 0, 1]
        im2, T2 = crop.get_image_crop_resize(im1, [0, 0, x1 - x0, y1 - y0], np.array([S, S]))
        assert im2.shape == (S, S) and np.array_equal(im2, g[f"stage2_{i}"]) and np.array_equal(T2[:2], g["T2"][i]), i
        K1, K1h = crop.get_K_crop_resize(g["box"][i], g["K"][i], [y1 - y0, x1 - x0])
        K2, K2h = crop.get_K_crop_resize(np.array([0, 0, x1 - x0, y1 - y0]), K1, [S, S])
        assert K2.shape == (3, 3) and K2h.shape == (3, 4) and K2.dtype == np.float64 and not K2h[:, 3].any()
        np.testing.assert_allclose(K2, g["K_crop"][i], rtol=1e-12, atol=0)


def test_boxes_from_poses_and_reproj(golden):
    g = golden
    K, pose, corners = (torch.from_numpy(g[k]).to(DEV) for k in ("sc_K", "sc_pose", "sc_corners"))
    box = crop.boxes_from_poses(K, pose, corners)
    assert box.dtype == torch.int32 and np.array_equal(box.cpu().numpy(), g["sc_box"])
    homo = torch.cat([pose, torch.tensor([0, 0, 0, 1.0], dtype=torch.float64, device=DEV).expand(len(pose), 1, 4)], dim=1)
    assert torch.equal(crop.boxes_from_poses(K, homo, corners), box)
    assert torch.equal(crop.boxes_from_poses(K[3], pose[3:4], corners[3]), box[3:4])              # shared K and box corners
    for i in range(len(pose)):
        p = crop.reproj(g["sc_K"][i], g["sc_pose"][i] if i % 2 else homo[i].cpu().numpy(), g["sc_corners"][i])
        assert p.shape == (8, 2) and p.dtype == np.float64
        np.testing.assert_allclose(p, g["sc_proj"][i], rtol=1e-12)


def test_unusable_pose_gives_the_empty_box_and_a_zero_image(golden):
    g = golden
    K, pose, corners = (torch.from_numpy(g[k][:4].copy()).to(DEV) for k in ("sc_K", "sc_pose", "sc_corners"))
    pose[0, 0, 3] = float("nan")
    pose[1, 2, 3] = float("inf")
    pose[2, 0, 3] = 1e9                                                    # finite, beyond int32
    frames = g["frame_tensors"][2][None].expand(4, -1, -1)
    bbox, image, K_crop = crop.previous_pose_detect(frames, K, pose, corners, crop_size=64)
    assert bbox[:3].tolist() == [[0, 0, 0, 0]] * 3 and np.array_equal(bbox[3].cpu().numpy(), g["sc_box"][3])
    out = crop.crop_frames(frames, bbox, K, 64)
    assert out["status"].tolist() == [0, 0, 0, 1]
    assert not image[:3].any() and image[3].any() and torch.equal(image, out["image"])
    assert torch.equal(K_crop[:3], K[:3]) and not out["trans"][:3].any()
    # boxes the crop rejects by itself: empty, inverted, too large, too far
    boxes = torch.tensor([[5, 5, 5, 9], [9, 5, 5, 9], [0, 0, 40000, 10], [1 << 21, 0, (1 << 21) + 9, 9]], dtype=torch.int32, device=DEV)
    assert crop.crop_frames(frames, boxes, K, 64)["status"].tolist() == [0, 0, 0, 0]


def test_strided_frames_and_batch_sizes_give_the_same_frames(golden):
    g = golden
    f = g["frame_images"][0]
    idx = [i for i in range(len(g["box"])) if g["case_frame"][i] == 0 and g["crop_size"][i] == 64]
    rng = np.random.default_rng(0)
    wide = torch.from_numpy(rng.integers(0, 256, (32, f.shape[0] + 6, f.shape[1] + 40), dtype=np.uint8)).to(DEV)
    view = wide[:, 3:3 + f.shape[0], 17:17 + f.shape[1]]
    view[::2] = torch.from_numpy(f).to(DEV)
    view[1::2] = torch.from_numpy(np.ascontiguousarray(f[::-1])).to(DEV)
    assert not view.is_contiguous()
    sel = [idx[k % len(idx)] for k in range(32)]
    boxes, K = torch.from_numpy(g["box"][sel]).to(DEV), torch.from_numpy(g["K"][sel]).to(DEV)
    full = crop.crop_frames(view, boxes, K, 64)
    for k in range(0, 32, 2):
        assert np.array_equal(full["image"][k, 0].cpu().numpy() * 255, g[f"stage2_{sel[k]}"]), k
    for B in (1, 3):
        for start in (0, 5):
            part = crop.crop_frames(view[start:start + B].contiguous(), boxes[start:start + B], K[start:start + B], 64)
            for key in ("image", "K_crop", "trans", "status"):
                assert torch.equal(part[key], full[key][start:start + B]), (B, start, key)


def test_results_on_a_side_stream_equal_the_default_stream(golden):
    g = golden
    f, S, idx = next(gr for gr in _groups(g) if gr[0] == 0 and gr[1] == 64)
    want = _crop(g, f, S, idx)
    sc = [torch.from_numpy(g[k]) for k in ("sc_K", "sc_pose", "sc_corners")]
    want_box = crop.boxes_from_poses(*(t.to(DEV) for t in sc))
    torch.cuda.synchronize()
    s = torch.cuda.Stream(DEV)
    with torch.cuda.stream(s):
        frames = (torch.from_numpy(g["frame_images"][f]).to(DEV, non_blocking=True).to(torch.int32) + 0).to(torch.uint8)   # made on s
        boxes = torch.from_numpy(g["box"][idx]).to(DEV) + 0
        got = crop.crop_frames(frames[None].expand(len(idx), -1, -1), boxes, torch.from_numpy(g["K"][idx]).to(DEV) * 1.0, S)
        got_box = crop.boxes_from_poses(*(t.to(DEV) * 1.0 for t in sc))
    s.synchronize()
    for key in ("image", "K_crop", "trans", "status"):
        assert torch.equal(got[key], want[key]), key
    assert torch.equal(got_box, want_box)


def test_every_output_element_is_written(golden, monkeypatch):
    g = golden
    made = []
    real_empty = torch.empty

    def poisoned(*a, **kw):
        t = real_empty(*a, **kw)
        t.fill_(float("nan") if t.dtype.is_floating_point else -1)
        made.append(t)
        return t

    monkeypatch.setattr(torch, "empty", poisoned)
    frames = g["frame_tensors"][0][None].expand(3, -1, -1)
    boxes = torch.tensor([[100, 80, 180, 150], [7, 7, 7, 7], [700, 100, 760, 150]], dtype=torch.int32, device=DEV)
    K = torch.from_numpy(g["K"][0]).to(DEV)
    out = crop.crop_frames(frames, boxes, K, 64)
    sc = [torch.from_numpy(g[k][:2]).to(DEV) for k in ("sc_K", "sc_pose", "sc_corners")]
    box = crop.boxes_from_poses(*sc)
    monkeypatch.undo()
    assert len(made) >= 5 and out["status"].tolist() == [1, 0, 1]
    for t in list(out.values()) + [box]:
        assert not (torch.isnan(t).any() if t.dtype.is_floating_point else (t == -1).any())
    assert not out["image"][1].any() and not out["image"][2].any() and out["image"][0].any()    # empty box; box outside the frame


def test_argument_mistakes_raise_before_any_launch(golden):
    g = golden
    frames = g["frame_tensors"][0][None]
    boxes = torch.tensor([[1, 1, 9, 9]], dtype=torch.int32, device=DEV)
    K = torch.eye(3, dtype=torch.float64, device=DEV)
    with pytest.raises(RuntimeError, match="no CPU path"):
        crop.crop_frames(frames.cpu(), boxes, K)
    with pytest.raises(RuntimeError, match="no CPU path"):
        crop.boxes_from_poses(K.cpu(), torch.zeros(1, 3, 4, dtype=torch.float64), torch.zeros(8, 3, dtype=torch.float64))
    with pytest.raises(RuntimeError, match="no CPU path"):
        crop.reproj(np.eye(3), np.eye(4), np.ones((8, 3)), device="cpu")
    for bad in (lambda: crop.crop_frames(frames.float(), boxes, K), lambda: crop.crop_frames(frames, boxes.long(), K),
                lambda: crop.crop_frames(frames, boxes, K, crop_size=100), lambda: crop.crop_frames(frames, boxes[:, :3], K),
                lambda: crop.crop_frames(frames[:, :, ::2], boxes, K), lambda: crop.crop_frames(frames, boxes, K[:2]),
                lambda: crop.boxes_from_poses(K, torch.zeros(1, 4, 3, dtype=torch.float64, device=DEV), torch.zeros(8, 3, dtype=torch.float64, device=DEV)),
                lambda: crop.get_image_crop_resize(g["frame_images"][0], [5, 5, 5, 9], [4, 4]),
                lambda: crop.get_image_crop_resize(g["frame_images"][0], [0.5, 0, 8, 8], [8, 8]),
                lambda: crop.get_K_crop_resize([0, 0, 8, 8], np.eye(4), [8, 8])):
        with pytest.raises(ValueError):
            bad()


def _look_at(t, rng):
    """A pose [3,4] with the object about 0.6 m in front of the camera, drifting and turning with t."""
    a, b = 0.3 + 0.08 * t, -0.2 + 0.05 * t
    Rz = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
    Rx = np.array([[1, 0, 0], [0, np.cos(b), -np.sin(b)], [0, np.sin(b), np.cos(b)]])
    return np.concatenate([Rx @ Rz, np.array([[-0.08 + 0.02 * t], [0.03 - 0.01 * t], [0.6 + 0.015 * t]])], axis=1)


def test_closed_loop_crop_pose_and_pixels_agree():
    """Frame t is cropped by the box of frame t-1's pose; the planted points' projections, carried into the crop by T2 . T1, give
    frame t's pose back through K_crop, and dots drawn at the projections in the full frame show up at the carried positions."""
    rng = np.random.default_rng(5)
    H, W, S, T, M = 480, 640, 512, 6, 80
    K = np.array([[620.0, 0, 318.5], [0, 615.0, 242.25], [0, 0, 1]])
    half = np.array([0.06, 0.045, 0.05])
    corners = np.array([[sx, sy, sz] for sx in (-1, 1) for sy in (-1, 1) for sz in (-1, 1)], np.float64) * half
    pts3d = rng.uniform(-1, 1, (M, 3)) * half * 0.9
    poses = np.stack([_look_at(t, rng) for t in range(T + 1)])
    proj = np.stack([cr.reproj(K, poses[t], pts3d) for t in range(1, T + 1)])                   # [T, M, 2] in the full frame
    frames = np.zeros((T, H, W), np.uint8)
    for t in range(T):
        for u, v in np.rint(proj[t]).astype(int):
            frames[t, max(v - 1, 0):v + 2, max(u - 1, 0):u + 2] = 255
    Kd = torch.from_numpy(K).to(DEV)
    bbox, image, K_crop = crop.previous_pose_detect(torch.from_numpy(frames).to(DEV), Kd, torch.from_numpy(poses[:T]).to(DEV),
                                                    torch.from_numpy(corners).to(DEV), crop_size=S)
    out = crop.crop_frames(torch.from_numpy(frames).to(DEV), bbox, Kd, S)
    assert out["status"].tolist() == [1] * T and torch.equal(out["image"], image)
    tr = out["trans"].cpu().numpy()
    kp = np.zeros((T, M, 2))
    for t in range(T):
        assert np.array_equal(bbox[t].cpu().numpy(), cr.box_from_pose(K, poses[t], corners))
        homo = [np.concatenate([tr[t, s], [[0, 0, 1.0]]]) for s in (0, 1)]
        kp[t] = (homo[1] @ homo[0] @ np.concatenate([proj[t], np.ones((M, 1))], axis=1).T).T[:, :2]
        np.testing.assert_allclose(homo[1] @ homo[0] @ K, K_crop[t].cpu().numpy(), rtol=1e-12)
    res = pnp.poses_from_matches(K_crop, torch.from_numpy(kp).to(DEV, torch.float32), torch.from_numpy(pts3d).to(DEV, torch.float32),
                                 torch.arange(M, device=DEV).expand(T, M), scale=1000)
    rot, trans = pnp.pose_errors(res["pose"], torch.from_numpy(poses[1:]).to(DEV))
    assert float(rot.max()) < 1.0 and float(trans.max()) < 1.0, (rot, trans)
    assert int(res["n_inliers"].min()) >= M - 2
    img = image[:, 0].cpu().numpy()
    seen = 0
    for t in range(T):
        for u, v in np.rint(kp[t]).astype(int):
            if 2 <= u < S - 2 and 2 <= v < S - 2:
                assert img[t, v - 1:v + 2, u - 1:u + 2].max() > 0.5, (t, u, v)
                seen += 1
    assert seen > T * M // 2 and img.mean() < 0.2                                                # dots, not a white image
