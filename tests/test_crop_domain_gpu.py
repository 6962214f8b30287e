"""The crop on the GPU (onepose_b200.crop / csrc/crop.cu) over the whole domain its entry points accept, against the numpy model
(tests/crop_reference.py, which equals cv2 4.13 on the CPU): uint8 pixels (image * 255), trans and status bit for bit, K_crop
to rtol 1e-12.  Outputs and boxes too large for the array model are compared at sampled positions through crop_pixels."""
import numpy as np
import pytest
import torch

from onepose_b200 import crop
from tests import crop_reference as cr

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
M20 = 1 << 20


def _probe_positions(h, w, n, seed):
    """Every pixel of the first and last rows and columns, and n seeded random positions: (xs, ys)."""
    rng = np.random.default_rng(seed)
    ex = np.concatenate([np.arange(w), np.arange(w), np.zeros(h, np.int64), np.full(h, w - 1)])
    ey = np.concatenate([np.zeros(w, np.int64), np.full(w, h - 1), np.arange(h), np.arange(h)])
    return np.concatenate([ex, rng.integers(0, w, n)]), np.concatenate([ey, rng.integers(0, h, n)])


def _model_K(box, K, S):
    """crop_img_by_bbox's K_crop without its images."""
    x0, y0, x1, y1 = (int(v) for v in box)
    K1, _ = cr.get_K_crop_resize(box, K, [y1 - y0, x1 - x0])
    return cr.get_K_crop_resize([0, 0, x1 - x0, y1 - y0], K1, [S, S])[0]


def _check_sampled(frame, out, k, box, K, S, seed):
    """Frame k of a crop_frames result against the model at the edges and 20000 random positions of its S x S image."""
    xs, ys = _probe_positions(S, S, 20000, seed)
    got = (out["image"][k, 0][torch.from_numpy(ys).to(DEV), torch.from_numpy(xs).to(DEV)] * 255).cpu().numpy()
    want = cr.crop_pixels(frame, box, S, xs, ys)
    bad = np.nonzero(got != want)[0]
    assert not len(bad), (box, S, "first differing pixel (x, y)", int(xs[bad[0]]), int(ys[bad[0]]), got[bad[0]], want[bad[0]])
    T1, T2 = cr.crop_transforms(box, S)
    assert np.array_equal(out["trans"][k].cpu().numpy(), np.stack([T1, T2])), box
    np.testing.assert_allclose(out["K_crop"][k].cpu().numpy(), _model_K(box, K, S), rtol=1e-12, atol=0)
    assert int(out["status"][k]) == 1


def _check_rejected(out, k, K):
    assert int(out["status"][k]) == 0 and not out["trans"][k].any() and not out["image"][k].any()
    assert torch.equal(out["K_crop"][k], K if K.dim() == 2 else K[k])


@pytest.fixture(scope="module")
def sweep():
    frames = [cr.synthetic_frame(h, w, k) for k, (h, w) in enumerate(cr.SWEEP_FRAMES)]
    return cr.sweep_cases(), frames, [torch.from_numpy(f).to(DEV) for f in frames]


def test_random_sweep_equals_the_model(sweep):
    """About 1000 boxes inside, crossing, outside and larger than six frames from 1 x 1 to 1440 x 1920, S = 8 .. 512 and two
    2048 crops that meet rounding ties, per-frame K: full images, transforms, K_crop and status."""
    cases, frames, frames_t = sweep
    groups = {}
    for i, (f, _, S, _) in enumerate(cases):
        groups.setdefault((f, S), []).append(i)
    for (f, S), idx in groups.items():
        boxes = torch.from_numpy(np.stack([cases[i][1] for i in idx])).to(DEV)
        K = torch.from_numpy(np.stack([cases[i][3] for i in idx])).to(DEV)
        out = crop.crop_frames(frames_t[f][None].expand(len(idx), -1, -1), boxes, K, S)
        img = out["image"][:, 0].cpu().numpy() * 255
        for k, i in enumerate(idx):
            _, box, _, Ki = cases[i]
            _, im2, T1, T2, K_crop = cr.crop_img_by_bbox(frames[f], box, Ki, S)
            bad = np.argwhere(img[k] != im2)
            assert not len(bad), (i, box.tolist(), S, "first differing pixel (y, x)", bad[0].tolist())
            assert np.array_equal(out["trans"][k].cpu().numpy(), np.stack([T1, T2])), (i, box.tolist())
            np.testing.assert_allclose(out["K_crop"][k].cpu().numpy(), K_crop, rtol=1e-12, atol=0)
        assert out["status"].tolist() == [1] * len(idx)


def test_one_stage_drop_ins_over_the_sweep(sweep):
    """opb_warp_crop_u8 in its three forms -- pixels, transform only, K only -- on every third sweep box, to a rectangular
    out_h x out_w of 1 .. 600 a side."""
    cases, frames, _ = sweep
    rng = np.random.default_rng(4)
    for i, (f, box, _, K) in enumerate(cases[::3]):
        oh, ow = (int(v) for v in np.exp(rng.uniform(0, np.log(601), 2)))
        im, T = crop.get_image_crop_resize(frames[f], box, [oh, ow], device=DEV)
        want, Tw = cr.get_image_crop_resize(frames[f], box, [oh, ow])
        assert im.shape == (oh, ow) and np.array_equal(im, want), (i, box.tolist(), oh, ow)
        assert np.array_equal(T, Tw), (i, box.tolist())
        _, T_only, _ = crop._warp_crop_np(None, box, None, [oh, ow], DEV)
        assert np.array_equal(T_only, Tw[:2]), (i, box.tolist())
        Kc, _ = crop.get_K_crop_resize(box, K, [oh, ow], device=DEV)
        np.testing.assert_allclose(Kc, cr.get_K_crop_resize(box, K, [oh, ow])[0], rtol=1e-12, atol=0)


EDGE_ACCEPTED = [(-100, -200, -100 + 32767, -200 + 32767),          # sides 32767
                 (5, 7, 6, 7 + 32767), (-M20, -M20, -M20 + 40, -M20 + 30), (M20 - 40, M20 - 30, M20, M20),
                 (-M20, M20 - 32767, -M20 + 32767, M20)]
EDGE_REJECTED = [(0, 0, 32768, 10), (0, 0, 10, 32768),                 # a side of 32768
                 (-M20 - 1, 0, -M20 + 9, 10), (M20 - 9, 0, M20 + 1, 10), (0, -M20 - 1, 10, -M20 + 9), (0, M20 - 9, 10, M20 + 1),
                 (5, 5, 5, 9), (5, 9, 15, 8)]                          # x1 = x0, y1 < y0


def test_domain_edges():
    frame = cr.synthetic_frame(480, 640, 1)
    boxes = EDGE_ACCEPTED + EDGE_REJECTED
    K = torch.tensor([[600.0, 0, 320.5], [0, 610.0, 240.25], [0, 0, 1]], dtype=torch.float64, device=DEV)
    out = crop.crop_frames(torch.from_numpy(frame).to(DEV)[None].expand(len(boxes), -1, -1),
                           torch.tensor(boxes, dtype=torch.int32, device=DEV), K, 512)
    for k, box in enumerate(EDGE_ACCEPTED):
        _check_sampled(frame, out, k, box, K.cpu().numpy(), 512, k)
    for k in range(len(EDGE_ACCEPTED), len(boxes)):
        _check_rejected(out, k, K)


@pytest.mark.parametrize("shape,box,S", [((480, 640), (300, 200, 301, 201), 2048),     # 1 x 1, dense with rounding ties
                                         ((1440, 1920), (-15000, -16000, -15000 + 32767, -16000 + 32767), 8),
                                         ((1440, 1920), (-15000, -16000, -15000 + 32767, -16000 + 32767), 512)])
def test_extreme_scales(shape, box, S):
    frame = cr.synthetic_frame(*shape, 2)
    K = np.array([[900.0, 0, shape[1] / 2], [0, 900.0, shape[0] / 2], [0, 0, 1]])
    out = crop.crop_frames(torch.from_numpy(frame).to(DEV)[None], torch.tensor([box], dtype=torch.int32, device=DEV),
                           torch.from_numpy(K).to(DEV), S)
    _check_sampled(frame, out, 0, box, K, S, 7)


def test_largest_crop_size():
    """One frame to S = 32760, the largest multiple of 8 the crop accepts.  Its fp32 image is 32760^2 * 4 B = 4.3 GB on the
    device; the test frees it before it returns."""
    frame = cr.synthetic_frame(480, 640, 3)
    box, S = (-37, 11, 611, 500), 32760
    K = np.array([[700.0, 0, 330.0], [0, 700.0, 250.0], [0, 0, 1]])
    torch.cuda.reset_peak_memory_stats(DEV)
    out = crop.crop_frames(torch.from_numpy(frame).to(DEV)[None], torch.tensor([box], dtype=torch.int32, device=DEV),
                           torch.from_numpy(K).to(DEV), S)
    _check_sampled(frame, out, 0, box, K, S, 9)
    print(f"S = {S}: peak device memory {torch.cuda.max_memory_allocated(DEV) / 2**30:.2f} GiB")
    del out
    torch.cuda.empty_cache()


@pytest.mark.parametrize("H,W", [(32767, 64), (64, 32767)])
def test_frames_at_the_side_limit(H, W):
    """Frames of 32767 pixels a side as strided views (row and frame strides beyond the frame), boxes on their far edges."""
    frame = cr.synthetic_frame(H, W, 4)
    buf = torch.zeros(2, H + 3, W + 24, dtype=torch.uint8, device=DEV)
    view = buf[:, 1:1 + H, 5:5 + W]
    view.copy_(torch.from_numpy(frame).to(DEV)[None].expand(2, -1, -1))
    assert not view.is_contiguous()
    far = [(W - 24, H - 60, W + 36, H + 20), (W - 1, H - 1, W + 1, H + 1)] if H > W else [(W - 60, H - 24, W + 20, H + 36), (W - 1, H - 1, W + 1, H + 1)]
    K = np.array([[500.0, 0, W / 2], [0, 500.0, H / 2], [0, 0, 1]])
    out = crop.crop_frames(view, torch.tensor(far, dtype=torch.int32, device=DEV), torch.from_numpy(K).to(DEV), 64)
    for k, box in enumerate(far):
        _, im2, T1, T2, K_crop = cr.crop_img_by_bbox(frame, box, K, 64)
        assert np.array_equal(out["image"][k, 0].cpu().numpy() * 255, im2), box
        assert np.array_equal(out["trans"][k].cpu().numpy(), np.stack([T1, T2])), box
        np.testing.assert_allclose(out["K_crop"][k].cpu().numpy(), K_crop, rtol=1e-12, atol=0)
    assert out["status"].tolist() == [1, 1] and out["image"].any()


def test_65535_frames_in_one_call():
    """The most frames one call takes: one frame at stride 0, a cycle of 7 distinct boxes.  Each box is compared with the model
    once, and every repeat must be bit-identical to its first crop."""
    frame = cr.synthetic_frame(96, 128, 6)
    distinct = [(10, 20, 60, 70), (-30, -10, 50, 40), (100, 80, 140, 120), (0, 0, 128, 96), (-200, -150, 300, 250),
                (127, 95, 128, 96), (500, 500, 510, 510)]
    B = crop.MAX_FRAMES
    cyc = torch.arange(B, device=DEV) % 7
    K = np.array([[300.0, 0, 64.0], [0, 300.0, 48.0], [0, 0, 1]])
    out = crop.crop_frames(torch.from_numpy(frame).to(DEV)[None].expand(B, -1, -1),
                           torch.tensor(distinct, dtype=torch.int32, device=DEV)[cyc], torch.from_numpy(K).to(DEV), 8)
    for k, box in enumerate(distinct):
        _, im2, T1, T2, K_crop = cr.crop_img_by_bbox(frame, box, K, 8)
        assert np.array_equal(out["image"][k, 0].cpu().numpy() * 255, im2), box
        assert np.array_equal(out["trans"][k].cpu().numpy(), np.stack([T1, T2])), box
        np.testing.assert_allclose(out["K_crop"][k].cpu().numpy(), K_crop, rtol=1e-12, atol=0)
    for key in ("image", "trans", "K_crop", "status"):
        assert torch.equal(out[key], out[key][:7][cyc]), key
    assert out["status"].sum().item() == B


def _random_poses(rng, B):
    """Poses with the object 1 .. 3 in front of the camera and principal points far enough from 0 that every projection
    is at least 25 pixels from it (so rtol bounds the difference of summation orders)."""
    q, _ = np.linalg.qr(rng.normal(size=(B, 3, 3)))
    t = np.stack([rng.uniform(-0.1, 0.1, B), rng.uniform(-0.1, 0.1, B), rng.uniform(1, 3, B)], 1)
    pose = np.concatenate([q, t[:, :, None]], axis=2)
    f = rng.uniform(300, 1500, B)
    K = np.zeros((B, 3, 3))
    K[:, 0, 0], K[:, 1, 1], K[:, 0, 2], K[:, 1, 2], K[:, 2, 2] = f, f * rng.uniform(0.9, 1.1, B), rng.uniform(400, 800, B), rng.uniform(400, 800, B), 1
    return K, pose


def test_boxes_from_poses_over_1000_poses():
    rng = np.random.default_rng(21)
    compared = skipped = 0
    for n in (1, 8, 100):
        for shared_K in (False, True):
            for shared_pts in (False, True):
                for homo in (False, True):
                    B = 42
                    K, pose = _random_poses(rng, B)
                    if shared_K:
                        K = np.broadcast_to(K[0], K.shape).copy()
                    pts = rng.uniform(-0.1, 0.1, (B, n, 3))
                    if shared_pts:
                        pts = np.broadcast_to(pts[0], pts.shape).copy()
                    P = np.concatenate([pose, np.broadcast_to([[[0, 0, 0, 1.0]]], (B, 1, 4))], axis=1) if homo else pose
                    args = (torch.from_numpy(K[0] if shared_K else K).to(DEV), torch.from_numpy(P).to(DEV),
                            torch.from_numpy(pts[0] if shared_pts else pts).to(DEV))
                    box, proj = crop._project(*args, True)
                    assert torch.equal(crop.boxes_from_poses(*args), box)
                    box, proj = box.cpu().numpy(), proj.cpu().numpy()
                    for b in range(B):
                        p = cr.reproj(K[b], pose[b], pts[b])
                        np.testing.assert_allclose(proj[b], p, rtol=1e-12, atol=0)
                        e = np.concatenate([p.min(axis=0), p.max(axis=0)])
                        if np.any(np.abs(e - np.rint(e)) < 1e-9):
                            skipped += 1
                            continue
                        compared += 1
                        assert np.array_equal(box[b], cr.box_from_pose(K[b], pose[b], pts[b])), (n, b)
    print(f"boxes_from_poses: {compared} boxes compared, {skipped} skipped with an extreme within 1e-9 of an integer")
    assert compared + skipped == 1008 and compared >= 1000


def test_boxes_from_poses_planted_cases():
    """A corner on the camera plane (p[2] = 0 exactly), corners behind the camera, and extremes just inside and just outside
    what int32 holds: K = I and pose = [I | 0] make the projection x / z exact."""
    eye = np.concatenate([np.eye(3), np.zeros((3, 1))], axis=1)
    cases = [([[1, 2, 0], [3, 4, 1]], [0, 0, 0, 0]),
             ([[1, 2, -2], [-3, 4, -0.5], [0.5, 0.5, -1]], None),
             ([[2147483647.5, 1, 1], [-5, -2147483648.75, 1]], [-5, -2147483648, 2147483647, 1]),
             ([[2147483648.0, 1, 1], [-5, 0, 1]], [0, 0, 0, 0]),
             ([[5, -2147483649.0, 1], [-5, 0, 1]], [0, 0, 0, 0]),
             ([[-2147483648.99, 7, 1], [3, 2147483647.99, 1]], [-2147483648, 7, 3, 2147483647])]
    n = max(len(c) for c, _ in cases)
    pts = np.stack([np.array(c + [c[-1]] * (n - len(c)), np.float64) for c, _ in cases])
    B = len(cases)
    box = crop.boxes_from_poses(torch.eye(3, dtype=torch.float64, device=DEV), torch.from_numpy(np.stack([eye] * B)).to(DEV),
                                torch.from_numpy(pts).to(DEV)).cpu().numpy()
    with np.errstate(divide="ignore", invalid="ignore"):
        for b, (_, want) in enumerate(cases):
            model = cr.box_from_pose(np.eye(3), eye, pts[b])
            assert np.array_equal(box[b], model), (b, box[b], model)
            if want is not None:
                assert box[b].tolist() == want, (b, box[b])
