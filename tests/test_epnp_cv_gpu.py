"""EPnP-RANSAC with OpenCV's loop on the GPU (opb_ransac_epnp_cv, ``method="epnp", confidence=c``) against
cv2.solvePnPRansac(EPNP) fixtures and the numpy restatement of OpenCV's loop (tests/opencv_ransac_reference.py,
tests/golden/pnp_epnp_cv_cases.npz made by tests/golden/make_epnp_cv.py).

- Sample sequence: the device's generator equals cv::RNG + getSubset, index for index, and so do the samples the loop
  evaluates across wave boundaries.
- Stopping rule: the restatement's scan over the kernel's own per-sample counts gives the kernel's winner and iteration
  count on every frame (this separates the schedule from EPnP's numerics).
- Noise-free scenes with outliers: every all-inlier sample gives the exact pose, so the counts, the iteration count and the
  inlier set equal OpenCV's, and the pose equals cv2's to 1e-6 (the inputs are rounded to fp32).
- Noisy scenes: a minimal EPnP on five noisy pairs depends on the null-space basis the eigen-solver picks (DESIGN 5.4), so a
  sample's count can differ from OpenCV's; the pose is held to 0.1 degree / 0.25 cm of cv2's and the agreement is printed.
"""
import os

import numpy as np
import pytest
import torch

from onepose_b200 import _lib, pnp
from tests import opencv_ransac_reference as O
from tests import pnp_reference as ref
from tests.golden_util import GOLDEN_DIR

pytestmark = pytest.mark.gpu

THR = 5.0
# the refit on the same inlier set: both EPnPs see the points rounded to fp32, which puts ~1e-7 relative noise on a
# noise-free scene, and on noisy points two valid EPnPs differ by the noise's effect (DESIGN 5.4, axis signs): 2e-8 to 4e-8
# measured
POSE_BAR = 1e-6


def _fixture():
    g = dict(np.load(os.path.join(GOLDEN_DIR, "pnp_epnp_cv_cases.npz"), allow_pickle=False))
    return g, [str(t) for t in g["c_tags"]]


def _case(g, i):
    return {k: g[f"c{i}_{k}"] for k in ("K", "uv", "P", "gt", "conf", "iters", "ok", "cv", "inliers", "iterations", "winner", "counts",
                                        "samples")}


def _pack(frames):
    off = np.concatenate([[0], np.cumsum([len(f[1]) for f in frames])]).astype(np.int32)
    total = int(off[-1])
    K = torch.from_numpy(np.stack([np.asarray(f[0], np.float64).reshape(9) for f in frames])).cuda()
    p2 = np.zeros((max(total, 1), 2))
    p3 = np.zeros((max(total, 1), 3))
    if total:
        p2[:total] = np.concatenate([np.asarray(f[1], np.float64).reshape(-1, 2) for f in frames])
        p3[:total] = np.concatenate([np.asarray(f[2], np.float64).reshape(-1, 3) for f in frames])
    return K, torch.from_numpy(p2).cuda(), torch.from_numpy(p3).cuda(), torch.from_numpy(off).cuda(), off


def _run(frames, conf, H=10000, wave=0, trace_cap=0, winner=False):
    """One opb_ransac_epnp_cv call (every frame at the same confidence).  With trace_cap, also the samples, counts and winner
    the device recorded (unevaluated samples keep -2); with winner only the winner."""
    lib = _lib.load()
    B = len(frames)
    K, p2, p3, offs, off = _pack(frames)
    total = int(off[-1])
    ws = torch.full((B * (H * 13 + 16),), float("nan"), dtype=torch.float64, device="cuda")
    pose = torch.full((B, 12), float("nan"), dtype=torch.float64, device="cuda")
    mask = torch.full((max(total, 1),), -1, dtype=torch.int32, device="cuda")
    cnt = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    its = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    tr = None
    if trace_cap:
        tr = {"samples": torch.full((B, trace_cap, 5), -2, dtype=torch.int32, device="cuda"),
              "counts": torch.full((B, trace_cap), -2, dtype=torch.int32, device="cuda"),
              "winner": torch.full((B,), -2, dtype=torch.int32, device="cuda")}
        assert lib.opb_debug_set_cv_trace(tr["samples"].data_ptr(), tr["counts"].data_ptr(), tr["winner"].data_ptr(), trace_cap) == 0
    elif winner:
        tr = {"winner": torch.full((B,), -2, dtype=torch.int32, device="cuda")}
        assert lib.opb_debug_set_cv_trace(None, None, tr["winner"].data_ptr(), 0) == 0
    assert lib.opb_debug_set_cv_wave(wave) == 0
    try:
        _lib.check(lib.opb_ransac_epnp_cv(K.data_ptr(), p2.data_ptr(), p3.data_ptr(), offs.data_ptr(), B, H, THR, float(conf), ws.data_ptr(),
                                          pose.data_ptr(), mask.data_ptr(), cnt.data_ptr(), its.data_ptr(), torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
    finally:
        lib.opb_debug_set_cv_wave(0)
        lib.opb_debug_set_cv_trace(None, None, None, 0)
    out = {"pose": pose.cpu().numpy().reshape(B, 3, 4), "mask": mask[:total].cpu().numpy(), "cnt": cnt.cpu().numpy(),
           "iterations": its.cpu().numpy(), "off": off}
    if tr is not None:
        out.update({k: v.cpu().numpy() for k, v in tr.items()})
    return out


def _frame_mask(out, b):
    return out["mask"][out["off"][b]:out["off"][b + 1]]


def _perr(a, b):
    return ref.pose_error(a[:, :3], a[:, 3], b[:, :3], b[:, 3])


def _cm_deg_mm(a, b):
    """(degrees, cm) between poses whose translations are in millimetres."""
    from oracle import pnp_oracle
    s = np.array([1, 1, 1, 1e-3])
    return pnp_oracle.pose_error(a * s, b * s)


@pytest.mark.parametrize("n", [5, 6, 7, 100, 1000, 65536])
def test_device_generator_draws_opencvs_samples(n):
    lib = _lib.load()
    count = 10000
    expect = [list(s) for s in O.subsets(n, count)]
    for chunk in (count, 37, 1):                       # the warp's jump-ahead, carried across calls as across waves
        out = torch.full((count, 5), -1, dtype=torch.int32, device="cuda")
        _lib.check(lib.opb_debug_cv_subsets(n, count, chunk, out.data_ptr(), torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        assert out.cpu().numpy().tolist() == expect, chunk


def test_loop_samples_across_wave_boundaries():
    """confidence 1 at 85 % outliers keeps the full budget of 1000: the samples the loop evaluated, wave after wave of 64 (and
    of 1000), are OpenCV's first 1000 for the frame's n."""
    from onepose_b200 import synthetic
    frames = [synthetic.make_pnp_scene(41 + i, n, outlier_frac=0.85)[:3] for i, n in enumerate((7, 100, 1000))]
    for wave in (64, 1000):
        out = _run(frames, 1.0, H=1000, wave=wave, trace_cap=1000)
        for b, (_, uv, _) in enumerate(frames):
            it = int(out["iterations"][b])
            drawn = int((out["samples"][b, :, 0] != -2).sum())   # the loop's samples, and the rest of their wave
            assert 0 < it <= drawn
            assert out["samples"][b, :drawn].tolist() == [list(s) for s in O.subsets(len(uv), drawn)], (wave, b)


def _all_frames(g, tags):
    return [(g[f"c{i}_K"], g[f"c{i}_uv"], g[f"c{i}_P"]) for i in range(len(tags))]


def test_stopping_rule_on_the_kernels_own_counts():
    g, tags = _fixture()
    frames = _all_frames(g, tags)
    conf = 0.99
    for wave in (0, 64, 50):                           # 50: a wave that ends inside a warp's 32 counts
        out = _run(frames, conf, wave=wave, trace_cap=10000)
        for b, tag in enumerate(tags):
            n = len(frames[b][1])
            if n <= 5:
                assert out["iterations"][b] == 0, tag
                continue
            it = int(out["iterations"][b])
            counts = out["counts"][b]
            assert np.all(counts[:it] >= -1), tag         # samples of the last wave past the exit are evaluated, then discarded
            w, best, it_r = O.scan(counts, n, conf, 10000)
            assert (w, it_r) == (int(out["winner"][b]), it), (tag, w, it_r, out["winner"][b], it)
            assert out["cnt"][b] == (best if w >= 0 else 0) == _frame_mask(out, b).sum(), tag


def _contaminated(c):
    """cv2's inlier set holds an outlier that projects within the threshold (more than 1e-3 px off under the true pose)."""
    gt, P, uv, K = c["gt"], c["P"][c["inliers"]], c["uv"][c["inliers"]], c["K"]
    X = P @ gt[:, :3].T + gt[:, 3]
    e = np.abs(X[:, :2] / X[:, 2:] * [K[0, 0], K[1, 1]] + K[:2, 2] - uv).max(1)
    return bool((e > 1e-3).any())


def _check_fixture_case(tag, c, out, b, report):
    n = len(c["uv"])
    mask = _frame_mask(out, b)
    inl = np.nonzero(mask)[0]
    same_set = inl.tolist() == c["inliers"].tolist()
    same_iterations = int(out["iterations"][b]) == int(c["iterations"])
    same_winner = int(out["winner"][b]) == int(c["winner"]) if n > 5 else True   # 4 or 5 pairs: no loop, no winner index
    report.append((tag, same_set, same_iterations, same_winner))
    if n < 4:
        assert np.array_equal(out["pose"][b], np.eye(4)[:3]) and out["cnt"][b] == 0 and not c["ok"], tag
        return
    if n <= 5:
        assert mask.all() and out["cnt"][b] == n and same_set and out["iterations"][b] == 0, tag
        d = _perr(out["pose"][b], c["cv"])
        deg, cm = _cm_deg_mm(out["pose"][b], c["cv"])
        print(f"{tag}: pose vs cv2 {d:.2e} ({deg:.4f} deg, {cm:.4f} cm)")
        if n == 4:
            # solvePnP(P3P) on the four pairs, no refit: P3P on 0-2, the solution that best reprojects 3, on the same fp32 points
            assert d <= POSE_BAR, (tag, d)
        else:
            # EPnP on five pairs: M^T M has an exact two-dimensional null space whose basis the eigen-solver picks, and on
            # noisy pairs the answer depends on it (DESIGN 5.4); the distance is printed, the pose must be finite
            assert np.all(np.isfinite(out["pose"][b])), tag
        return
    assert bool(c["ok"]) == (out["cnt"][b] > 0), tag
    if not c["ok"]:
        assert np.array_equal(out["pose"][b], np.eye(4)[:3]) and int(out["iterations"][b]) == int(c["iterations"]), tag
        return
    if tag.startswith("clean"):
        assert same_set, (tag, len(inl), len(c["inliers"]))
        assert int(out["iterations"][b]) == int(c["iterations"]), (tag, out["iterations"][b], c["iterations"])
        if _contaminated(c):                           # an outlier inside the threshold: the refit's points are not exact
            deg, cm = _cm_deg_mm(out["pose"][b], c["cv"])
            assert deg < 0.1 and cm < 0.25, (tag, deg, cm)
        else:
            assert _perr(out["pose"][b], c["cv"]) <= POSE_BAR, (tag, _perr(out["pose"][b], c["cv"]))
    else:
        deg, cm = _cm_deg_mm(out["pose"][b], c["cv"])
        assert deg < 0.1 and cm < 0.25, (tag, deg, cm)


def test_against_cv2_fixtures():
    g, tags = _fixture()
    frames = _all_frames(g, tags)
    groups = sorted({(float(g[f"c{i}_conf"]), int(g[f"c{i}_iters"])) for i in range(len(tags))})
    report = []
    for conf, iters in groups:                         # one call per (confidence, iterationsCount), its frames in one batch
        idx = [i for i in range(len(tags)) if (float(g[f"c{i}_conf"]), int(g[f"c{i}_iters"])) == (conf, iters)]
        out = _run([frames[i] for i in idx], conf, H=iters, winner=True)
        for b, i in enumerate(idx):
            _check_fixture_case(tags[i], _case(g, i), out, b, report)
    for tag, same_set, same_it, same_w in report:
        print(f"{tag}: inlier set {'=' if same_set else '!='} cv2's, iterations {'=' if same_it else '!='} OpenCV's, "
              f"winner index {'=' if same_w else '!='} OpenCV's")
    noisy = [r for r in report if not r[0].startswith("clean")]
    print(f"frames other than noise-free: inlier set equal on {sum(r[1] for r in noisy)} of {len(noisy)}, "
          f"iteration count on {sum(r[2] for r in noisy)}, winner index on {sum(r[3] for r in noisy)}")
    clean = [r for r in report if r[0].startswith("clean")]
    assert all(r[3] for r in clean), [r[0] for r in clean if not r[3]]


def test_four_noise_free_pairs_give_the_exact_pose():
    """4 pairs: OpenCV returns solvePnP(P3P) on them, with no refit; noise-free pairs give the true pose (to the fp32
    rounding of the inputs), as the same frames of 5 and 6 pairs do."""
    from onepose_b200 import synthetic
    frames, gts = [], []
    for seed, n in ((905, 4), (906, 4), (907, 5), (908, 6)):
        K, uv, P, gt = synthetic.make_pnp_scene(seed, n, outlier_frac=0.0, noise_px=0.0)
        frames.append((K, uv, P * 1000))
        gts.append(np.concatenate([gt[:, :3], gt[:, 3:] * 1000], 1))
    out = _run(frames, 0.99)
    for b, gt in enumerate(gts):
        d = _perr(out["pose"][b], gt)
        print(f"{len(frames[b][1])} noise-free pairs: pose vs ground truth {d:.2e}")
        assert d <= 1e-5 and out["cnt"][b] == len(frames[b][1]), (b, d)


def test_reference_call_through_ransac_PnP():
    """ransac_PnP(..., method="epnp", confidence=0.99) is the reference's call: pose and inliers as cv2's on the fixture's
    noise-free scenes (points in metres, scale 1000 as the reference passes them)."""
    g, tags = _fixture()
    for i, tag in enumerate(tags):
        c = _case(g, i)
        if not tag.startswith("clean") or float(g[f"c{i}_conf"]) != 0.99 or _contaminated(c):
            continue
        pose, _, inliers = pnp.ransac_PnP(c["K"], c["uv"], c["P"] / 1000, scale=1000, method="epnp", confidence=0.99)
        assert inliers.reshape(-1).tolist() == c["inliers"].tolist(), tag
        cv = c["cv"].copy()
        cv[:, 3] /= 1000
        assert _perr(pose, cv) <= POSE_BAR, tag


def test_batches_equal_single_frames_and_do_not_depend_on_the_wave():
    from onepose_b200 import synthetic
    g, tags = _fixture()
    frames = _all_frames(g, tags)                      # 31 frames: mixed inlier ratios, 3, 4, 5 and 6 pairs
    frames.append(synthetic.make_pnp_scene(77, 400, outlier_frac=0.8, noise_px=1.0)[:3])
    singles = [_run([f], 0.99) for f in frames]
    for B in (1, 8, 32):
        sub = frames[:B] if B < 32 else frames
        outs = [_run(sub, 0.99), _run(sub, 0.99, wave=64)]
        for out in outs:
            for b in range(len(sub)):
                s = singles[b]
                assert out["pose"][b].tobytes() == s["pose"][0].tobytes(), (B, b)
                assert np.array_equal(_frame_mask(out, b), s["mask"]), (B, b)
                assert out["cnt"][b] == s["cnt"][0] and out["iterations"][b] == s["iterations"][0], (B, b)
    its = [int(s["iterations"][0]) for s in singles]
    print("iterations per frame:", its)
    assert len(set(its)) > 5                           # frames stop at different waves


def test_two_calls_are_identical_and_do_not_block():
    from onepose_b200 import synthetic
    B, n = 8, 300
    scenes = [synthetic.make_pnp_scene(500 + b, n, outlier_frac=0.2 + 0.08 * b) for b in range(B)]
    K = torch.from_numpy(np.stack([s[0] for s in scenes])).cuda()
    p2 = torch.from_numpy(np.concatenate([s[1] for s in scenes])).cuda()
    p3 = torch.from_numpy(np.concatenate([s[2] for s in scenes]) * 1000).cuda()
    off = torch.arange(0, B * n + 1, n, dtype=torch.int32).cuda()
    its = torch.empty(B, dtype=torch.int32, device="cuda")
    a = pnp.ransac_pnp_batch(K, p2, p3, off, method="epnp", confidence=0.99, iterations_out=its)
    its_a = its.clone()
    torch.cuda.synchronize()
    start = torch.cuda.Event()
    torch.cuda._sleep(1 << 30)                         # ~0.5 s of device time ahead of the call
    start.record()
    b = pnp.ransac_pnp_batch(K, p2, p3, off, method="epnp", confidence=0.99, iterations_out=its)
    queued = not start.query()                         # the call returned while the device was still busy before it
    after = torch.ones(1, device="cuda") * 2
    torch.cuda.synchronize()
    assert queued
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    assert torch.equal(its, its_a) and float(after) == 2.0
    print("iterations:", its.tolist())


def test_python_options():
    from onepose_b200 import synthetic
    K, uv, P, _ = synthetic.make_pnp_scene(12, 200, outlier_frac=0.4)
    Kt = torch.from_numpy(K)[None].cuda()
    p2, p3 = torch.from_numpy(uv).cuda(), torch.from_numpy(P * 1000).cuda()
    off = torch.tensor([0, 200], dtype=torch.int32).cuda()
    with pytest.raises(ValueError):
        pnp.ransac_pnp_batch(Kt, p2, p3, off, confidence=0.99)                     # p3p
    with pytest.raises(ValueError):
        pnp.ransac_pnp_batch(Kt, p2, p3, off, method="epnp", iterations_out=torch.empty(1, dtype=torch.int32, device="cuda"))
    fixed = pnp.ransac_pnp_batch(Kt, p2, p3, off, method="epnp")
    again = pnp.ransac_pnp_batch(Kt, p2, p3, off, method="epnp", confidence=None)
    for x, y in zip(fixed, again):
        assert torch.equal(x, y)
    its = torch.empty(1, dtype=torch.int32, device="cuda")
    cv = pnp.ransac_pnp_batch(Kt, p2, p3, off, method="epnp", confidence=0.99, iterations_out=its)
    assert 0 < int(its[0]) < 10000 and int(cv[2][0]) > 100
    # the ends of the range follow RANSACUpdateNumIters' clamped formula: 0 stops after the first improvement; 1 lowers the
    # budget only as far as log(DBL_MIN) / log(1 - (1 - outlier ratio)^5) (about 8700 here)
    for c in (0.0, 1.0):
        out = _run([(K, uv, P * 1000)], c, trace_cap=10000)
        w, _, it = O.scan(out["counts"][0], 200, c, 10000)
        assert (w, it) == (out["winner"][0], out["iterations"][0]), c
        if c == 0.0:
            assert it == w + 1 == int(np.nonzero(out["counts"][0] > 4)[0][0]) + 1
        else:
            assert it > 5000
