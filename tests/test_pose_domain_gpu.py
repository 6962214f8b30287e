"""The pose solvers across the domain they accept: opb_ransac_pnp (P3P), opb_ransac_epnp, opb_ransac_epnp_cv (OpenCV's loop)
and opb_epnp, against the fp64 inlier rule, the numpy restatement of OpenCV's loop (tests/opencv_ransac_reference.py) and
cv2 fixtures (tests/golden/pnp_domain_cases.npz, made by tests/golden/make_pose_domain.py).

- Confidence mode: the fp32 threshold's rounding at the boundary, every tested threshold against the fixtures, budgets
  1, 2 and around the wave (and lowered onto it), confidences 0 .. 1, each against the restatement's scan over the kernel's
  own per-sample counts and OpenCV's sample sequence.
- P3P and EPnP-RANSAC: hypotheses 1 .. 65535 * 128; records past H are never written and records below H do not depend on
  H; mask and count follow the inlier rule under the reported pose; tiny and infinite thresholds.
- Every mode: frames of 0 .. 8 and 10^5 pairs in one ragged batch with empty frames, offsets[0] > 0 with the rows outside
  every frame untouched, NaN / inf rows that never count and change no other frame, more than 65535 frames, and a K with
  skew and a non-unit last row read as the clean K.
"""
import os

import numpy as np
import pytest
import torch

from onepose_b200 import _lib, synthetic
from tests import opencv_ransac_reference as O
from tests import pnp_reference as ref
from tests.golden_util import GOLDEN_DIR

pytestmark = pytest.mark.gpu

MAX_H = 65535 * 128
REC = 13
SENT = -12345.5                       # workspace sentinel: a record slot nobody wrote
MASK_SENT = -7                        # mask sentinel: a row outside every frame
MODES = ("p3p", "epnp", "cv")


def _dev(a, dtype):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=dtype)).cuda()


def _solve(mode, K, p2, p3, off, H=256, thr=5.0, conf=0.99, seed=0, ws_extra=0, wave=0, trace_cap=0):
    """One call of an entry point on host arrays: K [B,9], p2 [T,2], p3 [T,3], off [B+1] (offsets may start above 0 and end
    below T).  The mask holds T rows filled with MASK_SENT, the workspace ws_extra doubles past its size filled with SENT."""
    lib = _lib.load()
    B, T = len(off) - 1, len(p2)
    Kd, p2d, p3d, offd = _dev(K, np.float64), _dev(p2, np.float64), _dev(p3, np.float64), _dev(off, np.int32)
    pose = torch.full((B, 12), float("nan"), dtype=torch.float64, device="cuda")
    cnt = torch.full((B,), -3, dtype=torch.int32, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    out = {}
    if mode == "frames":
        _lib.check(lib.opb_epnp(Kd.data_ptr(), p2d.data_ptr(), p3d.data_ptr(), offd.data_ptr(), B, pose.data_ptr(), cnt.data_ptr(), st))
        torch.cuda.synchronize()
        return {"pose": pose.cpu().numpy().reshape(B, 3, 4), "status": cnt.cpu().numpy()}
    mask = torch.full((max(T, 1),), MASK_SENT, dtype=torch.int32, device="cuda")
    size = B * H * REC + (B * 16 if mode == "cv" else 0)
    ws = torch.full((size + ws_extra,), SENT, dtype=torch.float64, device="cuda")
    if mode == "cv":
        its = torch.full((B,), -3, dtype=torch.int32, device="cuda")
        tr = None
        if trace_cap:
            tr = {"samples": torch.full((B, trace_cap, 5), -2, dtype=torch.int32, device="cuda"),
                  "counts": torch.full((B, trace_cap), -2, dtype=torch.int32, device="cuda"),
                  "winner": torch.full((B,), -2, dtype=torch.int32, device="cuda")}
            assert lib.opb_debug_set_cv_trace(tr["samples"].data_ptr(), tr["counts"].data_ptr(), tr["winner"].data_ptr(), trace_cap) == 0
        assert lib.opb_debug_set_cv_wave(wave) == 0
        try:
            _lib.check(lib.opb_ransac_epnp_cv(Kd.data_ptr(), p2d.data_ptr(), p3d.data_ptr(), offd.data_ptr(), B, H, float(thr), float(conf),
                                              ws.data_ptr(), pose.data_ptr(), mask.data_ptr(), cnt.data_ptr(), its.data_ptr(), st))
            torch.cuda.synchronize()
        finally:
            lib.opb_debug_set_cv_wave(0)
            lib.opb_debug_set_cv_trace(None, None, None, 0)
        out["iterations"] = its.cpu().numpy()
        if tr is not None:
            out.update({k: v.cpu().numpy() for k, v in tr.items()})
    else:
        fn = lib.opb_ransac_pnp if mode == "p3p" else lib.opb_ransac_epnp
        _lib.check(fn(Kd.data_ptr(), p2d.data_ptr(), p3d.data_ptr(), offd.data_ptr(), B, H, float(thr), seed, ws.data_ptr(), pose.data_ptr(),
                      mask.data_ptr(), cnt.data_ptr(), st))
        torch.cuda.synchronize()
    out.update({"pose": pose.cpu().numpy().reshape(B, 3, 4), "mask": mask.cpu().numpy()[:T], "cnt": cnt.cpu().numpy(), "off": np.asarray(off)})
    if ws_extra or mode != "cv":
        out["ws"] = ws.cpu().numpy()
    del ws
    return out


def _pack(frames, lead=0, tail=0):
    """Frames (K [3,3], uv [n,2], P [n,3]) -> K [B,9], p2, p3, off with `lead` rows before the first frame and `tail` after
    the last (filled with finite junk a solver must not read)."""
    n = [len(f[1]) for f in frames]
    off = (lead + np.concatenate([[0], np.cumsum(n)])).astype(np.int32)
    T = int(off[-1]) + tail
    p2 = np.full((max(T, 1), 2), 1e3)
    p3 = np.full((max(T, 1), 3), 77.0)
    for b, f in enumerate(frames):
        p2[off[b]:off[b + 1]] = np.asarray(f[1], np.float64).reshape(-1, 2)
        p3[off[b]:off[b + 1]] = np.asarray(f[2], np.float64).reshape(-1, 3)
    K = np.stack([np.asarray(f[0], np.float64).reshape(9) for f in frames])
    return K, p2, p3, off


def _scene(seed, n, frac=0.4, noise=0.5):
    K, uv, P, gt = synthetic.make_pnp_scene(seed, n, outlier_frac=frac, noise_px=noise)
    return K, uv, P * 1000


def _frame(out, b, key="mask"):
    return out[key][out["off"][b]:out["off"][b + 1]]


def _is_identity(p):
    return np.array_equal(p, np.eye(4)[:3])


def _epnp_rule(pose, K, uv, P, thr):
    """opb_ransac_epnp's rule on fp32-rounded pairs: finite squared error <= thr^2 in fp64, no depth test; (inlier, border)."""
    P = P.astype(np.float32).astype(np.float64)
    uv = uv.astype(np.float32).astype(np.float64)
    X = P @ pose[:, :3].T + pose[:, 3]
    with np.errstate(all="ignore"):
        du = K[0, 0] * X[:, 0] / X[:, 2] + K[0, 2] - uv[:, 0]
        dv = K[1, 1] * X[:, 1] / X[:, 2] + K[1, 2] - uv[:, 1]
        e2 = du * du + dv * dv
    return (e2 <= thr * thr) & np.isfinite(e2), np.abs(e2 - thr * thr) <= ref.BORDER_PX2


# ---- confidence mode


@pytest.mark.parametrize("thr", [0.1, 0.7, 3.3, 5.3, 5.7])
def test_cv_threshold_boundary(thr):
    """The probe pair of the boundary scene (pinned to cv2 on the CPU) at one ulp below, at, and one ulp above each of the two
    candidate fp32 bounds: an inlier exactly when its fp32 error is <= fp32(fp32(thr)^2)."""
    t = O.fp32_threshold2(thr)
    t_late = np.float32(thr * thr)
    lo, hi = min(t, t_late), max(t, t_late)
    errs = [np.nextafter(lo, np.float32(0)), lo, hi, np.nextafter(hi, np.float32(np.inf))]
    frames = [O.boundary_scene(e) for e in errs]
    out = _solve("cv", *_pack(frames), H=1, thr=thr, trace_cap=1)
    for b, e in enumerate(errs):
        assert out["samples"][b, 0].tolist() == [9, 11, 4, 12, 7]
        m = _frame(out, b)
        assert m[1:].all() and m[0] == (e <= t), (thr, e, m[0])
        assert out["counts"][b, 0] == 12 + (e <= t) == out["cnt"][b] == m.sum(), (thr, e)
        assert out["iterations"][b] == 1 and out["winner"][b] == 0


def _fixture():
    g = dict(np.load(os.path.join(GOLDEN_DIR, "pnp_domain_cases.npz"), allow_pickle=False))
    return g, [str(t) for t in g["c_tags"]]


def test_cv_thresholds_against_cv2_fixtures():
    """Noise-free scenes with outliers at thresholds 0.05 .. inf: the samples, the counts of the samples OpenCV evaluated
    (every all-inlier sample is exact, so its count is OpenCV's), the winner, the iteration count and the mask equal the
    restatement's (and so cv2's); the pose equals cv2's to 1e-6 (ref.pose_error).  At thresholds 1e6 and inf the refit runs
    on every pair, 40 % gross outliers included, where two EPnPs need not agree: that pose must be finite."""
    g, tags = _fixture()
    for thr in sorted({float(g[f"c{i}_thr"]) for i in range(len(tags))}):
        idx = [i for i in range(len(tags)) if float(g[f"c{i}_thr"]) == thr]
        frames = [(g[f"c{i}_K"], g[f"c{i}_uv"], g[f"c{i}_P"]) for i in idx]
        out = _solve("cv", *_pack(frames), H=2000, thr=thr, conf=0.99, trace_cap=2000)
        for b, i in enumerate(idx):
            tag, n = tags[i], len(g[f"c{i}_uv"])
            it = int(g[f"c{i}_iterations"])
            assert out["iterations"][b] == it and out["winner"][b] == g[f"c{i}_winner"], tag
            assert out["samples"][b, :it].tolist() == g[f"c{i}_samples"].tolist(), tag
            counts, want = out["counts"][b, :it], g[f"c{i}_counts"]
            exact = want == max(want.max(), 0)
            assert np.array_equal(counts[exact], want[exact]), tag
            assert O.scan(out["counts"][b], n, 0.99, 2000) == (int(g[f"c{i}_winner"]), int(out["cnt"][b]), it), tag
            assert np.nonzero(_frame(out, b))[0].tolist() == g[f"c{i}_inliers"].tolist(), tag
            d = ref.pose_error(out["pose"][b][:, :3], out["pose"][b][:, 3], g[f"c{i}_cv"][:, :3], g[f"c{i}_cv"][:, 3])
            print(f"{tag}: pose vs cv2 {d:.2e}")
            assert d <= 1e-6 if thr < 1e3 else np.all(np.isfinite(out["pose"][b])), (tag, d)


def _scan_checks(out, frames, conf, H):
    for b, (_, uv, _) in enumerate(frames):
        n = len(uv)
        it = int(out["iterations"][b])
        if n <= 5:
            assert it == 0
            continue
        assert 1 <= it <= H
        assert out["samples"][b, :it].tolist() == [list(s) for s in O.subsets(n, it)], b
        assert np.all(out["counts"][b, :it] >= -1)
        w, best, it_r = O.scan(out["counts"][b], n, conf, H)
        assert (w, it_r) == (int(out["winner"][b]), it), (b, w, it_r, out["winner"][b], it)
        assert out["cnt"][b] == (best if w >= 0 else 0) == _frame(out, b).sum(), b


@pytest.mark.parametrize("wave", [128, 0])
def test_cv_budget_edges(wave):
    """Budgets 1, 2 and W - 1, W, W + 1 around the wave (128 set, or chosen from B: 128 .. 2048 here).  The loop exits at iter
    >= budget; results of the wave past the exit are discarded."""
    frames = [_scene(1800 + k, n, frac) for k, (n, frac) in enumerate(((40, 0.85), (100, 0.9), (300, 0.95), (7, 0.0)))]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    W = 128 if wave else (sms * 128 // len(frames) + 127) // 128 * 128
    for H in sorted({1, 2, W - 1, W, W + 1}):
        out = _solve("cv", *_pack(frames), H=H, conf=0.99, wave=wave, trace_cap=H)
        _scan_checks(out, frames, 0.99, H)
        assert out["iterations"][2] == H, H                          # 95 % outliers: no sample lowers the budget


@pytest.mark.parametrize("target", [128, 256])
def test_cv_budget_lowered_onto_a_wave_boundary(target):
    """A confidence chosen so that RANSACUpdateNumIters lowers the budget to exactly `target` (a multiple of the 128-sample
    wave) once an all-inlier sample wins: the loop ends at the wave's last sample."""
    K, uv, P, gt = synthetic.make_pnp_scene(1900, 100, outlier_frac=0.4, noise_px=0.0)
    P = P * 1000
    c = int(ref.classify(np.concatenate([gt[:, :3], gt[:, 3:] * 1000], 1), K, uv, P, 5.0)[0].sum())
    conf = 1 - (1 - (c / 100) ** 5) ** target
    assert O.update_num_iters(conf, (100 - c) / 100, 5, 10000) == target
    out = _solve("cv", *_pack([(K, uv, P)]), H=10000, conf=conf, wave=128, trace_cap=10000)
    _scan_checks(out, [(K, uv, P)], conf, 10000)
    assert out["iterations"][0] == target and out["cnt"][0] == c


@pytest.mark.parametrize("conf", [0.0, 1e-300, 0.5, 0.99, 1 - 2 ** -53, 1.0])
def test_cv_confidence_edges(conf):
    """0 and 1 follow RANSACUpdateNumIters' clamped formula (cv2 refuses both); the restatement's scan is the referee."""
    frames = [_scene(2000 + k, n, frac, 1.0) for k, (n, frac) in enumerate(((60, 0.3), (200, 0.7), (9, 0.0)))]
    out = _solve("cv", *_pack(frames), H=3000, conf=conf, trace_cap=3000)
    _scan_checks(out, frames, conf, 3000)
    if conf <= 1e-300:
        assert all(out["iterations"][b] == out["winner"][b] + 1 for b in range(3))


# ---- P3P and EPnP-RANSAC: the hypothesis records


@pytest.mark.parametrize("mode", ["p3p", "epnp"])
def test_hypothesis_counts(mode):
    """H = 1 .. 65535 * 128 on one frame: no record past H is written, record h < H is the same at every H, each record's count
    follows the inlier rule under its pose, and the mask and count follow it under the reported pose (P3P) or the winning
    record's pose (EPnP)."""
    K, uv, P = _scene(2100, 30, 0.3)
    frame = _pack([(K, uv, P)])
    need = (MAX_H + 1) * REC * 8
    free, _ = torch.cuda.mem_get_info()
    assert free > need + (1 << 30), f"{free} bytes free for a {need}-byte workspace"
    prev = None
    for H in (1, 2, 127, 128, 129, 4096, MAX_H):                     # increasing: each call's records extend the last's
        out = _solve(mode, *frame, H=H, ws_extra=REC, seed=5)
        ws = out["ws"]
        assert np.all(ws[H * REC:] == SENT), H
        rec = ws[:H * REC].reshape(H, REC)
        if prev is not None:
            assert rec[:len(prev)].tobytes() == prev.tobytes(), H
        prev = rec[:4096].copy()
        if H == 4096:
            for h in range(0, H, 97):
                c = rec[h, 0]
                if c > 0:
                    pose = np.concatenate([rec[h, 1:10].reshape(3, 3), rec[h, 10:13, None]], 1)
                    inl, border = ref.classify(pose, K, uv, P, 5.0) if mode == "p3p" else _epnp_rule(pose, K, uv, P, 5.0)
                    assert abs(inl.sum() - c) <= border.sum(), (h, c, inl.sum())
        counts = rec[:, 0]
        m = out["mask"]
        assert out["cnt"][0] == m.sum() and set(np.unique(m)) <= {0, 1}
        if counts.max() < 4:
            assert _is_identity(out["pose"][0]) and out["cnt"][0] == 0
            continue
        if mode == "p3p":
            inl, border = ref.classify(out["pose"][0], K, uv, P, 5.0)
        else:
            h = int(np.argmax(counts))
            assert out["cnt"][0] == counts[h]
            pose = np.concatenate([rec[h, 1:10].reshape(3, 3), rec[h, 10:13, None]], 1)
            inl, border = _epnp_rule(pose, K, uv, P, 5.0)
        assert np.all((m == inl) | border), H
        print(f"{mode} H={H}: {out['cnt'][0]} inliers")


@pytest.mark.parametrize("mode", MODES)
def test_threshold_extremes(mode):
    """A threshold no noisy pair meets: the identity and no inliers.  inf: every finite pair is an inlier (P3P: every one in
    front of the camera, which all are here; its refinement on 40 % gross outliers leaves the model, and the hypothesis is
    kept)."""
    frames = [_scene(2200 + k, n, 0.4, 1.0) for k, n in enumerate((50, 300))]
    tiny = _solve(mode, *_pack(frames), H=512, thr=1e-9)
    for b in range(2):
        assert _is_identity(tiny["pose"][b]) and tiny["cnt"][b] == 0 and not _frame(tiny, b).any(), b
    big = _solve(mode, *_pack(frames), H=512, thr=float("inf"))
    for b, f in enumerate(frames):
        assert big["cnt"][b] == len(f[1]) and _frame(big, b).all(), b
        assert np.all(np.isfinite(big["pose"][b]))


# ---- every mode: layout, frame sizes, non-finite pairs, K


def _layout_frames():
    """Frames of 0 .. 8 pairs, 10^4 and 10^5 pairs, and empty frames between them."""
    sizes = [0, 1, 2, 3, 4, 5, 6, 7, 8, 0, 10 ** 4, 0, 0, 10 ** 5, 8, 0]
    return [_scene(2300 + k, n, 0.3, 1.0) if n else (np.eye(3) * [600, 600, 1], np.zeros((0, 2)), np.zeros((0, 3)))
            for k, n in enumerate(sizes)]


def _same_frames(a, b, frames, skip=()):
    for f in range(len(frames)):
        if f in skip:
            continue
        assert a["pose"][f].tobytes() == b["pose"][f].tobytes(), f
        if "mask" in a:
            assert np.array_equal(_frame(a, f), _frame(b, f)) and a["cnt"][f] == b["cnt"][f], f
        if "iterations" in a:
            assert a["iterations"][f] == b["iterations"][f], f
        if "status" in a:
            assert a["status"][f] == b["status"][f], f


@pytest.mark.parametrize("mode", MODES + ("frames",))
def test_ragged_layout_and_leading_offset(mode):
    """One ragged batch, then the same frames behind 37 leading rows and before 11 trailing ones: every output is
    bit-identical, and no row outside the frames is written."""
    frames = _layout_frames()
    H = 512
    a = _solve(mode, *_pack(frames), H=H)
    K, p2, p3, off = _pack(frames, lead=37, tail=11)
    b = _solve(mode, K, p2, p3, off, H=H)
    _same_frames(a, b, frames)
    if mode != "frames":
        assert np.all(b["mask"][:37] == MASK_SENT) and np.all(b["mask"][off[-1]:] == MASK_SENT)
    for f, (_, uv, _) in enumerate(frames):
        n = len(uv)
        if mode == "frames":
            assert a["status"][f] == (n >= 4), f
            continue
        m = _frame(a, f)
        assert set(np.unique(m)) <= {0, 1} and a["cnt"][f] == m.sum(), f
        if n < 4:
            assert _is_identity(a["pose"][f]) and a["cnt"][f] == 0, f
        elif mode == "cv" and n <= 5:
            assert m.all(), f
        elif n >= 10 ** 4:
            assert a["cnt"][f] > 0.6 * n, (f, a["cnt"][f])


def test_ragged_batch_of_a_million_pairs():
    """~2^20 pairs in 64 frames of every size from 0 to 32768, P3P and EPnP-RANSAC: the count is the mask's sum and the mask
    follows the rule under the reported pose."""
    rs = np.random.RandomState(7)
    sizes = [int(s) for s in rs.randint(0, 32769, 64)]
    sizes[:4] = [0, 4, 5, 32768]
    frames = [_scene(2400 + k, n, 0.5, 1.0) for k, n in enumerate(sizes)]
    print("pairs:", sum(sizes))
    for mode in ("p3p", "epnp"):
        out = _solve(mode, *_pack(frames), H=256)
        for f, (K, uv, P) in enumerate(frames):
            m = _frame(out, f)
            assert out["cnt"][f] == m.sum(), (mode, f)
            if mode == "p3p" and out["cnt"][f] > 0:
                inl, border = ref.classify(out["pose"][f], K, uv, P, 5.0)
                assert np.all((m == inl) | border), (mode, f)


@pytest.mark.parametrize("mode", MODES + ("frames",))
def test_non_finite_pairs(mode):
    """NaN and +-inf in pts2d / pts3d, planted in frames 1 and 3 (frame 5 is all NaN): those rows are never inliers, the count is
    the mask's sum, the pose is finite or the identity, and every other frame is bit-identical to the call without them.
    Checked at threshold 5 and at inf."""
    frames = [_scene(2500 + k, n, 0.3, 1.0) for k, n in enumerate((60, 80, 7, 120, 200, 9))]
    bad_vals = (np.nan, np.inf, -np.inf)
    planted = []
    rows = {}
    for f, (K, uv, P) in enumerate(frames):
        if f in (1, 3):
            uv, P = uv.copy(), P.copy()
            r = np.arange(2, len(uv), 5)
            for k, i in enumerate(r):
                (uv if k % 2 else P)[i, k % (2 if k % 2 else 3)] = bad_vals[k % 3]
            rows[f] = r
        elif f == 5:
            uv, P = np.full_like(uv, np.nan), P
            rows[f] = np.arange(len(uv))
        planted.append((K, uv, P))
    for thr in (5.0, float("inf")):
        clean = _solve(mode, *_pack(frames), H=1024, thr=thr)
        dirty = _solve(mode, *_pack(planted), H=1024, thr=thr)
        _same_frames(clean, dirty, frames, skip=rows)
        for f, r in rows.items():
            p = dirty["pose"][f]
            if mode == "frames":
                assert dirty["status"][f] == 0 and _is_identity(p), f
                continue
            m = _frame(dirty, f)
            assert not m[r].any() and dirty["cnt"][f] == m.sum(), (thr, f)
            assert np.all(np.isfinite(p)) and (dirty["cnt"][f] > 0 or _is_identity(p)), (thr, f)
        if mode != "frames":
            assert _is_identity(dirty["pose"][5]) and dirty["cnt"][5] == 0


@pytest.mark.parametrize("mode", ["cv", "epnp", "frames"])
def test_more_than_65535_frames(mode):
    """70000 frames (grid x is the frame): a repeating set of 7 frames gives the same result wherever it sits in the batch."""
    base = [_scene(2600 + k, n, 0.3, 1.0) for k, n in enumerate((3, 4, 5, 6, 12, 20, 9))]
    B = 70000
    frames = [base[b % 7] for b in range(B)]
    out = _solve(mode, *_pack(frames), H=8)
    if mode == "epnp":                                                   # the sample stream depends on the frame's index
        for b in (0, 65534, 65535, 65536, B - 1):
            n = len(frames[b][1])
            assert out["cnt"][b] == _frame(out, b).sum(), b
            assert (n >= 4 and out["cnt"][b] >= 4) or _is_identity(out["pose"][b]), b
        return
    keys = ["pose"] + (["status"] if mode == "frames" else ["cnt", "iterations"])
    for b in list(range(65530, 65545)) + [B - 1]:
        r = b % 7
        for k in keys:
            assert out[k][b].tobytes() == out[k][r].tobytes(), (k, b)
        if mode == "cv":
            assert np.array_equal(_frame(out, b), _frame(out, r)), b


@pytest.mark.parametrize("mode", MODES + ("frames",))
def test_k_skew_and_last_row_are_ignored(mode):
    """Only fx, fy, cx, cy are read: a K with skew and a last row (0.3, -0.2, 7) gives bit-identical results."""
    frames = [_scene(2700 + k, n, 0.3, 1.0) for k, n in enumerate((4, 6, 50, 400))]
    K, p2, p3, off = _pack(frames)
    K2 = K.copy()
    K2[:, 1] = 3.5
    K2[:, 3] = -0.7
    K2[:, 6:] = [0.3, -0.2, 7.0]
    _same_frames(_solve(mode, K, p2, p3, off), _solve(mode, K2, p2, p3, off), frames)
