"""Detection by 2D-2D matching on the GPU (onepose_b200.detect / csrc/detect.cu): the estimator stage by stage against the numpy
restatement of cv2.estimateAffinePartial2D (tests/affine_ransac_reference.py), and boxes and crops against the reference
detector's own results (tests/golden/pnp_detect_cases.npz, made by tests/golden/make_detect.py with OpenCV 4.13)."""
import os

import numpy as np
import pytest
import torch

from onepose_b200 import _lib, crop, detect, pnp
from tests import affine_ransac_reference as A
from tests import crop_reference as cr
from tests.golden_util import GOLDEN_DIR

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
REFINE_RTOL = 1e-10          # the bar the restatement meets against cv2 (tests/test_affine_ransac_reference_cpu.py)
TRACE_CAP = 2000

try:
    import cv2  # noqa: F401
    MINIMAL = "cv2"          # each minimal model from OpenCV itself
except ImportError:
    MINIMAL = "closed"       # the closed form, equal to cv2's bit for bit (checked on the CPU)


def planted(seed, n, frac, noise=1.0):
    r = np.random.default_rng(seed)
    f = r.uniform([0, 0], [640, 480], (n, 2))
    a, s = r.uniform(-3, 3), r.uniform(0.3, 3)
    R = s * np.array([[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]])
    t = f @ R.T + r.uniform(-300, 300, 2) + r.normal(0, noise, (n, 2))
    out = r.random(n) < frac
    t[out] = r.uniform(0, 1500, (int(out.sum()), 2))
    return f.astype(np.float32), t.astype(np.float32)


def _batch(problems, **kw):
    offs = np.cumsum([0] + [len(f) for f, _ in problems]).astype(np.int32)
    f = torch.from_numpy(np.concatenate([p[0] for p in problems]).reshape(-1, 2)).to(DEV)
    t = torch.from_numpy(np.concatenate([p[1] for p in problems]).reshape(-1, 2)).to(DEV)
    return detect.affine_partial_batch(f, t, torch.from_numpy(offs).to(DEV), **kw), offs


class Trace:
    def __init__(self, B):
        self.samples = torch.full((B, TRACE_CAP, 2), -7, dtype=torch.int32, device=DEV)
        self.counts = torch.full((B, TRACE_CAP), -7, dtype=torch.int32, device=DEV)
        self.models = torch.full((B, TRACE_CAP, 6), float("nan"), dtype=torch.float64, device=DEV)

    def __enter__(self):
        _lib.check(_lib.load().opb_debug_set_affine_trace(self.samples.data_ptr(), self.counts.data_ptr(), self.models.data_ptr(), TRACE_CAP))
        return self

    def __exit__(self, *a):
        torch.cuda.synchronize()
        _lib.check(_lib.load().opb_debug_set_affine_trace(None, None, None, 0))


SCENES = [(900 + k, n, frac, thr, conf) for k, (n, frac, thr, conf) in enumerate(
    [(2, 0.0, 3, 0.99), (3, 0.0, 3, 0.99), (6, 0.3, 6, 0.99), (50, 0.3, 3, 0.9), (50, 0.9, 6, 0.99), (300, 0.5, 6, 0.999),
     (1000, 0.25, 6, 0.99), (1000, 0.9, 6, 0.99), (4096, 0.5, 3, 0.99), (4096, 0.9, 6, 0.9), (777, 0.7, 3, 0.99)])]


@pytest.mark.parametrize("refine", [0, 10])
def test_estimator_stage_by_stage_against_the_restatement(refine):
    """Per problem: the samples, per-sample counts and minimal models (bit-equal to cv2's 2-point runKernel), the iteration
    count, the mask; the affine bit-equal without refinement and within REFINE_RTOL of the restatement's LM with it.  Problems
    with different thresholds run in one call per threshold and confidence."""
    worst = 0.0
    for thr in (3, 6):
        for conf in (0.9, 0.99, 0.999):
            sc = [s for s in SCENES if s[3] == thr and s[4] == conf]
            if not sc:
                continue
            probs = [planted(seed, n, frac) for seed, n, frac, _, _ in sc]
            with Trace(len(probs)) as tr:
                out, offs = _batch(probs, threshold=thr, confidence=conf, refine_iters=refine)
            for b, (f, t) in enumerate(probs):
                H, m, info = A.estimate_affine_partial_2d(f, t, thr, 2000, conf, refine, minimal=MINIMAL)
                n, it = len(f), info["iterations"]
                assert int(out["iterations"][b]) == it and int(out["status"][b]) == (H is not None)
                assert np.array_equal(out["inliers"][offs[b]:offs[b + 1]].cpu().numpy(), m), (n, thr)
                k = min(it, TRACE_CAP)
                if n > 2:
                    assert tr.samples[b, :k].cpu().numpy().tolist() == [list(s) for s in info["samples"][:k]]
                    assert tr.counts[b, :k].cpu().tolist() == info["counts"][:k]
                    got = tr.models[b, :k].cpu().numpy().reshape(k, 2, 3)
                    assert got.tobytes() == np.stack(info["models"][:k]).tobytes()
                    assert A.scan(tr.counts[b, :k].cpu().numpy(), n, conf, 2000)[0] == info["winner"] or it > TRACE_CAP
                Hg = out["affine"][b].cpu().numpy()
                if H is None:
                    assert not Hg.any()
                elif refine == 0 or n == 2:
                    assert Hg.tobytes() == H.tobytes(), (n, Hg, H)
                else:
                    rel = float(np.abs(Hg - H).max() / np.abs(H).max())
                    worst = max(worst, rel)
                    assert rel <= REFINE_RTOL, (n, rel)
                print(f"n={n} thr={thr} conf={conf} refine={refine}: {it} iterations, winner {info['winner']}")
    print(f"refined affine, max relative difference from the restatement: {worst:.2e}")


def test_numpy_drop_in_and_degenerate_inputs():
    r = np.random.default_rng(3)
    f = r.uniform(0, 100, (40, 2))
    t = f * 1.5 + 7
    same = np.tile(f[:1], (40, 1))
    H, m = detect.estimate_affine_partial_2d(same, np.tile(t[:1], (40, 1)))                 # all identical: None, zero mask
    assert H is None and m.shape == (40, 1) and m.dtype == np.uint8 and not m.any()
    H, m = detect.estimate_affine_partial_2d(same, t)
    assert H is None and not m.any()
    H, m = detect.estimate_affine_partial_2d(f[:2], t[:2])                                  # 2 pairs: the model, both inliers
    assert m.ravel().tolist() == [1, 1] and H.tobytes() == A.run_kernel(f[:2].astype(np.float32), t[:2].astype(np.float32)).tobytes()
    H, m = detect.estimate_affine_partial_2d(same[:2], t[:2])                               # ... even a non-finite one, as cv2
    assert m.ravel().tolist() == [1, 1] and not np.isfinite(H).all()
    H, m = detect.estimate_affine_partial_2d(f[:1], t[:1])
    assert H is None and m.ravel().tolist() == [0]
    fp, tp = planted(5, 300, 0.4)
    H, m = detect.estimate_affine_partial_2d(fp.astype(np.float64), tp.astype(np.float64), ransacReprojThreshold=6)
    Hr, mr, _ = A.estimate_affine_partial_2d(fp, tp, 6.0, minimal=MINIMAL)
    assert np.array_equal(m.ravel(), mr) and np.abs(H - Hr).max() <= REFINE_RTOL * np.abs(Hr).max()
    for bad in (dict(confidence=1.0), dict(confidence=0.0), dict(maxIters=-1), dict(refineIters=-2), dict(ransacReprojThreshold=np.inf),
                dict(maxIters=2**31), dict(maxIters=2**32 + 5), dict(refineIters=2**31), dict(refineIters=2**32 + 1)):
        with pytest.raises(ValueError):
            detect.estimate_affine_partial_2d(fp, tp, **bad)
    with pytest.raises(ValueError):
        detect.estimate_affine_partial_2d(fp, tp[:5])


# ---- boxes and crops against the reference detector ----

@pytest.fixture(scope="module")
def golden():
    g = dict(np.load(os.path.join(GOLDEN_DIR, "pnp_detect_cases.npz"), allow_pickle=False))
    scenes = []
    for s in range(int(g["n_scenes"])):
        H, W, seed = (int(v) for v in g[f"s{s}_frame"])
        qs = [{k: g[f"s{s}_q{q}_{k}"] for k in ("keypoints", "matches0", "bbox", "view", "n_matches", "affine", "crop_size", "image_crop", "K_crop")}
              for q in range(int(g[f"s{s}_n_queries"]))]
        scenes.append({"frame": torch.from_numpy(cr.synthetic_frame(H, W, seed)).to(DEV), "hw": (H, W), "K": g[f"s{s}_K"], "queries": qs,
                       "ref": {"keypoints": torch.from_numpy(g[f"s{s}_ref_keypoints"]).to(DEV), "counts": torch.from_numpy(g[f"s{s}_ref_counts"]).to(DEV),
                               "sizes": torch.from_numpy(g[f"s{s}_ref_sizes"]).to(DEV)}})
    return scenes


def _query(qs, dtype=torch.int64):
    cap = max(max(len(q["keypoints"]) for q in qs), 1)
    kp = np.zeros((len(qs), cap, 2), np.float32)
    for b, q in enumerate(qs):
        kp[b, :len(q["keypoints"])] = q["keypoints"]
    query = {"keypoints": torch.from_numpy(kp).to(DEV), "counts": torch.tensor([len(q["keypoints"]) for q in qs], dtype=torch.int32, device=DEV)}
    m0 = torch.from_numpy(np.stack([q["matches0"] for q in qs])).to(DEV, dtype)
    return query, m0


def _near_integer_corner(affine, size_hw):
    h, w = (float(v) for v in size_hw)
    p = np.asarray(affine) @ np.array([[0, 0, 1], [w, 0, 1], [0, h, 1], [w, h, 1]], np.float64).T
    return bool(np.any(np.abs(p - np.rint(p)) < 1e-9))


def test_boxes_equal_the_reference(golden):
    near, worst = 0, 0.0
    for sc in golden:
        query, m0 = _query(sc["queries"])
        out = detect.boxes_from_matches(sc["ref"], query, m0, sc["hw"])
        out32 = detect.boxes_from_matches(sc["ref"], query, m0.to(torch.int32), sc["hw"])
        for k in out:
            assert torch.equal(out[k], out32[k]), k
        sizes = sc["ref"]["sizes"].cpu().numpy()
        for b, q in enumerate(sc["queries"]):
            assert int(out["view"][b]) == int(q["view"]) and int(out["n_matches"][b]) == int(q["n_matches"])
            st = int(out["status"][b])
            if int(q["n_matches"]) < detect.MIN_MATCHES:
                assert st == 2 and out["box"][b].tolist() == [0, 0, sc["hw"][0], sc["hw"][1]] == q["bbox"].tolist()
                continue
            assert st == 1
            Hg = out["affine"][b].cpu().numpy()
            worst = max(worst, float(np.abs(Hg - q["affine"]).max() / np.abs(q["affine"]).max()))
            assert np.abs(Hg - q["affine"]).max() <= REFINE_RTOL * np.abs(q["affine"]).max()
            if _near_integer_corner(Hg, sizes[int(q["view"])]):
                near += 1
                continue
            assert out["box"][b].tolist() == q["bbox"].tolist(), (b, out["box"][b], q["bbox"])
    print(f"boxes: {near} frames with a corner within 1e-9 of an integer (not compared); affine vs cv2 max rel. {worst:.2e}")
    assert near == 0


def test_crops_equal_the_reference(golden):
    for sc in golden:
        for S in sorted({int(q["crop_size"]) for q in sc["queries"]}):
            qs = [q for q in sc["queries"] if int(q["crop_size"]) == S]
            query, m0 = _query(qs)
            frames = sc["frame"][None].expand(len(qs), -1, -1)
            bbox, image, K_crop = detect.detect_from_matches(frames, torch.from_numpy(sc["K"]).to(DEV), sc["ref"], query, m0, crop_size=S)
            img = image.cpu().numpy()
            for b, q in enumerate(qs):
                assert bbox[b].tolist() == q["bbox"].tolist()
                assert np.array_equal(img[b, 0], q["image_crop"].astype(np.float32) / 255)
                np.testing.assert_allclose(K_crop[b].cpu().numpy(), q["K_crop"], rtol=1e-12, atol=0)


def test_quirks_and_the_no_model_departure(golden):
    sc = golden[1]                                                              # portrait 640 x 360
    ref = {k: v.clone() for k, v in sc["ref"].items()}
    V, cap = ref["keypoints"].shape[:2]
    n = int(ref["counts"][2])
    ref["keypoints"][2, :n] = ref["keypoints"][2, 0]                            # view 2's points all coincide
    qkp = torch.rand(3, 50, 2, device=DEV) * 300
    query = {"keypoints": qkp, "counts": torch.tensor([50, 50, 40], dtype=torch.int32, device=DEV)}
    m0 = torch.full((3, V, cap), -1, dtype=torch.int64, device=DEV)
    m0[0, 2, :20] = torch.arange(20)                                            # 20 matches of the coincident view: no model
    m0[1, 1, :5] = torch.arange(5)                                              # 5 and 5: below 6
    m0[1, 3, 3:8] = torch.arange(5)
    m0[2, 0, :30] = torch.arange(40, 70)                                        # indices >= counts[2] = 40 and < -1 are no match
    m0[2, 0, 30:40] = -5
    m0[2, 1, :4] = torch.arange(4)
    out = detect.boxes_from_matches(ref, query, m0, sc["hw"])
    assert out["status"].tolist() == [0, 2, 2] and out["view"].tolist() == [2, 0, 0] and out["n_matches"].tolist() == [20, 0, 0]
    assert out["box"].tolist() == [[0, 0, 0, 0], [0, 0, 640, 360], [0, 0, 640, 360]] and not out["affine"].any()
    frames = sc["frame"][None].expand(3, -1, -1)
    bbox, image, K_crop = detect.detect_from_matches(frames, torch.from_numpy(sc["K"]).to(DEV), ref, query, m0, crop_size=64)
    assert not image[0].any() and image[1].any() and torch.equal(K_crop[0], torch.from_numpy(sc["K"]).to(DEV))


def _random_case(rng, V, B, cap=300, qcap=400):
    sizes = rng.integers(100, 700, (V, 2))
    counts = rng.integers(1, cap + 1, V)
    kp = np.zeros((V, cap, 2), np.float32)
    for v in range(V):
        kp[v, :counts[v]] = np.stack([rng.integers(0, sizes[v, 1], counts[v]), rng.integers(0, sizes[v, 0], counts[v])], 1)
    qc = rng.integers(1, qcap + 1, B)
    qkp = rng.uniform(0, 800, (B, qcap, 2)).astype(np.float32)
    m0 = np.full((B, V, cap), -1, np.int64)
    for b in range(B):
        for v in range(V):
            k = int(rng.integers(0, min(counts[v], qc[b]) + 1)) if rng.random() < 0.7 else int(rng.integers(0, 7))
            k = min(k, counts[v], qc[b])
            m0[b, v, np.sort(rng.choice(counts[v], k, replace=False))] = rng.choice(qc[b], k, replace=False)
            if rng.random() < 0.5 and k > 10:                                   # a planted similarity for part of the matches
                S = np.array([[0.8, -0.3, 40.0], [0.3, 0.8, 25.0]])
                sel = np.nonzero(m0[b, v] >= 0)[0][: k // 2]
                qkp[b, m0[b, v, sel]] = np.round(kp[v, sel] @ S[:, :2].T + S[:, 2])
    return sizes, counts, kp, qc, qkp, m0


def _host_boxes(sizes, counts, kp, qc, qkp, m0, hw):
    """The reference's rule on the restatement: per frame the count, the choice and the box."""
    out = []
    for b in range(m0.shape[0]):
        n = [int(((m0[b, v, :counts[v]] >= 0) & (m0[b, v, :counts[v]] < qc[b])).sum()) for v in range(m0.shape[1])]
        key = [c if c >= 6 else 0 for c in n]
        win = int(np.argmax(key)) if max(key) else 0
        if max(key) == 0:
            out.append((win, n[win], [0, 0, hw[0], hw[1]], None))
            continue
        m = m0[b, win, :counts[win]]
        valid = (m >= 0) & (m < qc[b])
        H, _, _ = A.estimate_affine_partial_2d(kp[win, :counts[win]][valid], qkp[b, m[valid]], 6.0, minimal="closed")
        box = A.corners_box(H, sizes[win]) if H is not None else None
        out.append((win, n[win], box.tolist() if box is not None else [0, 0, 0, 0], H))
    return out


VIEWS_AND_FRAMES = [(1, 1, 300), (1, 64, 300), (7, 13, 300), (15, 8, 300), (32, 1, 300), (32, 64, 300),
                    (256, 4, 8192)]        # the most views and reference key points opb_boxes_from_matches takes


def _full_view(rng, sizes, counts, kp, qc, qkp, m0, b, v):
    """View v of frame b with all its cap reference key points matched, half of them to a planted similarity: the winner's pairs
    fill the kernel's dynamic shared memory (cap * 16 bytes) exactly."""
    cap = kp.shape[1]
    counts[v] = cap
    kp[v] = np.stack([rng.integers(0, sizes[v, 1], cap), rng.integers(0, sizes[v, 0], cap)], 1)
    qc[b] = max(qc[b], cap)
    m0[b, v] = rng.choice(qc[b], cap, replace=False)
    S = np.array([[0.9, 0.2, 30.0], [-0.2, 0.9, 12.0]])
    qkp[b, m0[b, v, :cap // 2]] = np.round(kp[v, :cap // 2] @ S[:, :2].T + S[:, 2])


@pytest.mark.parametrize("V,B,cap", VIEWS_AND_FRAMES, ids=[f"{V}-{B}" if cap == 300 else f"{V}-{B}-{cap}" for V, B, cap in VIEWS_AND_FRAMES])
def test_views_and_frames(V, B, cap):
    """Random views and frames against _host_boxes.  At cap = 8192 the query holds 16384 key points, and frame 0's winning view
    has all 8192 of its key points matched."""
    rng = np.random.default_rng(V * 100 + B)
    sizes, counts, kp, qc, qkp, m0 = _random_case(rng, V, B, cap, 400 if cap == 300 else 2 * cap)
    if cap == 8192:
        _full_view(rng, sizes, counts, kp, qc, qkp, m0, 0, V - 1)
    ref = {"keypoints": torch.from_numpy(kp).to(DEV), "counts": torch.from_numpy(counts).to(DEV), "sizes": torch.from_numpy(sizes).to(DEV)}
    query = {"keypoints": torch.from_numpy(qkp).to(DEV), "counts": torch.from_numpy(qc).to(DEV)}
    out = detect.boxes_from_matches(ref, query, torch.from_numpy(m0).to(DEV), (720, 960))
    near = 0
    for b, (win, n, box, H) in enumerate(_host_boxes(sizes, counts, kp, qc, qkp, m0, (720, 960))):
        assert int(out["view"][b]) == win and int(out["n_matches"][b]) == n, b
        if H is not None and _near_integer_corner(out["affine"][b].cpu().numpy(), sizes[win]):
            near += 1
            continue
        assert out["box"][b].tolist() == box, (b, out["box"][b], box)
    print(f"V={V} B={B} cap={cap}: {near} frames with a corner within 1e-9 of an integer")
    if cap == 8192:
        assert int(out["view"][0]) == V - 1 and int(out["n_matches"][0]) == cap and int(out["status"][0]) == 1
    one = detect.boxes_from_matches(ref, {k: v[B - 1:] for k, v in query.items()}, torch.from_numpy(m0[B - 1:]).to(DEV), (720, 960))
    for k in out:
        assert torch.equal(one[k][0], out[k][B - 1]), k


def test_strided_inputs_and_a_side_stream_equal_the_default_stream():
    rng = np.random.default_rng(77)
    sizes, counts, kp, qc, qkp, m0 = _random_case(rng, 9, 16)
    ref = {"keypoints": torch.from_numpy(kp).to(DEV), "counts": torch.from_numpy(counts).to(DEV), "sizes": torch.from_numpy(sizes).to(DEV)}
    query = {"keypoints": torch.from_numpy(qkp).to(DEV), "counts": torch.from_numpy(qc).to(DEV)}
    m = torch.from_numpy(m0).to(DEV)
    want = detect.boxes_from_matches(ref, query, m, (720, 960))
    wide = torch.full((16, 9, m.shape[2] * 2), -3, dtype=torch.int64, device=DEV)
    wide[:, :, ::2] = m
    got = detect.boxes_from_matches(ref, query, wide[:, :, ::2], (720, 960))
    for k in want:
        assert torch.equal(got[k], want[k]), k
    f, t = planted(8, 500, 0.5)
    want_a, _ = _batch([(f, t), (t, f)])
    torch.cuda.synchronize()
    s = torch.cuda.Stream(DEV)
    with torch.cuda.stream(s):
        m2 = m + 0
        got = detect.boxes_from_matches(ref, query, m2, (720, 960))
        got_a, _ = _batch([(f, t), (t, f)])
    s.synchronize()
    for k in want:
        assert torch.equal(got[k], want[k]), k
    for k in want_a:
        assert torch.equal(got_a[k], want_a[k]), k


def test_every_output_element_is_written(monkeypatch):
    made = []
    real_empty = torch.empty

    def poisoned(*a, **kw):
        t = real_empty(*a, **kw)
        t.view(torch.uint8).fill_(0xFF) if t.numel() else None
        made.append(t)
        return t

    rng = np.random.default_rng(9)
    sizes, counts, kp, qc, qkp, m0 = _random_case(rng, 5, 12)
    ref = {"keypoints": torch.from_numpy(kp).to(DEV), "counts": torch.from_numpy(counts).to(DEV), "sizes": torch.from_numpy(sizes).to(DEV)}
    query = {"keypoints": torch.from_numpy(qkp).to(DEV), "counts": torch.from_numpy(qc).to(DEV)}
    m = torch.from_numpy(m0).to(DEV)
    f, t = planted(4, 200, 0.5)
    probs = [(f, t), (f[:1], t[:1]), (f[:2], t[:2]), (np.tile(f[:1], (9, 1)), t[:9])]
    monkeypatch.setattr(torch, "empty", poisoned)
    out = detect.boxes_from_matches(ref, query, m, (720, 960))
    out_a, _ = _batch(probs)
    monkeypatch.undo()
    assert len(made) >= 9
    for k, v in list(out.items()) + list(out_a.items()):
        if v.dtype == torch.uint8:
            assert not (v == 0xFF).any(), k
        elif v.dtype == torch.float64:
            assert not torch.isnan(v).any(), k
        elif v.dtype == torch.int32:
            assert not (v == -1).any(), k
    assert set(out_a["inliers"].unique().tolist()) <= {0, 1} and out_a["status"].tolist() == [1, 0, 1, 0]


def test_argument_mistakes_raise():
    f, t = planted(1, 20, 0.0)
    ft, tt = torch.from_numpy(f).to(DEV), torch.from_numpy(t).to(DEV)
    offs = torch.tensor([0, 20], dtype=torch.int32, device=DEV)
    with pytest.raises(RuntimeError, match="no CPU path"):
        detect.affine_partial_batch(ft.cpu(), tt, offs)
    for bad in (lambda: detect.affine_partial_batch(ft, tt[:5], offs), lambda: detect.affine_partial_batch(ft, tt, offs.long()),
                lambda: detect.affine_partial_batch(ft, tt, offs[:1]), lambda: detect.affine_partial_batch(ft, tt, offs, confidence=1.0)):
        with pytest.raises(ValueError):
            bad()
    rng = np.random.default_rng(2)
    sizes, counts, kp, qc, qkp, m0 = _random_case(rng, 3, 2)
    ref = {"keypoints": torch.from_numpy(kp).to(DEV), "counts": torch.from_numpy(counts).to(DEV), "sizes": torch.from_numpy(sizes).to(DEV)}
    query = {"keypoints": torch.from_numpy(qkp).to(DEV), "counts": torch.from_numpy(qc).to(DEV)}
    m = torch.from_numpy(m0).to(DEV)
    for bad in (lambda: detect.boxes_from_matches(ref, query, m.float(), (720, 960)), lambda: detect.boxes_from_matches(ref, query, m[:, :2], (720, 960)),
                lambda: detect.boxes_from_matches(ref, query, m, (0, 960)), lambda: detect.boxes_from_matches({**ref, "sizes": ref["sizes"][:2]}, query, m, (720, 960)),
                lambda: detect.boxes_from_matches({**ref, "keypoints": torch.zeros(3, 9000, 2, device=DEV)}, query, m, (720, 960))):
        with pytest.raises(ValueError):
            bad()
    lib = _lib.load()
    assert lib.opb_boxes_from_matches(None, None, None, 0, 1, None, None, 1, None, 0, 1, 1, 1, None, None, None, None, None, None) == -1
    assert lib.opb_estimate_affine_partial(ft.data_ptr(), tt.data_ptr(), offs.data_ptr(), 1, 3.0, 2000, 1.5, 10, 0, 0, 0, 0, None) == -1


class StubExtractor:
    """Hands out the golden key points: the reference views first (one per constructor call), then the queries."""

    def __init__(self, views, queries):
        self.views, self.queries = list(views), queries

    def forward(self, inp):
        assert inp.dtype == torch.float32 and inp.dim() == 4 and float(inp.max()) <= 1.0
        if self.views:
            kp = self.views.pop(0)
            return {"keypoints": [kp], "scores": [torch.ones(len(kp), device=DEV)], "descriptors": [torch.zeros(256, len(kp), device=DEV)]}
        assert inp.shape[0] == len(self.queries)
        kps = [torch.from_numpy(q["keypoints"]).to(DEV) for q in self.queries]
        return {"keypoints": kps, "scores": [torch.ones(len(k), device=DEV) for k in kps], "descriptors": [torch.zeros(256, len(k), device=DEV) for k in kps]}


class StubMatcher(torch.nn.Module):
    """matches0 of (frame, view) in call order, checking the reference's match dict."""

    def __init__(self, queries, ref_counts, ref_sizes, hw):
        super().__init__()
        self.queries, self.counts, self.sizes, self.hw, self.calls = queries, ref_counts, ref_sizes, hw, 0

    def forward(self, data):
        V = len(self.counts)
        b, v = divmod(self.calls, V)
        self.calls += 1
        n = int(self.counts[v])
        assert tuple(data["keypoints0"].shape) == (1, n, 2) and tuple(data["descriptors0"].shape) == (1, 256, n)
        assert tuple(data["keypoints1"].shape) == (1, len(self.queries[b]["keypoints"]), 2)
        assert tuple(data["image0"].shape) == (1, 1, int(self.sizes[v][1]), int(self.sizes[v][0]))        # (1, 1) + size[::-1]
        assert tuple(data["image1"].shape) == (1, 1, self.hw[1], self.hw[0])
        return {"matches0": torch.from_numpy(self.queries[b]["matches0"][v, :n]).to(DEV)[None]}


def test_local_feature_object_detector_drop_in(golden):
    sc = golden[0]
    qs = [q for q in sc["queries"] if int(q["crop_size"]) == 128]
    counts, sizes = sc["ref"]["counts"].cpu().numpy(), sc["ref"]["sizes"].cpu().numpy()
    views = [sc["ref"]["keypoints"][v, :counts[v]] for v in range(len(counts))]
    imgs = [np.zeros((int(h), int(w)), np.uint8) for h, w in sizes]
    det = detect.LocalFeatureObjectDetector(StubExtractor(views, qs), StubMatcher(qs, counts, sizes, sc["hw"]), imgs, crop_size=128)
    frames = sc["frame"][None].expand(len(qs), -1, -1)
    bbox, image, K_crop = det.detect(frames, torch.from_numpy(sc["K"]).to(DEV))
    img = image.cpu().numpy()
    for b, q in enumerate(qs):
        assert bbox[b].tolist() == q["bbox"].tolist()
        assert np.array_equal(img[b, 0], q["image_crop"].astype(np.float32) / 255)
        np.testing.assert_allclose(K_crop[b].cpu().numpy(), q["K_crop"], rtol=1e-12, atol=0)


def test_closed_loop_detect_then_pose():
    """A planted object: reference view key points are its points seen from a reference pose; the frame's key points are the
    same points under a new pose plus clutter.  The detected box contains the object's projections, and the pose from the crop
    (the key points carried by T2 . T1, K_crop) is the planted one."""
    rng = np.random.default_rng(21)
    H, W, M = 720, 960, 120
    K = np.array([[800.0, 0, 480.5], [0, 800.0, 360.25], [0, 0, 1]])
    half = np.array([0.08, 0.06, 0.04])
    pts3d = rng.uniform(-1, 1, (M, 3)) * half
    pose = np.concatenate([np.eye(3), np.array([[0.05], [-0.02], [0.7]])], axis=1)
    a = 0.4
    ref_pose = np.concatenate([np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]]), np.array([[0.0], [0.0], [0.5]])], axis=1)
    ref_kp = cr.reproj(K, ref_pose, pts3d)[:, :2] - np.array([160, 80])                   # the reference view: a 480 x 640 crop
    q_kp = cr.reproj(K, pose, pts3d)
    clutter = rng.uniform([0, 0], [W, H], (200, 2))
    qk = np.concatenate([q_kp, clutter]).astype(np.float32)
    ref = {"keypoints": torch.from_numpy(ref_kp.astype(np.float32))[None].to(DEV), "counts": torch.tensor([M], dtype=torch.int32, device=DEV),
           "sizes": torch.tensor([[480, 640]], dtype=torch.int32, device=DEV)}
    query = {"keypoints": torch.from_numpy(qk)[None].to(DEV), "counts": torch.tensor([len(qk)], dtype=torch.int32, device=DEV)}
    m0 = np.arange(M)
    wrong = rng.random(M) < 0.3
    m0[wrong] = rng.integers(M, len(qk), int(wrong.sum()))                                # 30 % wrong matches
    m0 = torch.from_numpy(m0)[None, None].to(DEV)
    frames = torch.zeros(1, H, W, dtype=torch.uint8, device=DEV)
    for u, v in np.rint(q_kp).astype(int):
        frames[0, max(v - 1, 0):v + 2, max(u - 1, 0):u + 2] = 255
    out = detect.boxes_from_matches(ref, query, m0, (H, W))
    box = out["box"][0].tolist()
    assert int(out["status"][0]) == 1
    assert box[0] <= q_kp[:, 0].min() and box[1] <= q_kp[:, 1].min() and box[2] >= q_kp[:, 0].max() - 1 and box[3] >= q_kp[:, 1].max() - 1, box
    res = crop.crop_frames(frames, out["box"], torch.from_numpy(K).to(DEV), 512)
    tr = res["trans"][0].cpu().numpy()
    homo = [np.concatenate([tr[s], [[0, 0, 1.0]]]) for s in (0, 1)]
    kp = (homo[1] @ homo[0] @ np.concatenate([q_kp, np.ones((M, 1))], axis=1).T).T[:, :2]
    pose_res = pnp.poses_from_matches(res["K_crop"], torch.from_numpy(kp)[None].to(DEV, torch.float32), torch.from_numpy(pts3d).to(DEV, torch.float32),
                                      torch.arange(M, device=DEV)[None], scale=1000)
    rot, trans = pnp.pose_errors(pose_res["pose"], torch.from_numpy(pose)[None].to(DEV))
    assert float(rot[0]) < 1.0 and float(trans[0]) < 1.0 and int(pose_res["n_inliers"][0]) >= M - 2
    assert res["status"].tolist() == [1] and res["image"][0].any() and res["image"][0].mean() < 0.5
