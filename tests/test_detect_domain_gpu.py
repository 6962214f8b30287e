"""The detector (csrc/detect.cu) across the domain it accepts: the estimator against cv2 4.13's results at every threshold,
budget, confidence, problem size, non-finite row, refinement length and sub-unit fit (tests/golden/pnp_detect_domain_cases.npz, made by
tests/golden/make_detect_domain.py), its loop at the 32-sample wave, ragged and offset layouts, the view choice at its edges and
the box of exact scenes at the int32 edge.  The restatement (tests/affine_ransac_reference.py) referees the samples and counts."""
import os
import re

import numpy as np
import pytest
import torch

from onepose_b200 import _lib, detect
from tests import affine_ransac_reference as A
from tests.golden_util import GOLDEN_DIR
from tests.opencv_ransac_reference import update_num_iters

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
REFINE_RTOL = 1e-10          # the restatement's bar against cv2 (tests/test_affine_ransac_reference_cpu.py)
WAVE = 32                    # samples per round of the device loop (kAffWave)
UNTOUCHED = -7


def planted(seed, n, frac, noise=1.0, shift=0.0):
    r = np.random.default_rng(seed)
    f = r.uniform([0, 0], [640, 480], (n, 2))
    a, s = r.uniform(-3, 3), r.uniform(0.3, 3)
    R = s * np.array([[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]])
    t = f @ R.T + r.uniform(-300, 300, 2) + r.normal(0, noise, (n, 2))
    out = r.random(n) < frac
    t[out] = r.uniform(0, 1500, (int(out.sum()), 2))
    return (f + shift).astype(np.float32), (t + shift).astype(np.float32)


class Trace:
    def __init__(self, B, cap):
        self.cap = cap
        self.samples = torch.full((B, cap, 2), UNTOUCHED, dtype=torch.int32, device=DEV)
        self.counts = torch.full((B, cap), UNTOUCHED, dtype=torch.int32, device=DEV)
        self.models = torch.full((B, cap, 6), float("nan"), dtype=torch.float64, device=DEV)

    def __enter__(self):
        _lib.check(_lib.load().opb_debug_set_affine_trace(self.samples.data_ptr(), self.counts.data_ptr(), self.models.data_ptr(), self.cap))
        return self

    def __exit__(self, *a):
        torch.cuda.synchronize()
        _lib.check(_lib.load().opb_debug_set_affine_trace(None, None, None, 0))


def _batch(problems, **kw):
    offs = np.cumsum([0] + [len(f) for f, _ in problems]).astype(np.int32)
    f = torch.from_numpy(np.concatenate([p[0] for p in problems]).reshape(-1, 2).astype(np.float32)).to(DEV)
    t = torch.from_numpy(np.concatenate([p[1] for p in problems]).reshape(-1, 2).astype(np.float32)).to(DEV)
    out = detect.affine_partial_batch(f, t, torch.from_numpy(offs).to(DEV), **kw)
    return {k: v.cpu().numpy() for k, v in out.items()}, offs


def _rel(H, ref):
    return float(np.abs(H - ref).max() / np.abs(ref).max())


# ---- the estimator against cv2 across the domain ----

@pytest.fixture(scope="module")
def cases():
    g = np.load(os.path.join(GOLDEN_DIR, "pnp_detect_domain_cases.npz"), allow_pickle=False)
    keys = ("from", "to", "thr", "conf", "max_iters", "refine", "ok", "affine", "mask", "iterations", "winner", "counts", "samples", "models")
    return [dict(tag=str(tag), **{k: g[f"c{i}_{k}"] for k in keys}) for i, tag in enumerate(g["c_tags"])]


CATEGORIES = ("thr", "conf", "iters", "n", "nonfinite", "refine", "subunit")
_worst = {}


@pytest.mark.parametrize("category", CATEGORIES)
def test_cases_against_cv2(cases, category):
    """Every case of a category, one call per (threshold, confidence, maxIters, refineIters): the samples, per-sample counts and
    minimal models equal the restatement's, the winner follows its scan, and the iteration count, the status and the mask equal
    cv2's; the affine is cv2's bit for bit without refinement (and for 2 pairs) and within REFINE_RTOL with it."""
    sel = [c for c in cases if re.match("[a-z]+", c["tag"]).group() == category]
    assert sel
    groups = {}
    for c in sel:
        groups.setdefault((float(c["thr"]), float(c["conf"]), int(c["max_iters"]), int(c["refine"])), []).append(c)
    for (thr, conf, max_iters, ri), cs in groups.items():
        cap = max(max(int(c["iterations"]) for c in cs), 1) + WAVE
        with Trace(len(cs), cap) as tr:
            out, offs = _batch([(c["from"], c["to"]) for c in cs], threshold=thr, confidence=conf, max_iters=max_iters, refine_iters=ri)
        samples, counts, models = tr.samples.cpu().numpy(), tr.counts.cpu().numpy(), tr.models.cpu().numpy()
        for b, c in enumerate(cs):
            n, it = len(c["from"]), int(c["iterations"])
            assert int(out["iterations"][b]) == it and int(out["status"][b]) == int(c["ok"]), c["tag"]
            assert np.array_equal(out["inliers"][offs[b]:offs[b + 1]], c["mask"]), c["tag"]
            if n > 2:
                assert np.array_equal(samples[b, :it], c["samples"]) and np.array_equal(counts[b, :it], c["counts"]), c["tag"]
                assert models[b, :it].reshape(it, 2, 3).tobytes() == c["models"].tobytes(), c["tag"]
                assert A.scan(counts[b, :it], n, conf, max_iters) == (int(c["winner"]), int(counts[b, c["winner"]]) if c["winner"] >= 0 else 0, it)
                if it == max(max_iters, 1):                 # a budget no sample lowered: nothing is drawn past it
                    assert (counts[b, it:] == UNTOUCHED).all(), c["tag"]
            H = out["affine"][b]
            if not c["ok"]:
                assert not H.any(), c["tag"]
            elif ri == 0 or n == 2:
                assert H.tobytes() == c["affine"].tobytes(), c["tag"]
            else:
                rel = _rel(H, c["affine"])
                key = c["tag"].rsplit("_s", 1)[0]
                _worst[key] = max(_worst.get(key, 0.0), rel)
                assert rel <= REFINE_RTOL, (c["tag"], rel)
            print(f"{c['tag']}: {it} iterations, winner {int(c['winner'])}, {int(c['mask'].sum())} inliers")
    print(f"{category}: refined affine vs cv2, max relative difference:", {k: f"{v:.1e}" for k, v in _worst.items() if k.startswith(category)})


# ---- the loop at the 32-sample wave ----

@pytest.mark.parametrize("target", (WAVE, 2 * WAVE))
def test_budget_lowered_onto_a_wave_boundary(target):
    """A confidence chosen so that RANSACUpdateNumIters lowers the budget to exactly `target` (a multiple of the wave) once an
    all-inlier sample wins: the loop ends on the wave's last sample and no later wave is drawn."""
    f, t = planted(1900, 100, 0.4, 0.0)
    _, m, info = A.estimate_affine_partial_2d(f, t, 3.0, 2000, 0.5, 0, minimal="closed")
    c = int(m.sum())
    conf = 1 - (1 - (c / 100) ** 2) ** target
    assert update_num_iters(conf, (100 - c) / 100, 2, 2000) == target
    _, _, info = A.estimate_affine_partial_2d(f, t, 3.0, 2000, conf, 0, minimal="closed")
    assert info["iterations"] == target and max(info["counts"]) == c and info["winner"] < target
    with Trace(1, 4 * WAVE) as tr:
        out, _ = _batch([(f, t)], threshold=3.0, confidence=conf, max_iters=2000, refine_iters=0)
    counts = tr.counts[0].cpu().numpy()
    assert int(out["iterations"][0]) == target and counts[:target].tolist() == info["counts"]
    assert (counts[target:] == UNTOUCHED).all()


# ---- layouts ----

def _solo(f, t, **kw):
    out, _ = _batch([(f, t)], **kw)
    return out


def test_ragged_batch_and_independence():
    """Problems of 0 to 10^5 pairs in one call: each equals the restatement (samples, counts, iterations, mask, and the affine to
    REFINE_RTOL) and is bit-identical to the same problem alone and in a reversed batch."""
    sizes = (0, 1, 2, 3, 31, 32, 33, 255, 256, 257, 100000)
    probs = [planted(2000 + k, n, 0.5) if n else (np.zeros((0, 2), np.float32), np.zeros((0, 2), np.float32)) for k, n in enumerate(sizes)]
    with Trace(len(probs), 2000) as tr:
        out, offs = _batch(probs, threshold=3.0)
    rev, roffs = _batch(probs[::-1], threshold=3.0)
    for b, (f, t) in enumerate(probs):
        n = len(f)
        H, m, info = A.estimate_affine_partial_2d(f, t, 3.0, 2000, 0.99, 10, minimal="closed")
        it = info["iterations"]
        assert int(out["iterations"][b]) == it and int(out["status"][b]) == (H is not None), n
        assert np.array_equal(out["inliers"][offs[b]:offs[b + 1]], m), n
        if n > 2:
            assert tr.counts[b, :it].cpu().tolist() == info["counts"] and tr.samples[b, :it].cpu().numpy().tolist() == [list(s) for s in info["samples"]]
        if H is None:
            assert not out["affine"][b].any()
        elif n == 2:
            assert out["affine"][b].tobytes() == H.tobytes()
        else:
            assert _rel(out["affine"][b], H) <= REFINE_RTOL, n
        r = len(probs) - 1 - b
        assert out["affine"][b].tobytes() == rev["affine"][r].tobytes() and out["iterations"][b] == rev["iterations"][r]
        assert np.array_equal(out["inliers"][offs[b]:offs[b + 1]], rev["inliers"][roffs[r]:roffs[r + 1]])
        if n in (3, 257, 100000):
            one = _solo(f, t, threshold=3.0)
            assert one["affine"][0].tobytes() == out["affine"][b].tobytes() and np.array_equal(one["inliers"], out["inliers"][offs[b]:offs[b + 1]])
        print(f"n={n}: {it} iterations, winner {info['winner']}")


def test_more_than_65535_problems():
    """70001 problems, seven distinct ones in turn: every result equals its period's, and the seven equal the restatement."""
    base = [planted(2100 + k, n, frac, 0.0) for k, (n, frac) in enumerate(((2, 0), (3, 0), (6, 0.3), (8, 0.5), (12, 0.4), (5, 0.0), (40, 0.6)))]
    B = 70001
    probs = [base[b % 7] for b in range(B)]
    out, offs = _batch(probs, threshold=3.0)
    aff = out["affine"].reshape(B, 6)
    for k, (f, t) in enumerate(base):
        H, m, info = A.estimate_affine_partial_2d(f, t, 3.0, 2000, 0.99, 10, minimal="closed")
        idx = np.arange(k, B, 7)
        assert (out["iterations"][idx] == info["iterations"]).all() and (out["status"][idx] == (H is not None)).all()
        assert (aff[idx].view(np.int64) == aff[k].view(np.int64)).all()
        masks = np.stack([out["inliers"][offs[b]:offs[b + 1]] for b in idx[:: max(len(idx) // 500, 1)]] + [out["inliers"][offs[idx[-1]]:offs[idx[-1] + 1]]])
        assert (masks == m).all()
        if H is not None and len(f) == 2:
            assert aff[k].tobytes() == H.reshape(6).tobytes()
        elif H is not None:
            assert _rel(aff[k].reshape(2, 3), H) <= REFINE_RTOL


def test_offsets_start_past_zero_and_rows_outside_are_not_written():
    """offsets[0] > 0, a gap of rows between two problems is impossible (offsets are one table), so rows before offsets[0] and past
    offsets[B] are the rows outside every problem: poisoned, they stay poisoned."""
    p = [planted(2200, 50, 0.3), planted(2201, 33, 0.5)]
    lead, tail = 7, 5
    f = np.concatenate([np.full((lead, 2), 9.0, np.float32), p[0][0], p[1][0], np.full((tail, 2), 9.0, np.float32)])
    t = np.concatenate([np.full((lead, 2), 3.0, np.float32), p[0][1], p[1][1], np.full((tail, 2), 3.0, np.float32)])
    offs = torch.tensor([lead, lead + 50, lead + 83], dtype=torch.int32, device=DEV)
    ft, tt = torch.from_numpy(f).to(DEV), torch.from_numpy(t).to(DEV)
    mask = torch.full((len(f),), 0xAB, dtype=torch.uint8, device=DEV)
    aff = torch.empty(2, 2, 3, dtype=torch.float64, device=DEV)
    it = torch.empty(2, dtype=torch.int32, device=DEV)
    st = torch.empty(2, dtype=torch.int32, device=DEV)
    _lib.call(torch.device(DEV), "opb_estimate_affine_partial", ft, tt, offs, 2, 3.0, 2000, 0.99, 10, aff, mask, it, st)
    mk = mask.cpu().numpy()
    assert (mk[:lead] == 0xAB).all() and (mk[lead + 83:] == 0xAB).all()
    for b, (pf, pt) in enumerate(p):
        one = _solo(pf, pt, threshold=3.0)
        o = lead + (0, 50)[b]
        assert np.array_equal(mk[o:o + len(pf)], one["inliers"]) and aff[b].cpu().numpy().tobytes() == one["affine"][0].tobytes()
        assert int(it[b]) == int(one["iterations"][0]) and int(st[b]) == int(one["status"][0])


# ---- the view choice ----

def _host_choice(counts, qc, m0, cap_ref, cap_q):
    """match_worker's counts with the kernel's clamps (ref count to [0, cap_ref], query count to [0, cap_q]) and the choice: the
    most matches among views with >= 6, the first on a tie, view 0 and status 2 when none has 6."""
    out = []
    for b in range(m0.shape[0]):
        nq = min(max(int(qc[b]), 0), cap_q)
        rows = [m0[b, v, :min(max(int(counts[v]), 0), cap_ref)] for v in range(m0.shape[1])]
        n = [int(((m >= 0) & (m < nq)).sum()) for m in rows]
        key = [c if c >= 6 else 0 for c in n]
        win = int(np.argmax(key)) if max(key) else 0
        out.append((win, n[win], max(key) > 0))
    return out


def _run_choice(kp, counts, sizes, qkp, qc, m0, hw=(720, 960)):
    ref = {"keypoints": torch.from_numpy(kp).to(DEV), "counts": torch.from_numpy(np.asarray(counts, np.int32)).to(DEV),
           "sizes": torch.from_numpy(np.asarray(sizes, np.int32)).to(DEV)}
    query = {"keypoints": torch.from_numpy(qkp).to(DEV), "counts": torch.from_numpy(np.asarray(qc, np.int32)).to(DEV)}
    m = torch.from_numpy(m0).to(DEV)
    out = {k: v.cpu().numpy() for k, v in detect.boxes_from_matches(ref, query, m, hw).items()}
    B, V = m0.shape[:2]
    objs = detect.boxes_from_matches_objects(ref, np.zeros(B, np.int32), np.full(B, V, np.int32), query, np.arange(B, dtype=np.int32), m, hw)
    for k, v in objs.items():
        assert np.array_equal(v.cpu().numpy(), out[k]), k
    if m0.dtype == np.int64 and np.abs(m0).max() < 2**31:
        o32 = detect.boxes_from_matches(ref, query, m.to(torch.int32), hw)
        for k, v in o32.items():
            assert np.array_equal(v.cpu().numpy(), out[k]), k
    return out


def _choice_case(rng, V, B, cap, qcap):
    sizes = np.tile([[480, 640]], (V, 1))
    kp = rng.uniform(0, 600, (V, cap, 2)).astype(np.float32)
    qkp = rng.uniform(0, 900, (B, qcap, 2)).astype(np.float32)
    return kp, sizes, qkp, np.full((B, V, cap), -1, np.int64)


def test_view_choice_edges():
    """Ties between views (the first wins), 5 against 6 matches (6 counts, 5 does not), the winner as the 256th view, counts
    above the caps and negative (clamped), int64 entries at +-2^31 and beyond (never an index), duplicate matches to one query
    point, and cap_ref 1; boxes_from_matches_objects on the same rows agrees field for field."""
    rng = np.random.default_rng(31)
    V, B, cap, qcap = 256, 9, 40, 50
    kp, sizes, qkp, m0 = _choice_case(rng, V, B, cap, qcap)
    counts, qc = np.full(V, cap), np.full(B, qcap)
    m0[0, 3, :10] = np.arange(10)                                  # frame 0: views 3 and 7 tie at 10, view 9 has 9
    m0[0, 7, 5:15] = np.arange(20, 30)
    m0[0, 9, :9] = np.arange(9)
    m0[1, 0, :5] = np.arange(5)                                    # frame 1: 5 at view 0, 6 at view 200
    m0[1, 200, 10:16] = np.arange(6)
    m0[2, 4, :5] = np.arange(5)                                    # frame 2: 5 and 5: no view counts
    m0[2, 5, :5] = np.arange(5)
    m0[3, 254, :20] = np.arange(20)                                # frame 3: the winner is the 256th view
    m0[3, 255, :21] = np.arange(21)
    m0[4, 1, :cap] = np.arange(cap)                                # frame 4: view 1's count above cap_ref, view 2's negative
    m0[4, 2, :cap] = np.arange(cap)
    counts[1], counts[2] = 10**6, -5
    m0[5, 0, :30] = np.arange(30)                                  # frame 5: query count above cap_q
    qc[5] = 10**6
    m0[6, 0, :30] = np.arange(30)                                  # frame 6: query count 0 (and frame 7 negative)
    qc[6], qc[7] = 0, -3
    m0[7, 0, :30] = np.arange(30)
    m0[8, 0, :12] = [2**31, -2**31, 2**32, 2**32 + 3, -2**32 + 3, 2**63 - 1, -2**63, 2**31 - 1, 3, 3, 3, 3]   # 4 valid (3, 3, 3, 3)
    m0[8, 6, :8] = 17                                               # 8 matches, all to query point 17
    sizes[200] = (300, 200)
    out = _run_choice(kp, counts, sizes, qkp, qc, m0)
    want = _host_choice(counts, qc, m0, cap, qcap)
    for b, (win, n, ok) in enumerate(want):
        assert (int(out["view"][b]), int(out["n_matches"][b])) == (win, n), b
        assert (int(out["status"][b]) == 2) == (not ok), b
    assert [w for w, _, _ in want] == [3, 200, 0, 255, 1, 0, 0, 0, 6] and want[4][1] == cap and want[8][1] == 8
    cap1 = _choice_case(rng, 3, 2, 1, 8)                            # cap_ref 1: one key point per view
    kp1, s1, q1, m1 = cap1
    m1[:, :, 0] = [[2, 5, 5], [-1, 7, 2**40]]
    out = _run_choice(kp1, [1, 1, 1], s1, q1, [8, 8], m1)
    assert out["status"].tolist() == [2, 2] and out["n_matches"].tolist() == [1, 0]


# ---- boxes of exact scenes: truncation toward zero and the int32 edge ----

def _exact_scene(a, tx, ty):
    """Six pairs with dyadic coordinates under the similarity (a, 0, tx, ty); the first sample OpenCV draws for 6 pairs is (3, 4),
    which sit (0.5, 0.5) apart, so the 2-point model is exact, every pair has error 0 and the refinement keeps the model."""
    f = np.array([[0.25, 0.0], [0.0, 0.75], [1.0, 0.25], [0.0, 0.0], [0.5, 0.5], [0.75, 1.0]], np.float32)
    assert A.subsets(6, 1) == [(3, 4)]
    t = np.stack([a * f[:, 0] + tx, a * f[:, 1] + ty], 1).astype(np.float32)
    assert np.array_equal(t.astype(np.float64), np.stack([a * f[:, 0].astype(np.float64) + tx, a * f[:, 1].astype(np.float64) + ty], 1))
    return f, t


CORNERS = [  # a, tx, ty, (h, w), status, box
    (1.0, -1.5, -0.5, (100, 100), 1, [-1, 0, 98, 99]),
    (1.0, 3.0, -7.0, (100, 100), 1, [3, -7, 103, 93]),
    (1.0, 0.5, 2.5, (11, 13), 1, [0, 2, 13, 13]),
    (2.0**20, -0.5, 0.0, (1, 2048), 1, [0, 0, 2147483647, 2**20]),
    (2.0**20, 0.0, 0.0, (1, 2048), 0, [0, 0, 0, 0]),
    (-(2.0**20), -0.5, 0.0, (1, 2048), 1, [-2147483648, -(2**20), 0, 0]),
    (-(2.0**20), -1.0, 0.0, (1, 2048), 0, [0, 0, 0, 0]),
]


@pytest.mark.parametrize("a,tx,ty,hw,status,box", CORNERS)
def test_exact_corners(a, tx, ty, hw, status, box):
    """Corners at -1.5, -0.5, integers, x.5, 2147483647.5 and 2147483648 (and their negatives): the cast truncates toward zero,
    2147483647.5 is still int32 and 2147483648 or -2147483649 is not (status 0, the empty box)."""
    f, t = _exact_scene(a, tx, ty)
    H, m, _ = A.estimate_affine_partial_2d(f, t, 6.0, 2000, 0.99, 10, minimal="closed")
    assert np.array_equal(H, [[a, 0, tx], [0, a, ty]]) and m.all()
    kp = np.zeros((1, 8, 2), np.float32)
    kp[0, :6] = f
    qkp = np.zeros((1, 8, 2), np.float32)
    qkp[0, :6] = t
    m0 = np.full((1, 1, 8), -1, np.int64)
    m0[0, 0, :6] = np.arange(6)
    out = _run_choice(kp, [6], [hw], qkp, [6], m0)
    assert np.array_equal(out["affine"][0], [[a, 0, tx], [0, a, ty]])
    assert int(out["status"][0]) == status and out["box"][0].tolist() == box
    hb = A.corners_box(H, hw)
    assert (hb is None) == (status == 0) and (hb is None or hb.tolist() == box)


# ---- every box from its affine ----

def _box_from_affine(H, hw):
    """The kernel's box: per corner ((H[r,0] cx + H[r,1] cy) + H[r,2]) in fp64, each operation rounded on its own, truncated
    toward zero; None where a corner is not finite or outside (-2147483649, 2147483648)."""
    h, w = float(hw[0]), float(hw[1])
    lo, hi = [2**31 - 1] * 2, [-(2**31)] * 2
    for cx, cy in ((0.0, 0.0), (w, 0.0), (0.0, h), (w, h)):
        for r in range(2):
            p = (np.float64(H[r, 0]) * cx + np.float64(H[r, 1]) * cy) + np.float64(H[r, 2])
            if not (-2147483649.0 < p < 2147483648.0):
                return None
            q = int(np.trunc(p))
            lo[r], hi[r] = min(lo[r], q), max(hi[r], q)
    return [lo[0], lo[1], hi[0], hi[1]]


def test_every_box_from_its_affine():
    """Random views and frames: the view, the count and the affine against the restatement, and every box recomputed from the
    returned affine -- no frame skipped for a corner near an integer."""
    from tests.test_detect_gpu import _host_boxes, _random_case
    total = 0
    for seed, V, B in ((3100, 5, 64), (3101, 17, 40), (3102, 1, 64)):
        rng = np.random.default_rng(seed)
        sizes, counts, kp, qc, qkp, m0 = _random_case(rng, V, B)
        out = _run_choice(kp, counts, sizes, qkp, qc, m0)
        for b, (win, n, box, H) in enumerate(_host_boxes(sizes, counts, kp, qc, qkp, m0, (720, 960))):
            assert int(out["view"][b]) == win and int(out["n_matches"][b]) == n
            st = int(out["status"][b])
            if n < 6:
                assert st == 2
                continue
            if H is None:
                assert st == 0 and not out["affine"][b].any()
                continue
            assert _rel(out["affine"][b], H) <= REFINE_RTOL
            want = _box_from_affine(out["affine"][b], sizes[win])
            assert st == (1 if want is not None else 0)
            assert out["box"][b].tolist() == (want if want is not None else [0, 0, 0, 0]), (b, out["box"][b], want)
            total += 1
    print(f"{total} boxes recomputed")
    assert total > 50
