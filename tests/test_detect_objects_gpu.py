"""Detection and crops of several objects in the same frames (detect.boxes_from_matches_objects / detect_from_matches_objects /
ObjectDetectors, crop.crop_frames(..., frame_index)): every pair against the single-object calls on its object and frame alone,
bit for bit, the reference detector's goldens regrouped as objects, and a closed loop from planted matches to poses."""
import os

import numpy as np
import pytest
import torch

from onepose_b200 import GATsSuperGlue, _lib, crop, detect, pnp, synthetic
from tests import crop_reference as cr
from tests.golden_util import GOLDEN_DIR

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TRACE_CAP = 2000
HW = (720, 960)


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


def _scene(rng, views_per_object, F, pairs, cap=300, qcap=400):
    """A table of ragged objects, F frames of key points and matches0 [B, V_max, cap] of every pair; rows past a pair's own
    views hold junk that must never be read.  Part of each (pair, view)'s matches follow a planted similarity."""
    n_views = sum(views_per_object)
    first = np.cumsum([0] + list(views_per_object))
    sizes = rng.integers(100, 700, (n_views, 2))
    counts = rng.integers(1, cap + 1, n_views)
    kp = np.zeros((n_views, cap, 2), np.float32)
    for v in range(n_views):
        kp[v, :counts[v]] = np.stack([rng.integers(0, sizes[v, 1], counts[v]), rng.integers(0, sizes[v, 0], counts[v])], 1)
    qc = rng.integers(1, qcap + 1, F)
    qkp = rng.uniform(0, 800, (F, qcap, 2)).astype(np.float32)
    V_max = max(views_per_object[o] for _, o in pairs)
    m0 = rng.integers(-3, qcap, (len(pairs), V_max, cap))
    for b, (f, o) in enumerate(pairs):
        m0[b, :views_per_object[o]] = -1
        for v in range(views_per_object[o]):
            g = first[o] + v
            k = int(rng.integers(0, min(counts[g], qc[f]) + 1)) if rng.random() < 0.7 else int(rng.integers(0, 7))
            k = min(k, counts[g], qc[f])
            m0[b, v, np.sort(rng.choice(counts[g], k, replace=False))] = rng.choice(qc[f], k, replace=False)
            if rng.random() < 0.5 and k > 10:
                S = np.array([[0.8, -0.3, 40.0], [0.3, 0.8, 25.0]])
                sel = np.nonzero(m0[b, v] >= 0)[0][: k // 2]
                qkp[f, m0[b, v, sel]] = np.round(kp[g, sel] @ S[:, :2].T + S[:, 2])
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)  # noqa: E731
    refs = {"keypoints": t(kp), "counts": t(counts), "sizes": t(sizes)}
    query = {"keypoints": t(qkp), "counts": t(qc)}
    vf = np.array([first[o] for _, o in pairs], np.int32)
    vc = np.array([views_per_object[o] for _, o in pairs], np.int32)
    fi = np.array([f for f, _ in pairs], np.int32)
    return refs, query, t(m0), t(vf), t(vc), t(fi)


def _single(refs, query, m0, vf, vc, fi, b, dtype=torch.int64):
    """Pair b through boxes_from_matches on its object's views and its frame alone."""
    v0, n, f = int(vf[b]), int(vc[b]), int(fi[b])
    ref = {k: v[v0:v0 + n] for k, v in refs.items()}
    q = {k: v[f:f + 1] for k, v in query.items()}
    return detect.boxes_from_matches(ref, q, m0[b:b + 1, :n].to(dtype), HW)


CASES = [(1, 1, 1, 1, 0), (3, 7, 2, 9, 1), (16, 32, 8, 40, 2), (5, 12, 4, 20, 3)]      # (objects, most views, frames, pairs, seed)


@pytest.mark.parametrize("K,Vmax,F,B,seed", CASES, ids=[f"K{c[0]}-V{c[1]}-F{c[2]}-B{c[3]}" for c in CASES])
def test_every_pair_equals_its_single_object_call(K, Vmax, F, B, seed):
    """Ragged objects (1 .. Vmax views), pairs in mixed order with repeated frames and objects: per pair the outputs bit-equal
    to boxes_from_matches on its object alone, and under the trace hook the same samples, counts, models and loop length."""
    rng = np.random.default_rng(seed)
    vpo = [int(v) for v in rng.integers(1, Vmax + 1, K)]
    vpo[int(rng.integers(0, K))] = Vmax
    pairs = [(int(rng.integers(0, F)), int(rng.integers(0, K))) for _ in range(B)]
    pairs[0] = pairs[-1]                                                        # a repeated pair
    refs, query, m0, vf, vc, fi = _scene(rng, vpo, F, pairs)
    with Trace(B) as tr:
        out = detect.boxes_from_matches_objects(refs, vf, vc, query, fi, m0, HW)
    out32 = detect.boxes_from_matches_objects(refs, vf.cpu(), vc.cpu().long(), query, fi.cpu().tolist(), m0.to(torch.int32), HW)
    for k in out:
        assert torch.equal(out[k], out32[k]), k
    status = out["status"].tolist()
    for b in range(B):
        with Trace(1) as one_tr:
            one = _single(refs, query, m0, vf, vc, fi, b)
        for k in out:
            assert out[k][b].cpu().numpy().tobytes() == one[k][0].cpu().numpy().tobytes(), (b, k)
        assert torch.equal(tr.samples[b], one_tr.samples[0]) and torch.equal(tr.counts[b], one_tr.counts[0]), b
        assert tr.models[b].cpu().numpy().tobytes() == one_tr.models[0].cpu().numpy().tobytes(), b
    print(f"K={K} B={B}: status {[status.count(s) for s in (0, 1, 2)]} (0 / 1 / 2)")
    assert B == 1 or status.count(1) > 0


@pytest.fixture(scope="module")
def golden():
    g = dict(np.load(os.path.join(GOLDEN_DIR, "pnp_detect_cases.npz"), allow_pickle=False))
    scenes = []
    for s in range(int(g["n_scenes"])):
        H, W, seed = (int(v) for v in g[f"s{s}_frame"])
        qs = [{k: g[f"s{s}_q{q}_{k}"] for k in ("keypoints", "matches0", "bbox", "crop_size", "image_crop", "K_crop")}
              for q in range(int(g[f"s{s}_n_queries"]))]
        scenes.append({"frame": torch.from_numpy(cr.synthetic_frame(H, W, seed)).to(DEV), "hw": (H, W), "K": g[f"s{s}_K"], "queries": qs,
                       "ref": {k: g[f"s{s}_ref_{k}"] for k in ("keypoints", "counts", "sizes")}})
    return scenes


def test_goldens_regrouped_as_objects(golden):
    """Each golden scene's views become an object of one table shared with two decoy objects; each query is a frame of key
    points and the scene's frame is cropped by index.  The boxes and crops are the reference detector's."""
    rng = np.random.default_rng(5)
    for sc in golden:
        decoys = [(np.zeros((n, 30, 2), np.float32), np.full(n, 30), np.full((n, 2), 200)) for n in (3, 2)]
        kp_s = sc["ref"]["keypoints"]
        cap = max(kp_s.shape[1], 30)
        parts = [decoys[0], (kp_s, sc["ref"]["counts"], sc["ref"]["sizes"]), decoys[1]]
        kp = np.concatenate([np.pad(p[0], ((0, 0), (0, cap - p[0].shape[1]), (0, 0))) for p in parts])
        refs = {"keypoints": torch.from_numpy(kp).to(DEV), "counts": torch.from_numpy(np.concatenate([p[1] for p in parts])).to(DEV, torch.int32),
                "sizes": torch.from_numpy(np.concatenate([p[2] for p in parts])).to(DEV, torch.int32)}
        V = len(sc["ref"]["counts"])
        for S in sorted({int(q["crop_size"]) for q in sc["queries"]}):
            qs = [q for q in sc["queries"] if int(q["crop_size"]) == S]
            order = rng.permutation(len(qs))
            qcap = max(len(q["keypoints"]) for q in qs)
            qkp = np.zeros((len(qs), qcap, 2), np.float32)
            for r, q in enumerate(qs):
                qkp[r, :len(q["keypoints"])] = q["keypoints"]
            query = {"keypoints": torch.from_numpy(qkp).to(DEV), "counts": torch.tensor([len(q["keypoints"]) for q in qs], dtype=torch.int32, device=DEV)}
            m0 = np.full((len(qs), V, cap), -1, np.int64)
            for b, r in enumerate(order):
                m0[b, :, :kp_s.shape[1]] = qs[r]["matches0"]
            m0 = torch.from_numpy(m0).to(DEV)
            first = torch.full((len(qs),), 3, dtype=torch.int32, device=DEV)
            count = torch.full((len(qs),), V, dtype=torch.int32, device=DEV)
            qi = torch.from_numpy(order.astype(np.int32)).to(DEV)
            out = detect.boxes_from_matches_objects(refs, first, count, query, qi, m0, sc["hw"])
            frames = sc["frame"][None].expand(len(qs), -1, -1)                   # query row r is frame r (all the same image)
            bbox, image, K_crop = detect.detect_from_matches_objects(frames, qi, torch.from_numpy(sc["K"]).to(DEV), refs, first, count, query, m0, S)
            assert torch.equal(bbox, out["box"])
            shared = crop.crop_frames(sc["frame"][None], bbox, torch.from_numpy(sc["K"]).to(DEV), S, frame_index=torch.zeros_like(qi))
            assert torch.equal(shared["image"], image) and torch.equal(shared["K_crop"], K_crop)
            img = image.cpu().numpy()
            for b, r in enumerate(order):
                q = qs[r]
                assert bbox[b].tolist() == q["bbox"].tolist(), (b, bbox[b], q["bbox"])
                assert np.array_equal(img[b, 0], q["image_crop"].astype(np.float32) / 255)
                np.testing.assert_allclose(K_crop[b].cpu().numpy(), q["K_crop"], rtol=1e-12, atol=0)


def test_quirks_per_pair(golden):
    """Per pair: no view with 6 matches, the winner without an affine (empty box), int32 and int64 matches0, view_count 1 and
    256, and the pairs whose view range or query row is out of bounds."""
    sc = golden[1]
    kp = torch.from_numpy(sc["ref"]["keypoints"]).to(DEV).clone()
    V, cap = kp.shape[:2]
    n = int(sc["ref"]["counts"][2])
    kp[2, :n] = kp[2, 0]                                                        # view 2's points all coincide
    big = 256
    bkp = torch.rand(big, cap, 2, device=DEV) * 300
    refs = {"keypoints": torch.cat([kp, bkp]),
            "counts": torch.cat([torch.from_numpy(sc["ref"]["counts"]).long(), torch.full((big,), 50)]).to(DEV, torch.int32),
            "sizes": torch.cat([torch.from_numpy(sc["ref"]["sizes"]).long(), torch.full((big, 2), 300)]).to(DEV, torch.int32)}
    qkp = torch.rand(2, 80, 2, device=DEV) * 300
    query = {"keypoints": qkp, "counts": torch.tensor([80, 40], dtype=torch.int32, device=DEV)}
    # (first, count, query row): the golden object, the 256-view object, its last view alone, and four out-of-bounds pairs
    table = [(0, V, 0), (0, V, 1), (0, V, 0), (V, big, 1), (V + big - 1, 1, 0), (V + big - 1, 2, 0), (0, 0, 0), (-1, 1, 0), (0, V, 2)]
    B = len(table)
    m0 = torch.full((B, big, cap), -1, dtype=torch.int64, device=DEV)
    m0[0, 2, :20] = torch.arange(20)                                            # 20 matches of the coincident view: no model
    m0[1, 1, :5] = torch.arange(5)                                              # 5 and 5: below 6
    m0[1, 3, 3:8] = torch.arange(5)
    m0[2, 0, :30] = torch.arange(40, 70)                                        # row 0 has 80 points: these count
    m0[3, 255, :30] = torch.arange(30)                                          # the 256th view wins
    m0[3, 100, :10] = torch.arange(10)
    m0[4, 0, :12] = torch.arange(12)
    m0[4, 1:] = 7                                                               # never read: one view
    vf, vc, qi = (torch.tensor([t[k] for t in table], dtype=torch.int32, device=DEV) for k in range(3))
    out = detect.boxes_from_matches_objects(refs, vf, vc, query, qi, m0, sc["hw"])
    out32 = detect.boxes_from_matches_objects(refs, vf, vc, query, qi, m0.to(torch.int32), sc["hw"])
    for k in out:
        assert torch.equal(out[k], out32[k]), k
    assert out["status"][:3].tolist() == [0, 2, 1] and out["view"][:5].tolist() == [2, 0, 0, 255, 0]
    assert out["n_matches"][:5].tolist() == [20, 0, 30, 30, 12]
    assert out["box"][:2].tolist() == [[0, 0, 0, 0], [0, 0, 640, 360]] and not out["affine"][:2].any()
    for b in range(5):
        f, c, q = table[b]
        one = detect.boxes_from_matches({k: v[f:f + c] for k, v in refs.items()}, {k: v[q:q + 1] for k, v in query.items()}, m0[b:b + 1, :c],
                                        sc["hw"])
        for k in out:
            assert out[k][b].cpu().numpy().tobytes() == one[k][0].cpu().numpy().tobytes(), (b, k)
    bad = slice(5, B)
    assert out["status"][bad].tolist() == [0] * 4 and out["view"][bad].tolist() == [0] * 4 and out["n_matches"][bad].tolist() == [0] * 4
    assert not out["box"][bad].any() and not out["affine"][bad].any()
    big_index = detect.boxes_from_matches_objects(refs, vf.long() + (1 << 32), vc, query, qi, m0, sc["hw"])   # no wrap into range
    assert big_index["status"].tolist() == [0] * B


def _frames(rng, F, H, W):
    base = torch.from_numpy(rng.integers(0, 256, (2 * F, H, W + 13), dtype=np.uint8)).to(DEV)
    return base[::2, :, 5:5 + W]                                                # frame and row strides of their own


def test_indexed_crop_equals_the_crop_of_gathered_frames():
    rng = np.random.default_rng(11)
    F, H, W, S = 5, 240, 320, 64
    frames = _frames(rng, F, H, W)
    index = torch.tensor([3, 0, 3, 4, -1, 5, 1, 1, 2, 3, 1 << 20], dtype=torch.int64)
    B = len(index)
    x0, y0 = rng.integers(-40, 300, B), rng.integers(-40, 220, B)
    boxes = np.stack([x0, y0, x0 + rng.integers(1, 200, B), y0 + rng.integers(1, 150, B)], 1).astype(np.int32)
    boxes[2] = [10, 10, 10, 40]                                                 # a rejected box
    boxes = torch.from_numpy(boxes).to(DEV)
    K = torch.from_numpy(np.stack([np.array([[300.0 + b, 0, 160], [0, 310.0, 120 + b], [0, 0, 1]]) for b in range(B)])).to(DEV)
    got = crop.crop_frames(frames, boxes, K, S, frame_index=index.to(DEV))
    got32 = crop.crop_frames(frames, boxes, K, S, frame_index=index.clamp(-1, F).to(torch.int32).tolist())
    valid = (index >= 0) & (index < F)
    gathered = frames[index.clamp(0, F - 1).to(DEV)]
    want = crop.crop_frames(gathered, boxes, K, S)
    for k in got:
        assert torch.equal(got[k], got32[k]), k
    for b in range(B):
        if valid[b]:
            for k in got:
                assert got[k][b].cpu().numpy().tobytes() == want[k][b].cpu().numpy().tobytes(), (b, k)
        else:
            assert int(got["status"][b]) == 0 and not got["image"][b].any() and not got["trans"][b].any(), b
            assert torch.equal(got["K_crop"][b], K[b]), b
    assert got["status"].tolist() == [1, 1, 0, 1, 0, 0, 1, 1, 1, 1, 0]
    one = crop.crop_frames(frames[3:4].expand(4, -1, -1), boxes[[0, 2, 3, 9]], K[[0, 2, 3, 9]], S)   # the stride-0 form agrees
    sel = crop.crop_frames(frames, boxes[[0, 2, 3, 9]], K[[0, 2, 3, 9]], S, frame_index=[3, 3, 3, 3])
    for k in one:
        assert torch.equal(one[k], sel[k]), k


def test_previous_pose_detect_per_object():
    """previous_pose_detect for three objects in two frames equals it on the gathered frames."""
    rng = np.random.default_rng(3)
    frames = _frames(rng, 2, 480, 640)
    K = torch.tensor([[500.0, 0, 320], [0, 500.0, 240], [0, 0, 1]], dtype=torch.float64, device=DEV)
    pose = torch.zeros(3, 3, 4, dtype=torch.float64, device=DEV)
    pose[:, :, :3] = torch.eye(3, dtype=torch.float64)
    pose[:, :, 3] = torch.tensor([[0.05, 0.0, 0.8], [-0.1, 0.05, 1.0], [0.0, -0.05, 0.6]], dtype=torch.float64)
    bbox3d = torch.from_numpy(np.array([[x, y, z] for x in (-0.05, 0.05) for y in (-0.04, 0.04) for z in (-0.03, 0.03)])).to(DEV)
    index = torch.tensor([1, 0, 1], dtype=torch.int32, device=DEV)
    got = crop.previous_pose_detect(frames, K, pose, bbox3d, 128, frame_index=index)
    want = crop.previous_pose_detect(frames[index.long()], K, pose, bbox3d, 128)
    for g, w in zip(got, want):
        assert torch.equal(g, w)


class CountingExtractor:
    """Reference views carry their tag in pixel (0, 0); frames are the [F, 1, H, W] calls.  Key points from tables."""

    def __init__(self, view_kp, frame_kp, hw):
        self.view_kp, self.frame_kp, self.hw, self.frame_calls = view_kp, frame_kp, hw, 0

    def _out(self, kps):
        return {"keypoints": kps, "scores": [torch.ones(len(k), device=DEV) for k in kps], "descriptors": [torch.zeros(256, len(k), device=DEV) for k in kps]}

    def forward(self, inp):
        if tuple(inp.shape[2:]) == self.hw:
            self.frame_calls += 1
            assert inp.shape[0] == len(self.frame_kp)
            return self._out(list(self.frame_kp))
        return self._out([self.view_kp[int(round(float(inp[0, 0, 0, 0]) * 255))]])


class TableMatcher(torch.nn.Module):
    """matches0 of (view, frame), told apart by their key-point counts (distinct by construction)."""

    def __init__(self, table):
        super().__init__()
        self.table, self.calls = table, 0

    def forward(self, data):
        self.calls += 1
        return {"matches0": self.table[(data["keypoints0"].shape[1], data["keypoints1"].shape[1])][None]}


def test_object_detectors_equal_single_object_detectors():
    rng = np.random.default_rng(8)
    H, W, F, S = 360, 480, 3, 64
    vpo = [3, 1, 4, 2]
    tags = np.cumsum([0] + vpo)
    n_view = [40 + 7 * g for g in range(tags[-1])]
    n_frame = [300 + 11 * f for f in range(F)]
    view_kp = [torch.from_numpy(rng.uniform(0, 200, (n, 2)).astype(np.float32)).to(DEV) for n in n_view]
    frame_kp = [rng.uniform(0, [W, H], (n, 2)).astype(np.float32) for n in n_frame]
    table = {}
    for g, n in enumerate(n_view):
        for f, nf in enumerate(n_frame):
            k = int(rng.integers(0, 60))
            m = np.full(n, -1, np.int64)
            idx = rng.choice(n, min(k, n), replace=False)
            m[idx] = rng.choice(nf, len(idx), replace=False)
            if k > 12:                                                          # half of them on a planted similarity
                a, s = rng.uniform(-0.5, 0.5), rng.uniform(0.8, 1.5)
                R = s * np.array([[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]])
                h = idx[: len(idx) // 2]
                frame_kp[f][m[h]] = view_kp[g][h].cpu().numpy() @ R.T + rng.uniform(50, 200, 2)
            table[(n, nf)] = torch.from_numpy(m).to(DEV)
    frame_kp = [torch.from_numpy(k).to(DEV) for k in frame_kp]
    ext = CountingExtractor(view_kp, frame_kp, (H, W))
    matcher = TableMatcher(table)
    images = []
    for o, nv in enumerate(vpo):
        imgs = [np.zeros((200 + 10 * v, 220), np.uint8) for v in range(nv)]
        for v in range(nv):
            imgs[v][0, 0] = tags[o] + v
        images.append(imgs)
    singles = [detect.LocalFeatureObjectDetector(ext, matcher, imgs, crop_size=S) for imgs in images]
    multi = detect.ObjectDetectors(ext, matcher, crop_size=S)
    ids = [multi.add_object(imgs) for imgs in images]
    frames = torch.from_numpy(rng.integers(0, 256, (F, H, W), dtype=np.uint8)).to(DEV)
    K = torch.tensor([[400.0, 0, 240], [0, 400.0, 180], [0, 0, 1]], dtype=torch.float64, device=DEV)
    want = [s.detect(frames, K) for s in singles]
    pairs = [(2, ids[1]), (0, ids[0]), (0, ids[2]), (1, ids[3]), (2, ids[0]), (0, ids[0]), (1, ids[2]), (2, ids[3])]
    ext.frame_calls, matcher.calls = 0, 0
    bbox, image, K_crop = multi.detect(frames, K, pairs)
    assert ext.frame_calls == 1 and matcher.calls == sum(vpo[ids.index(o)] for _, o in pairs)
    for b, (f, o) in enumerate(pairs):
        w = want[ids.index(o)]
        assert torch.equal(bbox[b], w[0][f]) and torch.equal(image[b], w[1][f]) and torch.equal(K_crop[b], w[2][f]), (b, f, o)
    assert len({tuple(v) for v in bbox.tolist()}) > 2
    multi.remove_object(ids[1])
    with pytest.raises(ValueError):
        multi.detect(frames, K, [(0, ids[1])])
    with pytest.raises(ValueError):
        multi.detect(frames, K, [(3, ids[0])])
    again = multi.detect(frames, K, pairs[1:3])
    for b in range(2):
        assert torch.equal(again[0][b], bbox[b + 1]) and torch.equal(again[1][b], image[b + 1])


def test_closed_loop_three_objects_in_one_frame():
    """Three planted objects in one 720 x 960 frame: boxes from planted matches (30 % wrong), the crops, match_objects on the
    planted descriptors of the crops, then poses_from_matches_objects.  Every object within 1 cm and 1 degree."""
    rng = np.random.default_rng(4)
    H, W, S, N = 720, 960, 512, 1024
    m = GATsSuperGlue(dict(synthetic.DEFAULT_HPARAMS)).eval()
    m.load_state_dict({k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in synthetic.make_state_dict(0).items()})
    m = m.cuda()
    specs = [(4, 1500, 501, (40, 60)), (5, 1200, 502, (380, 330)), (6, 1800, 503, (660, 120))]
    scenes = [synthetic.make_planted_scene(o, [f], N, M) for o, M, f, _ in specs]
    ids = [m.add_object(torch.from_numpy(s["desc3d"]).cuda(), torch.from_numpy(s["desc2d_db"]).cuda()) for s in scenes]
    w = 256                                                                     # each object's box in the frame: w x w
    kp_f, K_f = [], []
    for s, (_, _, _, (x0, y0)) in zip(scenes, specs):
        kp_f.append(s["keypoints2d"][0].astype(np.float64) * (w / S) + np.array([x0, y0]))
        Kc = s["K"][0]
        K_f.append(np.array([[Kc[0, 0] * w / S, 0, Kc[0, 2] * w / S + x0], [0, Kc[1, 1] * w / S, Kc[1, 2] * w / S + y0], [0, 0, 1]]))
    qkp = np.concatenate(kp_f).astype(np.float32)[None]
    refs = {"keypoints": torch.from_numpy(np.stack([s["keypoints2d"][0] for s in scenes])).to(DEV),      # each view: the object's crop
            "counts": torch.full((3,), N, dtype=torch.int32, device=DEV), "sizes": torch.full((3, 2), S, dtype=torch.int32, device=DEV)}
    m0 = np.stack([np.arange(N) + o * N for o in range(3)])[:, None]
    wrong = rng.random(m0.shape) < 0.3
    m0[wrong] = rng.integers(0, 3 * N, int(wrong.sum()))
    query = {"keypoints": torch.from_numpy(qkp).to(DEV), "counts": torch.tensor([3 * N], dtype=torch.int32, device=DEV)}
    frames = torch.from_numpy(rng.integers(0, 256, (1, H, W), dtype=np.uint8)).to(DEV)
    zeros = torch.zeros(3, dtype=torch.int32, device=DEV)
    ones = torch.ones(3, dtype=torch.int32, device=DEV)
    Kd = torch.from_numpy(np.stack(K_f)).to(DEV)
    boxes = detect.boxes_from_matches_objects(refs, torch.arange(3, dtype=torch.int32, device=DEV), ones, query, zeros, torch.from_numpy(m0).to(DEV),
                                              (H, W))
    assert boxes["status"].tolist() == [1, 1, 1]
    for o, (_, _, _, (x0, y0)) in enumerate(specs):
        assert np.abs(np.array(boxes["box"][o].tolist()) - [x0, y0, x0 + w, y0 + w]).max() <= 1, boxes["box"][o]
    bbox, image, K_crop = detect.detect_from_matches_objects(frames, zeros, Kd, refs, torch.arange(3, dtype=torch.int32, device=DEV), ones, query,
                                                             torch.from_numpy(m0).to(DEV), S)
    assert torch.equal(bbox, boxes["box"])
    tr = crop.crop_frames(frames, bbox, Kd, S, frame_index=zeros)["trans"].cpu().numpy()
    kp_c = []
    for o in range(3):
        homo = [np.concatenate([tr[o, s], [[0, 0, 1.0]]]) for s in (0, 1)]
        kp_c.append((homo[1] @ homo[0] @ np.concatenate([kp_f[o], np.ones((N, 1))], axis=1).T).T[:, :2])
    q = torch.from_numpy(np.stack([s["descriptors2d"][0] for s in scenes])).cuda()
    out = m.match_objects(q, ids, return_conf=False)
    kp3 = {ids[o]: torch.from_numpy(scenes[o]["keypoints3d"]).cuda() for o in range(3)}
    res = pnp.poses_from_matches_objects(K_crop, torch.from_numpy(np.stack(kp_c)).to(DEV, torch.float32), kp3, ids, out["matches0"],
                                         out["matching_scores0"])
    rot, trans = pnp.pose_errors(res["pose"], torch.from_numpy(np.stack([s["pose_gt"][0] for s in scenes])).to(DEV))
    print("rot err deg", rot.tolist(), "trans err cm", trans.tolist())
    assert float(rot.max()) < 1.0 and float(trans.max()) < 1.0


def test_side_stream_and_every_output_written(monkeypatch):
    rng = np.random.default_rng(9)
    pairs = [(1, 0), (0, 2), (1, 1), (0, 0), (1, 2)]
    refs, query, m0, vf, vc, fi = _scene(rng, [4, 2, 6], 2, pairs)
    want = detect.boxes_from_matches_objects(refs, vf, vc, query, fi, m0, HW)
    frames = _frames(rng, 2, *HW)
    K = torch.eye(3, dtype=torch.float64, device=DEV)
    want_c = detect.detect_from_matches_objects(frames, fi, K, refs, vf, vc, query, m0, 64)
    torch.cuda.synchronize()
    s = torch.cuda.Stream(DEV)
    with torch.cuda.stream(s):
        m2 = m0 + 0
        got = detect.boxes_from_matches_objects(refs, vf, vc, query, fi, m2, HW)
        got_c = detect.detect_from_matches_objects(frames, fi, K, refs, vf, vc, query, m2, 64)
    s.synchronize()
    for k in want:
        assert torch.equal(got[k], want[k]), k
    for g, w in zip(got_c, want_c):
        assert torch.equal(g, w)
    made = []
    real_empty = torch.empty

    def poisoned(*a, **kw):
        t = real_empty(*a, **kw)
        t.view(torch.uint8).fill_(0xFF) if t.numel() else None
        made.append(t)
        return t

    vf_bad = vf.clone()
    vf_bad[2] = 100                                                             # one pair out of bounds
    index = torch.tensor([0, 1, 7, 1, 0], dtype=torch.int32, device=DEV)        # one frame out of bounds

    def run():
        out = detect.boxes_from_matches_objects(refs, vf_bad, vc, query, fi, m0, HW)
        return out, crop.crop_frames(frames, out["box"], K, 64, frame_index=index)

    clean, clean_c = run()
    monkeypatch.setattr(torch, "empty", poisoned)
    out, res = run()
    monkeypatch.undo()
    assert len(made) >= 9
    for k in out:
        assert torch.equal(out[k], clean[k]), k
    for k in res:
        assert torch.equal(res[k], clean_c[k]), k
    for k, v in list(out.items()) + list(res.items()):
        if v.dtype.is_floating_point:
            assert not torch.isnan(v).any(), k
    assert not (out["status"] == -1).any() and not (out["view"] == -1).any() and not (res["status"] == -1).any()
    assert int(out["status"][2]) == 0 and int(res["status"][2]) == 0


def test_argument_mistakes_raise():
    rng = np.random.default_rng(2)
    pairs = [(0, 0), (1, 1)]
    refs, query, m0, vf, vc, fi = _scene(rng, [3, 2], 2, pairs)
    call = lambda **kw: detect.boxes_from_matches_objects(**{**dict(refs=refs, view_first=vf, view_count=vc, query=query, query_index=fi,  # noqa: E731
                                                                    matches0=m0, query_size=HW), **kw})
    for bad in (dict(matches0=m0.float()), dict(matches0=m0[0]), dict(matches0=m0[:, :, :5]), dict(matches0=torch.zeros(2, 257, m0.shape[2], dtype=torch.int64, device=DEV)),
                dict(view_first=vf[:1]), dict(view_count=vc.float()), dict(query_index=[0, 1, 0]), dict(query_size=(0, 5)),
                dict(refs={**refs, "sizes": refs["sizes"][:2]}), dict(query={**query, "counts": query["counts"][:1]})):
        with pytest.raises(ValueError):
            call(**bad)
    with pytest.raises(RuntimeError, match="no CPU path"):
        call(matches0=m0.cpu())
    frames = _frames(rng, 2, *HW)
    K = torch.eye(3, dtype=torch.float64, device=DEV)
    for bad in (lambda: detect.detect_from_matches_objects(frames[:1], fi, K, refs, vf, vc, query, m0),
                lambda: detect.detect_from_matches_objects(frames, fi, K, refs, vf, vc, query, m0, crop_size=60),
                lambda: detect.detect_from_matches_objects(frames, fi, K[None].expand(3, 3, 3), refs, vf, vc, query, m0),
                lambda: crop.crop_frames(frames, torch.zeros(2, 4, dtype=torch.int32, device=DEV), K, 64, frame_index=[0, 1, 1]),
                lambda: crop.crop_frames(frames, torch.zeros(2, 4, dtype=torch.int32, device=DEV), K, 64, frame_index=[0.0, 1.0]),
                lambda: crop.crop_frames(frames, torch.zeros(0, 4, dtype=torch.int32, device=DEV), K, 64, frame_index=[])):
        with pytest.raises(ValueError):
            bad()
