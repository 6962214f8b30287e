"""sfm.postprocess on the device against the reference's output (tests/golden/pnp_sfm_cases.npz) and against the numpy model
(tests/sfm_reference.py) on generated models: every count, id and order exactly, every value bit for bit."""
import os

import numpy as np
import pytest
import torch

from onepose_b200 import _lib, sfm
from tests import sfm_reference as sr

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pnp_sfm_cases.npz")


def _features(seed, F, D, cap, counts, dev):
    sc, de = sr.features(seed, F, D, cap)
    sc, de = sc.copy(), de.copy()
    for f, n in enumerate(counts):                     # garbage past each image's count: never read
        sc[f, n:] = np.nan
        de[f, :, n:] = np.nan
    return {"scores": torch.from_numpy(sc).to(dev), "descriptors": torch.from_numpy(de).to(dev)}, sr.features(seed, F, D, cap)


def _check(out, m):
    assert out["track_length"] == m["track_length"]
    o = out["group_offsets"]
    groups = [out["group_ids"][o[g]:o[g + 1]] for g in range(len(o) - 1)]
    assert len(groups) == len(m["groups"]) and all(np.array_equal(a, b) for a, b in zip(groups, m["groups"]))
    assert np.array_equal(out["idxs"], m["idxs"]) and out["idxs"].dtype == np.int64
    for k in ("keypoints3d", "descriptors3d", "scores3d", "descriptors3d_collect", "scores3d_collect"):
        v = out[k].cpu().numpy()
        assert v.dtype == np.float64 and v.shape == m[k].shape, k
        assert np.array_equal(v, m[k]), k


@pytest.fixture(scope="module")
def golden(tmp_path_factory):
    z = dict(np.load(GOLDEN))
    d = tmp_path_factory.mktemp("model")
    z["points3d_bin"].tofile(d / "points3D.bin")
    z["images_bin"].tofile(d / "images.bin")
    z["dir"] = d
    return z


def test_fixture_matches_the_reference(golden):
    z = golden
    names = list(z["names"])
    images = dict(sfm.read_images_bin(z["dir"] / "images.bin"))
    counts = [len(images[n]) for n in names]
    feats, _ = _features(int(z["seed"]), len(names), int(z["D"]), int(z["cap"]), counts, "cuda")
    out = sfm.postprocess(z["dir"], z["dir"], feats, z["corners"], int(z["max_num_kp3d"]), float(z["dist_threshold"]), image_names=names)
    assert out["track_length"] == int(z["track_length"])
    assert np.array_equal(out["group_offsets"], z["group_offsets"]) and np.array_equal(out["group_ids"], z["group_ids"])
    assert np.array_equal(out["idxs"], z["idxs"])
    assert np.array_equal(out["keypoints3d"].cpu().numpy(), z["keypoints3d"])
    assert np.array_equal(out["descriptors3d"].cpu().numpy(), z["descriptors3d"])
    assert np.array_equal(out["scores3d"].cpu().numpy(), z["scores3d"])
    sc, de = sr.features(int(z["seed"]), len(names), int(z["D"]), int(z["cap"]))
    obs = z["obs"]
    assert np.array_equal(out["descriptors3d_collect"].cpu().numpy(), de[obs[:, 0], :, obs[:, 1]].astype(np.float64).T)
    assert np.array_equal(out["scores3d_collect"].cpu().numpy()[:, 0], sc[obs[:, 0], obs[:, 1]].astype(np.float64))


def _generated(seed, P, F, cap, dense=False):
    rng = np.random.default_rng(seed)
    corners = np.array([[0, 1, 0], [1, 1, 0], [1, 1, 1], [0, 1, 1], [0, 0, 0], [1, 0, 0], [1, 0, 1], [0, 0, 1]], np.float64) * 0.3 + 0.01
    if dense:                                          # clusters a few tenths of a millimetre wide
        centres = rng.uniform(-0.02, 0.33, (max(P // 6, 1), 3))
        xyz = centres[rng.integers(0, len(centres), P)] + rng.normal(scale=3e-4, size=(P, 3))
    else:                                              # a quarter outside the box, along one axis
        xyz = rng.uniform(0.02, 0.30, (P, 3))
        out = np.nonzero(rng.random(P) < 0.25)[0]
        out = out[out >= 2]                            # the one- and two-point models keep their points
        xyz[out, rng.integers(0, 3, len(out))] += 0.35
    ids = rng.choice(np.arange(P * 5 + 10, dtype=np.int64), P, replace=False) + (np.int64(1) << 40) * rng.integers(0, 2, P)
    lens = rng.integers(2, 60, P).astype(np.int64)
    obs = [[] for _ in range(F)]
    for i in rng.permutation(P):                       # every point seen once or twice, never past an image's capacity
        for f in rng.choice(F, min(F, 1 + int(rng.integers(0, 2))), replace=False):
            if len(obs[f]) < cap - 1:
                obs[f].append(int(ids[i]))
    images = []
    for f in range(F):
        p = np.array(obs[f] + [-1] * int(rng.integers(0, 3)), np.int64)[:cap]
        images.append((f"{f}.png", p[rng.permutation(len(p))]))
    seen = set(np.concatenate([p for _, p in images]).tolist())
    keep = np.array([int(q) in seen for q in ids])     # a point no image observes would be the reference's KeyError
    return ids[keep], xyz[keep], lens[keep], images, corners


CASES = [  # P, F, cap, D, max_num_kp3d relative to P ("below", "at", "above"), dense
    (1, 1, 4, 1, "above", False),
    (2, 2, 4, 32, "at", False),
    (37, 5, 64, 257, "below", True),
    (2500, 40, 512, 256, "below", False),
    (2500, 30, 1024, 32, "above", True),
    (50000, 300, 4096, 32, "above", False),
    (50000, 120, 2048, 1, "below", False),
]


@pytest.mark.parametrize("P,F,cap,D,rel,dense", CASES)
def test_device_equals_the_model(P, F, cap, D, rel, dense):
    ids, xyz, lens, images, corners = _generated(P * 7 + D, P, F, cap, dense)
    n = len(ids)
    mx = {"below": max(n // 3, 0), "at": n, "above": n + 5}[rel]
    counts = [len(p) for _, p in images]
    feats, (sc, de) = _features(P + D, F, D, cap, counts, "cuda")
    m = sr.postprocess(ids, xyz, lens, [p for _, p in images], sc, de, corners, mx, 1e-3)
    out = sfm.postprocess((ids, xyz, lens), images, feats, corners, mx, 1e-3)
    _check(out, m)


def test_save_anno_writes_the_reference_files(golden, tmp_path):
    z = golden
    names = list(z["names"])
    images = dict(sfm.read_images_bin(z["dir"] / "images.bin"))
    feats, _ = _features(int(z["seed"]), len(names), int(z["D"]), int(z["cap"]), [len(images[n]) for n in names], "cuda")
    out = sfm.postprocess(z["dir"], z["dir"], feats, z["corners"], int(z["max_num_kp3d"]), image_names=names)
    sfm.save_anno(tmp_path, out)
    avg, clt = np.load(tmp_path / "anno_3d_average.npz"), np.load(tmp_path / "anno_3d_collect.npz")
    idxs = np.load(tmp_path / "idxs.npy")
    n, total, D = len(z["idxs"]), int(z["idxs"].sum()), int(z["D"])
    assert sorted(avg.files) == sorted(clt.files) == ["descriptors3d", "keypoints3d", "scores3d"]
    assert avg["keypoints3d"].shape == (n, 3) and avg["descriptors3d"].shape == (D, n) and avg["scores3d"].shape == (n, 1)
    assert clt["keypoints3d"].shape == (n, 3) and clt["descriptors3d"].shape == (D, total) and clt["scores3d"].shape == (total, 1)
    assert all(a[k].dtype == np.float64 for a in (avg, clt) for k in a.files) and idxs.dtype == np.int64
    assert np.array_equal(avg["descriptors3d"], z["descriptors3d"]) and np.array_equal(avg["scores3d"], z["scores3d"])
    assert np.array_equal(clt["keypoints3d"], z["keypoints3d"]) and np.array_equal(idxs, z["idxs"])


def test_results_on_the_callers_stream(golden):
    z = golden
    names = list(z["names"])
    images = dict(sfm.read_images_bin(z["dir"] / "images.bin"))
    src, _ = _features(int(z["seed"]), len(names), int(z["D"]), int(z["cap"]), [len(images[n]) for n in names], "cuda")
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(200_000_000)                 # the caller's stream is busy, then makes the features: the steps must wait
        feats = {k: v * 1.0 for k, v in src.items()}   # queued behind the sleep; the uploads in postprocess do not block the host
        out = sfm.postprocess(z["dir"], z["dir"], feats, z["corners"], int(z["max_num_kp3d"]), image_names=names)
        avg = out["descriptors3d"].cpu().numpy()
        clt = out["descriptors3d_collect"].cpu().numpy()
    assert np.array_equal(avg, z["descriptors3d"])
    sc, de = sr.features(int(z["seed"]), len(names), int(z["D"]), int(z["cap"]))
    assert np.array_equal(clt, de[z["obs"][:, 0], :, z["obs"][:, 1]].astype(np.float64).T)


def _small():
    ids = np.array([3, 1], np.int64)
    xyz = np.array([[0.1, 0.1, 0.1], [0.2, 0.2, 0.2]])
    lens = np.array([3, 3], np.int64)
    images = [("a", np.array([1, 3, -1], np.int64))]
    corners = np.array([[0, 1, 0], [1, 1, 0], [1, 1, 1], [0, 1, 1], [0, 0, 0], [1, 0, 0], [1, 0, 1], [0, 0, 1]], np.float64)
    feats = {"scores": torch.ones(1, 4, device="cuda"), "descriptors": torch.ones(1, 8, 4, device="cuda")}
    return (ids, xyz, lens), images, feats, corners


def test_refusals_name_the_entry_point():
    pts, images, feats, corners = _small()
    sfm.postprocess(pts, images, feats, corners)
    bad = [
        ({"scores": feats["scores"].double(), "descriptors": feats["descriptors"]}, "opb_sfm_gather_features"),
        ({"scores": feats["scores"].cpu(), "descriptors": feats["descriptors"]}, "opb_sfm_gather_features"),
        ({"scores": feats["scores"], "descriptors": feats["descriptors"][0]}, "opb_sfm_gather_features"),
        ({"scores": feats["scores"], "descriptors": torch.ones(1, 8, 5, device="cuda")}, "opb_sfm_gather_features"),
        # channel-last descriptors [F, cap, D]: D and cap swapped
        ({"scores": feats["scores"], "descriptors": torch.ones(1, 4, 8, device="cuda")}, "opb_sfm_gather_features"),
        ({"scores": feats["scores"], "descriptors": torch.ones(2, 8, 4, device="cuda")}, "opb_sfm_gather_features"),
        ({"scores": feats["scores"][:, :2], "descriptors": feats["descriptors"][:, :, :2]}, "opb_sfm_gather_observations"),
    ]
    for f, name in bad:
        with pytest.raises(ValueError, match=name):
            sfm.postprocess(pts, images, f, corners)
    with pytest.raises(ValueError, match="opb_sfm_gather_observations: point 3 "):
        sfm.postprocess(pts, [("a", np.array([1, -1, -1], np.int64))], feats, corners)
    with pytest.raises(ValueError):
        sfm.postprocess(pts, images, feats, corners, max_num_kp3d=-1)
    with pytest.raises(ValueError):
        sfm.postprocess((pts[0][:0], pts[1][:0], pts[2][:0]), images, feats, corners)
    with pytest.raises(ValueError, match="no point passes"):
        sfm.postprocess(pts, images, feats, corners + 5.0)
    lib = _lib.load()
    x = torch.zeros(16, dtype=torch.int64, device="cuda")
    for name, args in (("opb_sfm_filter_points", (x, x, x, 2, -1, x, x, 1 << 20, x, x, x, x)),
                       ("opb_sfm_merge_points", (x, x, x, 2, 0.0, x, 1 << 20, x, x, x, x, x, x, x)),
                       ("opb_sfm_gather_features", (x, 5, 1, 4, 0, x, x, x, x))):
        with pytest.raises(_lib.OpbError, match=name):
            _lib.call(x.device, name, *args)


def _close_tail(P):
    """P points inside the box, every one kept (max_num_kp3d >= P); the two largest ids are 0.5 mm apart, so the last rows the
    merge walks form a group after every other point is in one."""
    rng = np.random.default_rng(P)
    xyz = np.stack([np.linspace(0.02, 0.28, P), np.full(P, 0.15), np.full(P, 0.15)], axis=1)
    xyz[-1] = xyz[-2] + [0.0, 5e-4, 0.0]
    if P >= 3:
        xyz[-3] = xyz[-2] + [0.0, 0.0, 6e-4]           # a point that neighbours the pair but comes before it
    ids = np.arange(P, dtype=np.int64) * 3 + 7
    perm = rng.permutation(P)
    images = [("a.png", ids[perm].copy()), ("b.png", ids[::-1].copy())]
    return ids[perm], xyz[perm], np.full(P, 5, np.int64), images


@pytest.mark.parametrize("P", [2, 3, 128])
def test_close_points_at_the_end_when_every_point_is_kept(P):
    ids, xyz, lens, images = _close_tail(P)
    corners = np.array([[0, 1, 0], [1, 1, 0], [1, 1, 1], [0, 1, 1], [0, 0, 0], [1, 0, 0], [1, 0, 1], [0, 0, 1]], np.float64) * 0.3 + 0.01
    feats, (sc, de) = _features(P, 2, 32, P, [P, P], "cuda")
    m = sr.postprocess(ids, xyz, lens, [p for _, p in images], sc, de, corners, P, 1e-3)
    assert len(m["kept_ids"]) == P and len(m["groups"][-1]) > 1
    _check(sfm.postprocess((ids, xyz, lens), images, feats, corners, P, 1e-3), m)


@pytest.mark.parametrize("P", [2, 3, 128])
def test_merge_writes_nothing_past_its_rows(P):
    """opb_sfm_merge_points with n == cap: sentinels past row cap - 1 of every per-row output stay as they were."""
    ids, xyz, _, _ = _close_tail(P)
    order = np.argsort(ids)
    dev = torch.device("cuda")
    x = torch.from_numpy(xyz[order].astype(np.float32)).to(dev)
    i = torch.from_numpy(ids[order]).to(dev)
    n = torch.tensor([P], dtype=torch.int64, device=dev)
    pad = 64
    merged = torch.full((P + pad, 3), -7.0, dtype=torch.float64, device=dev)
    offsets = torch.full((P + 1 + pad,), -7, dtype=torch.int32, device=dev)
    member_ids = torch.full((P + pad,), -7, dtype=torch.int64, device=dev)
    member_index = torch.full((P + pad,), -7, dtype=torch.int32, device=dev)
    slot_of = torch.full((P + pad,), -7, dtype=torch.int32, device=dev)
    counts = torch.zeros(2, dtype=torch.int64, device=dev)
    ws = sfm._ws(dev, "opb_sfm_merge_workspace_bytes", P)
    _lib.call(dev, "opb_sfm_merge_points", x, i, n, P, 1e-3, ws, ws.numel(), merged, offsets, member_ids, member_index, slot_of, counts[0:1],
              counts[1:2])
    torch.cuda.synchronize()
    n_groups, n_members = (int(v) for v in counts.cpu())
    assert n_members <= P and n_groups < P
    assert bool((merged[P:] == -7.0).all()) and bool((offsets[P + 1:] == -7).all())
    for t in (member_ids, member_index, slot_of):
        assert bool((t[P:] == -7).all())
    m_pos, m_groups = sr.merge(xyz[order].astype(np.float32), ids[order])
    assert n_groups == len(m_groups) and n_members == sum(len(g) for g in m_groups)
    assert np.array_equal(member_index[:n_members].cpu().numpy(), np.concatenate(m_groups))


def test_postprocess_feeds_the_matcher_as_the_models_arrays_do():
    """postprocess -> pad_features3d_random / build_features3d_leaves under a fixed np.random.seed -> matcher.add_object ->
    matches on synthetic frames, against the same chain fed from the model's arrays: equal objects and equal matches."""
    from onepose_b200 import GATsSuperGlue, features3d, synthetic
    P, F, cap, D, L, N = 600, 40, 256, 256, 8, 256
    ids, xyz, lens, images, corners = _generated(91, P, F, cap, dense=True)
    rng = np.random.default_rng(5)
    de = rng.standard_normal((F, D, cap)).astype(np.float32)
    de /= np.linalg.norm(de, axis=1, keepdims=True)
    sc = rng.uniform(0.01, 1.0, (F, cap)).astype(np.float32)
    feats = {"scores": torch.from_numpy(sc).cuda(), "descriptors": torch.from_numpy(de).cuda()}
    out = sfm.postprocess((ids, xyz, lens), images, feats, corners, 400, 1e-3)
    m = sr.postprocess(ids, xyz, lens, [p for _, p in images], sc, de, corners, 400, 1e-3)
    n3d = m["keypoints3d"].shape[0]
    assert out["keypoints3d"].shape[0] == n3d and any(len(g) > 1 for g in m["groups"])

    def objects(avg_d, avg_s, clt_d, clt_s, idxs):
        db, _ = features3d.pad_features3d_random(avg_d, avg_s, n3d)
        np.random.seed(3)
        leaves, _ = features3d.build_features3d_leaves(clt_d, clt_s, idxs, n3d, L)
        return db, leaves

    dev_obj = objects(out["descriptors3d"], out["scores3d"], out["descriptors3d_collect"], out["scores3d_collect"], out["idxs"])
    mod_obj = objects(m["descriptors3d"], m["scores3d"], m["descriptors3d_collect"], m["scores3d_collect"], m["idxs"])
    assert torch.equal(dev_obj[0], mod_obj[0]) and torch.equal(dev_obj[1], mod_obj[1])

    hp = dict(synthetic.DEFAULT_HPARAMS)
    hp["match_threshold"] = 1e-4                      # synthetic weights: keep every mutual nearest neighbour as a match
    sd = synthetic.make_state_dict(4)
    matcher = GATsSuperGlue(dict(hp)).eval()
    matcher.load_state_dict({k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in sd.items()}, strict=True)
    matcher = matcher.cuda()
    a, b = matcher.add_object(*dev_obj), matcher.add_object(*mod_obj)
    db_real = dev_obj[0].cpu().numpy()
    q = torch.from_numpy(np.ascontiguousarray(np.stack([synthetic.make_frame(f, db_real, N)[0] for f in range(4)]), np.float32)).cuda()
    ra = matcher.match_objects(q, [a] * 4)
    rb = matcher.match_objects(q, [b] * 4)
    assert torch.equal(ra["matches0"], rb["matches0"]) and torch.equal(ra["matching_scores0"], rb["matching_scores0"])
    assert torch.equal(ra["conf_matrix"], rb["conf_matrix"])
    assert int((ra["matches0"] > -1).sum()) > 0
