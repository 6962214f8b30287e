"""The matcher -> PnP hand-off on the GPU: opb_gather_matches against the numpy restatement of the reference's masking
(inference.py:147-152), poses_from_matches end to end on planted scenes against the ground truth and the reference-style host
loop, the extractor's padded output fed through the matcher into the gather, and the pose metric on the device."""
import os

import numpy as np
import pytest
import torch

from onepose_b200 import GATsSuperGlue, SuperPoint, _lib, pnp, synthetic
from tests.gather_oracle import gather_matches as gather_oracle, gather_objects_numpy
from tests.golden_util import GOLDEN_DIR

pytestmark = pytest.mark.gpu


def _random_matches(rs, B, N, M):
    """Matches with every kind of entry: -1, valid indices, indices >= M and < -1; frame 0 without pairs and frame 1 fully
    matched when there are enough frames."""
    m0 = np.full((B, N), -1, np.int64)
    u = rs.rand(B, N)
    valid = rs.randint(0, M, size=(B, N))
    m0[u < 0.5] = valid[u < 0.5]
    m0[(u >= 0.5) & (u < 0.6)] = M + rs.randint(0, 5, size=int(((u >= 0.5) & (u < 0.6)).sum()))
    m0[(u >= 0.6) & (u < 0.65)] = -rs.randint(2, 1 << 40, size=int(((u >= 0.6) & (u < 0.65)).sum()))
    if B >= 3:
        m0[0] = -1
        m0[1] = valid[1]
    return m0


def _assert_same(got, ref):
    off = got["offsets"].cpu().numpy()
    assert np.array_equal(off, ref["offsets"]), (off, ref["offsets"])
    T = int(off[-1])
    for key in ("pts2d", "pts3d", "mconf", "query_index"):
        if ref[key] is None or got.get(key) is None:
            continue
        assert got[key][:T].cpu().numpy().tobytes() == ref[key].tobytes(), key


@pytest.mark.parametrize("M", [1, 7000])
@pytest.mark.parametrize("N", [1, 37, 1024, 4096, 9000])
@pytest.mark.parametrize("B", [1, 3, 32])
def test_gather_matches_equals_numpy_masking(B, N, M):
    rs = np.random.RandomState(B * 100003 + N * 7 + M)
    m0 = _random_matches(rs, B, N, M)
    kp2 = rs.uniform(0, 512, size=(B, N, 2)).astype(np.float32)
    kp2[(m0 < 0) | (m0 >= M)] = np.nan                     # rows of unmatched entries must never be read
    kp3 = (0.05 * rs.randn(M, 3)).astype(np.float32)
    sc = rs.rand(B, N).astype(np.float32)
    ref = gather_oracle(m0, kp2, kp3, sc)
    args = [torch.from_numpy(x).cuda() for x in (m0, kp2, kp3)]
    a = pnp.gather_matches(*args, matching_scores0=torch.from_numpy(sc).cuda())
    b = pnp.gather_matches(*args, matching_scores0=torch.from_numpy(sc).cuda())
    _assert_same(a, ref)
    _assert_same(b, ref)
    # optional outputs NULL, straight through the C ABI
    lib = _lib.load()
    T = int(ref["offsets"][-1])
    p2 = torch.empty(B * N, 2, dtype=torch.float64, device="cuda")
    p3 = torch.empty(B * N, 3, dtype=torch.float64, device="cuda")
    off = torch.empty(B + 1, dtype=torch.int32, device="cuda")
    _lib.check(lib.opb_gather_matches(args[0].data_ptr(), None, args[1].data_ptr(), args[2].data_ptr(), B, N, M, p2.data_ptr(),
                                      p3.data_ptr(), None, None, off.data_ptr(), torch.cuda.current_stream().cuda_stream))
    _assert_same({"pts2d": p2, "pts3d": p3, "offsets": off}, dict(ref, mconf=None, query_index=None))
    assert a["pts2d"][:T].isfinite().all()
    nostores = pnp.gather_matches(*args)
    assert nostores["mconf"] is None
    _assert_same(nostores, ref)


def test_gather_matches_without_query_points():
    m0 = torch.empty(3, 0, dtype=torch.int64, device="cuda")
    out = pnp.gather_matches(m0, torch.empty(3, 0, 2, device="cuda"), torch.zeros(5, 3, device="cuda"))
    assert out["offsets"].cpu().tolist() == [0, 0, 0, 0]
    with pytest.raises(ValueError):
        pnp.gather_matches(torch.zeros(2, 4, dtype=torch.int64, device="cuda"), torch.zeros(2, 5, 2, device="cuda"),
                           torch.zeros(5, 3, device="cuda"))


# ---- past the first tile of the gather's scans: offsets over more than 1024 frames, compaction past 256 entries ----

EDGE_FRAMES = list(range(1022, 1027)) + list(range(2046, 2051))
OBJECT_M = [1, 300, 700]                 # the objects of the mixed gather
FILL = 0xA5


def _tile_edge_matches(rs, Mb, N, fill):
    """matches0 [B, N] for frames of Mb[b] 3D key points: "empty" (T = 0), "full" (every entry a match), or "mixed": -1, matches,
    indices >= M_b and below -1, with the frames at 1022-1026 and 2046-2050 (the edges of gather_scan's 1024-frame tiles)
    alternately empty and fully matched."""
    B = len(Mb)
    valid = (rs.rand(B, N) * Mb[:, None]).astype(np.int64)
    if fill == "empty":
        return np.full((B, N), -1, np.int64)
    if fill == "full":
        return valid
    u = rs.rand(B, N)
    m0 = np.full((B, N), -1, np.int64)
    m0[u < 0.5] = valid[u < 0.5]
    beyond = (u >= 0.5) & (u < 0.6)
    m0[beyond] = (Mb[:, None] + rs.randint(0, 5, (B, N)))[beyond]
    neg = (u >= 0.6) & (u < 0.65)
    m0[neg] = -rs.randint(2, 1 << 40, size=int(neg.sum()))
    for k, b in enumerate(e for e in EDGE_FRAMES if e < B):
        m0[b] = -1 if (k + N) % 2 else valid[b]
    return m0


def _inputs(rs, m0, Mb):
    kp2 = rs.uniform(0, 512, size=(*m0.shape, 2)).astype(np.float32)
    kp2[(m0 < 0) | (m0 >= Mb[:, None])] = np.nan              # rows of unmatched entries must never be read
    return kp2, rs.rand(*m0.shape).astype(np.float32)


def _filled(shape, dtype):
    n = int(np.prod(shape)) * torch.empty(0, dtype=dtype).element_size()
    return torch.full((n,), FILL, dtype=torch.uint8, device="cuda").view(dtype).reshape(shape)


def _gather_abi(name, m0, sc, kp2, mid, B, N, ref):
    """Entry point `name` (arguments m0, sc, kp2, *mid, then the outputs) into outputs whose bytes are FILL first, each with 8
    spare rows past its capacity: offsets equal the oracle's int32 cumsum exactly, every row below T is byte-equal, and no row at
    or past T, nor an offset past B, is written."""
    cap = B * N + 8
    out = {"pts2d": _filled((cap, 2), torch.float64), "pts3d": _filled((cap, 3), torch.float64), "mconf": _filled((cap,), torch.float32),
           "query_index": _filled((cap,), torch.int32), "offsets": _filled((B + 1 + 8,), torch.int32)}
    _lib.call(torch.device("cuda"), name, m0, sc, kp2, *mid, out["pts2d"], out["pts3d"], out["mconf"], out["query_index"], out["offsets"])
    off = out["offsets"].cpu()
    assert np.array_equal(off[:B + 1].numpy(), ref["offsets"]) and bool((off[B + 1:].view(torch.uint8) == FILL).all())
    T = int(ref["offsets"][-1])
    for key in ("pts2d", "pts3d", "mconf", "query_index"):
        v = out[key].cpu()
        assert v[:T].numpy().tobytes() == ref[key].tobytes(), key
        assert bool((v[T:].contiguous().view(torch.uint8) == FILL).all()), key


GATHER_CASES = [(B, N, fill) for B in (1023, 1024, 1025, 2048, 2049) for N in (1, 255, 256, 257) for fill in ("mixed", "empty", "full")]
GATHER_CASES.append((70000, 3, "mixed"))


@pytest.mark.parametrize("B,N,fill", GATHER_CASES, ids=[f"B{c[0]}-N{c[1]}-{c[2]}" for c in GATHER_CASES])
def test_gather_past_one_scan_tile(B, N, fill):
    """gather_matches and gather_matches_objects at more than 1024 frames (gather_scan carries a running total from tile to
    tile) and at N around gather_compact's 256-entry tiles, against the numpy oracles, through the Python API and through the C
    ABI into pre-filled outputs."""
    rs = np.random.RandomState(B * 1000 + N * 3 + len(fill))
    M = 7000
    Mb = np.full(B, M)
    m0 = _tile_edge_matches(rs, Mb, N, fill)
    kp2, sc = _inputs(rs, m0, Mb)
    kp3 = (0.05 * rs.randn(M, 3)).astype(np.float32)
    ref = gather_oracle(m0, kp2, kp3, sc)
    kept = ((m0 >= 0) & (m0 < M)).sum(1)
    assert np.array_equal(ref["offsets"], np.concatenate([[0], np.cumsum(kept)]).astype(np.int32))
    assert (ref["offsets"][-1] == 0) == (fill == "empty") and (ref["offsets"][-1] == B * N) == (fill == "full")
    d = [torch.from_numpy(x).cuda() for x in (m0, kp2, kp3, sc)]
    _assert_same(pnp.gather_matches(d[0], d[1], d[2], d[3]), ref)
    _gather_abi("opb_gather_matches", d[0], d[3], d[1], (d[2], B, N, M), B, N, ref)

    ids = rs.randint(0, len(OBJECT_M), B)                      # frames of three objects, mixed
    Mb = np.array(OBJECT_M)[ids]
    m0 = _tile_edge_matches(rs, Mb, N, fill)
    kp2, sc = _inputs(rs, m0, Mb)
    objs = {i: (0.05 * rs.randn(m, 3)).astype(np.float32) for i, m in enumerate(OBJECT_M)}
    ref = gather_objects_numpy(m0, kp2, objs, ids.tolist(), sc)
    d = [torch.from_numpy(x).cuda() for x in (m0, kp2, sc)]
    _assert_same(pnp.gather_matches_objects(d[0], d[1], {i: torch.from_numpy(v).cuda() for i, v in objs.items()}, ids.tolist(), d[2]), ref)
    kp3_all = torch.from_numpy(np.concatenate([objs[i] for i in range(len(OBJECT_M))])).cuda()
    first = np.concatenate([[0], np.cumsum(OBJECT_M)[:-1]])[ids].astype(np.int32)
    tab = [torch.from_numpy(t).cuda() for t in (first, Mb.astype(np.int32))]
    _gather_abi("opb_gather_matches_objects", d[0], d[2], d[1], (kp3_all, tab[0], tab[1], B, N), B, N, ref)


def test_poses_from_matches_past_one_scan_tile():
    """poses_from_matches on 1100 frames of 0 to 12 pairs (make_pnp_scene's points and outliers, as test_pose_domain_gpu.py's
    _scene makes them; the frames at 1022-1026 empty or full) against ransac_pnp_batch on the numpy-gathered lists with the same
    seed: pose, inlier mask and inlier counts bit for bit."""
    B, N, seed = 1100, 12, 5
    rs = np.random.RandomState(3)
    n_b = rs.randint(0, N + 1, B)
    n_b[1022:1027] = [0, N, 0, N, 0]
    K = np.zeros((B, 3, 3))
    kp2 = np.full((B, N, 2), np.nan, np.float32)
    kp3 = np.zeros((B * N, 3), np.float32)
    m0 = np.full((B, N), -1, np.int64)
    for b in range(B):
        K[b], uv, P, _ = synthetic.make_pnp_scene(b, max(int(n_b[b]), 1))
        slots = np.sort(rs.choice(N, n_b[b], replace=False))
        kp2[b, slots] = uv[:n_b[b]]
        kp3[b * N:b * N + n_b[b]] = P[:n_b[b]]
        m0[b, slots] = b * N + np.arange(n_b[b])
    m0[m0 < 0] = np.where(rs.rand(int((m0 < 0).sum())) < 0.5, -1, B * N + 3)    # unmatched: -1 or past M
    sc = rs.rand(B, N).astype(np.float32)
    d = [torch.from_numpy(x).cuda() for x in (K, kp2, kp3, m0, sc)]
    res = pnp.poses_from_matches(d[0], d[1], d[2], d[3], d[4], seed=seed)
    ref = gather_oracle(m0, kp2, kp3, sc)
    off = torch.from_numpy(ref["offsets"]).cuda()
    pose, mask, cnt = pnp.ransac_pnp_batch(d[0], torch.from_numpy(ref["pts2d"]).cuda(), torch.from_numpy(ref["pts3d"]).cuda() * 1000.0, off,
                                           seed=seed)
    pose[:, :, 3] /= 1000.0
    T = int(ref["offsets"][-1])
    assert torch.equal(res["offsets"], off)
    assert torch.equal(res["pose"], pose) and torch.equal(res["n_inliers"], cnt) and torch.equal(res["inlier_mask"][:T], mask)
    few = torch.from_numpy(n_b < 4).cuda()                     # fewer than 4 pairs: the identity pose and no inliers
    assert not cnt[few].any() and int((cnt > 0).sum()) > 400


def _matcher(desc3d, desc2d_db):
    mm = GATsSuperGlue(dict(synthetic.DEFAULT_HPARAMS)).eval()
    mm.load_state_dict({k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in synthetic.make_state_dict(0).items()})
    mm = mm.cuda()
    mm.set_object(torch.as_tensor(desc3d).cuda(), torch.as_tensor(desc2d_db).cuda())
    return mm


def test_poses_from_matches_on_planted_scenes():
    """Eight frames of a 2500-point object whose planted query columns sit at the projections of their 3D points (0.5 px noise)
    and one frame of unplanted queries: matcher -> poses_from_matches.  Every planted frame passes 1cm@1degree; every frame's
    pose is the one the reference-style host loop (numpy mask, then ransac_PnP(K, mkpts2d, mkpts3d, scale=1000)) gets from
    the same matches, with as many inliers; the unplanted frame gets the identity pose and no inliers."""
    B, N, M = 8, 1024, 2500
    s = synthetic.make_planted_scene(4, list(range(401, 401 + B)) + [499], N, M, unplanted=(499,))
    mm = _matcher(s["desc3d"], s["desc2d_db"])
    out = mm.match_frames(torch.from_numpy(s["descriptors2d"]).cuda(), return_conf=False)
    kp2, kp3, K = (torch.from_numpy(s[k]).cuda() for k in ("keypoints2d", "keypoints3d", "K"))
    res = pnp.poses_from_matches(K, kp2, kp3, out["matches0"], out["matching_scores0"])
    assert res["pose"].shape == (B + 1, 3, 4) and res["pose_homo"].shape == (B + 1, 4, 4) and res["pose"].is_cuda
    assert torch.equal(res["pose_homo"][:, :3], res["pose"]) and torch.equal(res["pose_homo"][:, 3], torch.tensor([0, 0, 0, 1.0]).expand(B + 1, 4).cuda())
    rot, trans = pnp.pose_errors(res["pose"][:B], torch.from_numpy(s["pose_gt"][:B]).cuda())
    print("planted frames: rot err deg", rot.cpu().numpy(), "trans err cm", trans.cpu().numpy(), "inliers", res["n_inliers"].cpu().numpy())
    assert pnp.cm_degree(rot, trans)["1cm@1degree"] == 1.0
    m0 = out["matches0"].cpu().numpy()
    s0 = out["matching_scores0"].cpu().numpy()
    off = res["offsets"].cpu().numpy()
    mask = res["inlier_mask"].cpu().numpy()
    for b in range(B + 1):
        valid = m0[b] > -1
        mkpts2d, mkpts3d, mconf = s["keypoints2d"][b][valid], s["keypoints3d"][m0[b][valid]], s0[b][valid]
        pose, _, inliers = pnp.ransac_PnP(s["K"][b], mkpts2d, mkpts3d, scale=1000)
        np.testing.assert_allclose(res["pose"][b].cpu().numpy(), pose, rtol=0, atol=1e-12)
        assert int(res["n_inliers"][b]) == len(inliers) == int(mask[off[b]:off[b + 1]].sum())
        assert np.array_equal(res["mconf"][off[b]:off[b + 1]].cpu().numpy(), mconf)
        assert np.array_equal(res["query_index"][off[b]:off[b + 1]].cpu().numpy(), np.nonzero(valid)[0])
    assert np.array_equal(res["pose"][B].cpu().numpy(), np.eye(4)[:3]) and int(res["n_inliers"][B]) == 0
    # a shared [3,3] camera: frame 0 alone, same bits as in the batch (frame 0's samples do not depend on the batch)
    solo = pnp.poses_from_matches(K[0], kp2[:1], kp3, out["matches0"][:1], out["matching_scores0"][:1])
    assert torch.equal(solo["pose"][0], res["pose"][0]) and torch.equal(solo["n_inliers"][0], res["n_inliers"][0])
    again = pnp.poses_from_matches(K, kp2, kp3, out["matches0"], out["matching_scores0"])
    assert torch.equal(again["pose"], res["pose"]) and torch.equal(again["n_inliers"], res["n_inliers"])


def test_extractor_padded_output_through_matcher_into_gather():
    """SuperPoint.forward_padded -> match_frames(lengths=counts) -> gather_matches equals the numpy restatement on the same
    tensors; key-point rows past each frame's count hold NaN, so a read of them would show.  The descriptors of seeded random
    SuperPoint weights are too alike for the matcher's 0.2 threshold, so each frame's first counts[b] descriptor columns are
    replaced by make_frame's planted ones; the padded layout, key points and counts are the extractor's."""
    sp = SuperPoint({"nms_radius": 3, "max_keypoints": 256}).eval()
    sp.load_state_dict({k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in synthetic.make_superpoint_state_dict(0, 4.0).items()},
                       strict=True)
    sp = sp.cuda()
    img = torch.from_numpy(np.stack([synthetic.make_image(i, 96, 128) for i in (11, 12, 13)], 0)).cuda()
    det = sp.forward_padded(img)
    counts = det["counts"].cpu().tolist()
    assert len(set(counts)) > 1 or counts[0] < 256, counts               # a ragged batch
    kp = det["keypoints"]
    desc = det["descriptors"]
    db, leaves = synthetic.make_object(6, 300, 8)
    for b, n in enumerate(counts):
        kp[b, n:] = float("nan")
        desc[b, :, :n] = torch.from_numpy(synthetic.make_frame(61 + b, db, n)[0]).cuda()
    mm = _matcher(db, leaves)
    out = mm.match_frames(desc, return_conf=False, lengths=det["counts"])
    kp3 = torch.from_numpy((0.05 * np.random.RandomState(0).randn(db.shape[1], 3)).astype(np.float32)).cuda()
    got = pnp.gather_matches(out["matches0"], kp, kp3, out["matching_scores0"])
    ref = gather_oracle(out["matches0"].cpu().numpy(), kp.cpu().numpy(), kp3.cpu().numpy(), out["matching_scores0"].cpu().numpy())
    _assert_same(got, ref)
    T = int(ref["offsets"][-1])
    print("extractor feed: key points", counts, "pairs per frame", np.diff(ref["offsets"]))
    assert T > 0 and bool(got["pts2d"][:T].isfinite().all())


def test_pose_errors_on_device_equal_cpu():
    g = dict(np.load(os.path.join(GOLDEN_DIR, "pnp_pose_metrics.npz"), allow_pickle=False))
    p, q = torch.from_numpy(g["pose_pred"]), torch.from_numpy(g["pose_gt"])
    rc, tc = pnp.pose_errors(p, q)
    rg, tg = pnp.pose_errors(p.cuda(), q.cuda())
    assert rg.is_cuda and tg.is_cuda
    np.testing.assert_allclose(rg.cpu().numpy(), rc.numpy(), rtol=1e-12, atol=0, equal_nan=True)
    np.testing.assert_allclose(tg.cpu().numpy(), tc.numpy(), rtol=1e-12, atol=0, equal_nan=True)
    assert pnp.cm_degree(rg, tg) == pnp.cm_degree(rc, tc)
