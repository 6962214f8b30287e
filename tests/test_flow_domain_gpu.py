"""The tracker's flow step on the GPU (onepose_b200.flow / csrc/flow.cu) over the whole domain its entry points accept.

LK against the numpy model (tests/lk_reference.py, which test_lk_reference_cpu.py pins to cv2 4.13 in every row): next_pts of
every row -- status 0 included, NaN equal to NaN, every other value bit for bit -- status, and err (0 where status is 0) bit
for bit; the pyramids read back from the workspace bit for bit.  The compaction and the reprojection distance against numpy,
called directly, and flow_track at the keyframe cap of the benchmarked configuration against its parts.  The scenes are
tests/flow_scenes.py's cv2-free ones."""
import numpy as np
import pytest
import torch

from onepose_b200 import _lib, flow, pnp
from tests import flow_scenes as FS
from tests import lk_reference as L

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TRACK = (flow.TRACK_WIN, flow.TRACK_LEVELS, flow.TRACK_CRITERIA)
WIDTHS = list(range(3, 32, 2))
# every odd width, each with another odd height (WIDTHS rotated by 7): every split of a row into 8-column blocks and a tail,
# and windows wider than tall and taller than wide
WINS = [(w, WIDTHS[(i + 7) % len(WIDTHS)]) for i, w in enumerate(WIDTHS)]
CRITS = [(1, 1, 0.0), (1, 100, 0.0), (2, 0, 0.0), (2, 0, 0.5), (3, 5, 20.0), (3, 10, 0.03)]
MIN_EIGS = [0.0, 1e-4, 1e-3, 1e-2]
SMALL_SIZES = [(1, 1), (1, 9), (9, 1), (2, 2), (3, 5), (4, 40), (5, 7), (9, 9), (12, 30), (16, 16), (20, 20), (31, 33), (33, 31),
               (47, 63)]
SMALL_WINS = [(3, 3), (5, 11), (15, 15), (31, 31)]
TALLY = {"configurations": 0, "points": 0, "status-0 rows": 0, "pyramid levels": 0}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("flow domain: compared " + ", ".join(f"{v} {k}" for k, v in TALLY.items()))


def _model(prev, nxt, pts, win, lev, crit, min_eig=1e-4):
    with np.errstate(invalid="ignore"):                 # the cast of NaN and inf points to int64
        return L.calc_optical_flow_pyr_lk(prev, nxt, pts, win, lev, crit, min_eig)


def _bits_differ(a, b):
    """Indices where fp32 arrays a and b differ: NaN equals NaN, every other value bit for bit."""
    na, nb = np.isnan(a), np.isnan(b)
    return np.nonzero((na != nb) | (~na & ~nb & (a.view(np.uint32) != b.view(np.uint32))))[0]


def _check(got, want, tag):
    """Device (next_pts, status, err) against the model's, every row."""
    p, s, e = (x.cpu().numpy() for x in got)
    wp, ws, we = want
    assert p.shape == wp.shape and s.shape == ws.shape and e.shape == we.shape, tag
    bad = np.nonzero(s != ws)[0]
    assert not len(bad), (tag, "status differs at row", int(bad[0]), int(s[bad[0]]), int(ws[bad[0]]))
    bad = _bits_differ(p.reshape(-1), wp.reshape(-1)) // 2
    assert not len(bad), (tag, "next_pts differ at row", int(bad[0]), p[bad[0]].tolist(), wp[bad[0]].tolist(), int(ws[bad[0]]))
    bad = _bits_differ(e, we)
    assert not len(bad), (tag, "err differs at row", int(bad[0]), float(e[bad[0]]), float(we[bad[0]]))
    TALLY["points"] += len(s)
    TALLY["status-0 rows"] += int((ws == 0).sum())


def _check_pyramid(ws, B, H, W, lev, win, b, prev, nxt, tag):
    """Pair b's pyramid in the workspace against the model's of its own images."""
    P, dP = L.build_pyramid(prev, win, lev)
    N, _ = L.build_pyramid(nxt, win, lev)
    got = flow.pyramid_views(ws, B, H, W, lev, win, b, size=prev.shape)
    assert len(got) == len(P), (tag, len(got), len(P))
    for level, (ip, inx, der) in enumerate(got):
        assert np.array_equal(der.cpu().numpy(), dP[level]), (tag, "derivatives", level)
        if level:
            assert np.array_equal(ip.cpu().numpy(), P[level]), (tag, "prev", level)
            assert np.array_equal(inx.cpu().numpy(), N[level]), (tag, "next", level)
    TALLY["pyramid levels"] += len(P)


def _dev(x, dtype=None):
    return torch.as_tensor(np.ascontiguousarray(x), dtype=dtype).to(DEV)


def _offsets(counts):
    return _dev(np.concatenate([[0], np.cumsum(counts)]).astype(np.int32))


def _lk(prev, nxt, pts, counts, win, lev, crit, min_eig=1e-4, **kw):
    return flow.lk_batch(prev, nxt, _dev(pts), _offsets(counts), win, lev, crit, min_eig, **kw)


# ----------------------------------------------------------------------------- the parameters
@pytest.fixture(scope="module")
def scenes():
    """Two pairs of 120 x 160: sub-pixel and large motion."""
    return [FS.warp_scene(31, 120, 160, "affine"), FS.warp_scene(32, 120, 160, "large")]


def _param_configs():
    """Each window with a level count, criteria and min_eig in turn; then every criteria x min_eig at 15 x 15, 2 levels."""
    out = [(win, i % 5, CRITS[i % len(CRITS)], MIN_EIGS[i % len(MIN_EIGS)]) for i, win in enumerate(WINS)]
    return out + [((15, 15), 2, c, m) for c in CRITS for m in MIN_EIGS]


@pytest.mark.parametrize("win,lev,crit,min_eig", _param_configs())
def test_parameters(scenes, win, lev, crit, min_eig):
    """Both pairs in one launch, 500 scene points each and the border points of every level of their pyramids."""
    pts, counts = [], []
    for k, (prev, _) in enumerate(scenes):
        h, w = prev.shape
        p = np.concatenate([FS.scene_points(40 + k, h, w, 500), FS.border_points(h, w, win, L.n_levels(h, w, win, lev))])
        pts.append(p)
        counts.append(len(p))
    prev_t = _dev(np.stack([s[0] for s in scenes]))
    next_t = _dev(np.stack([s[1] for s in scenes]))
    ws = torch.full((flow.workspace_bytes(2, 120, 160, lev),), 0xAB, dtype=torch.uint8, device=DEV)
    got = _lk(prev_t, next_t, np.concatenate(pts), counts, win, lev, crit, min_eig, workspace=ws)
    want = [_model(s[0], s[1], p, win, lev, crit, min_eig) for s, p in zip(scenes, pts)]
    _check(got, [np.concatenate(x) for x in zip(*want)], (win, lev, crit, min_eig))
    for k, (prev, nxt) in enumerate(scenes):
        _check_pyramid(ws, 2, 120, 160, lev, win, k, prev, nxt, (win, lev, k))
    assert 0 < int((want[0][1] == 1).sum()) < counts[0]
    TALLY["configurations"] += 1


# ----------------------------------------------------------------------------- the benchmarked shape and flow_track's cap
BENCH_B, BENCH_S, BENCH_CAP = 32, 512, 2000
K_BENCH = np.array([[600.0, 0, 256.0], [0, 600.0, 256.0], [0, 0, 1]])


@pytest.fixture(scope="module")
def bench():
    """tools/flow_bench.py's 32 pairs of 512 x 512 crops, with sub-pixel motion and 2000 points each (flow_bench's 1000 are the
    first 1000), and the model's results for every point at the tracker's parameters."""
    pairs = [FS.warp_scene(100 + b, BENCH_S, BENCH_S, "affine") for b in range(BENCH_B)]
    pts = np.stack([FS.scene_points(100 + b, BENCH_S, BENCH_S, BENCH_CAP) for b in range(BENCH_B)])
    want = [_model(a, n, p, *TRACK) for (a, n), p in zip(pairs, pts)]
    return pairs, pts, want


@pytest.mark.parametrize("B", [32, 8, 1])
def test_benchmarked_shape(bench, B):
    pairs, pts, want = bench
    n = 1000
    got = _lk(_dev(np.stack([a for a, _ in pairs[:B]])), _dev(np.stack([x for _, x in pairs[:B]])), pts[:B, :n].reshape(-1, 2), [n] * B,
              *TRACK)
    _check(got, [np.concatenate([w[i][:n] for w in want[:B]]) for i in range(3)], ("benchmarked shape", B))
    TALLY["configurations"] += 1


def _compact_model(status, p2, p3, counts, cap):
    """np.where(status == 1) of each track's first counts[b] rows (clamped to [0, cap]): (rows2d, rows3d, offsets, n_tracked,
    pad2d, pad3d) as opb_flow_compact defines them."""
    B = len(counts)
    r2, r3, n_tr = [], [], []
    pad2, pad3 = np.zeros((B, cap, 2), np.float32), np.zeros((B, cap, 3), np.float32)
    for b in range(B):
        n = min(max(int(counts[b]), 0), cap)
        keep = np.nonzero(status[b, :n] == 1)[0]
        r2.append(p2[b, keep])
        r3.append(p3[b, keep])
        pad2[b, :len(keep)] = p2[b, keep]
        pad3[b, :len(keep)] = p3[b, keep]
        n_tr.append(len(keep))
    off = np.concatenate([[0], np.cumsum(n_tr)]).astype(np.int32)
    return (np.concatenate(r2).astype(np.float64), np.concatenate(r3).astype(np.float64), off, np.array(n_tr, np.int32), pad2, pad3)


def _kpt_dist(K, pose, p2, p3):
    """tracking_utils.project's mean distance in fp64, summed in row order (NaN for no rows)."""
    if len(p2) == 0:
        return np.nan
    x = p3 @ pose[:, :3].T + pose[:, 3]
    x = x @ K.T
    d = np.sqrt(((x[:, :2] / x[:, 2:] - p2) ** 2).sum(1))
    return np.add.accumulate(d)[-1] / len(d)


def test_flow_track_at_cap_2000(bench):
    """flow_track on the 32 pairs with the matcher's N = 2000 keyframe rows, counts 0 .. > cap (most of them past 1024 rows,
    the compaction's chunk), against its parts: n_tracked and the compacted rows from the model's status and points, the pose
    bit-equal to ransac_pnp_batch on those rows, kpt_dist to 1e-9, and accept and the new keyframe state by their rule."""
    pairs, pts, want = bench
    B, cap = BENCH_B, BENCH_CAP
    rs = np.random.RandomState(8)
    counts = np.array([[cap, 1500, 1025, 1024, 0, 3, cap + 500, -1][b % 8] if b < 16 else int(rs.randint(1, cap + 1)) for b in range(B)],
                      np.int32)
    # 3D points seen at the keyframe points from [I | 0] at depths 0.4 .. 0.6 m: the tracked points are near the identity pose
    ray = np.concatenate([pts, np.ones((B, cap, 1))], 2) @ np.linalg.inv(K_BENCH).T
    p3 = (ray * rs.uniform(0.4, 0.6, (B, cap, 1))).astype(np.float32)
    ref = np.tile(np.eye(4), (B, 1, 1))
    ref[1::2, 2, 3] = 0.1                               # 10 cm away: these tracks are not accepted
    kf = {"image": _dev(np.stack([a for a, _ in pairs])), "pts2d": _dev(pts), "pts3d": _dev(p3), "counts": _dev(counts)}
    query = _dev(np.stack([n for _, n in pairs]))
    K = _dev(K_BENCH)
    out = flow.flow_track(kf, query, K, _dev(ref))
    status = np.stack([w[1] for w in want])
    tracked = np.stack([w[0] for w in want])
    r2, r3, off, n_tr, pad2, pad3 = _compact_model(status, tracked, p3, counts, cap)
    assert out["n_tracked"].cpu().numpy().tolist() == n_tr.tolist()
    pose, _, n_in = pnp.ransac_pnp_batch(K.expand(B, 3, 3).contiguous(), _dev(r2), _dev(r3), _dev(off), reproj_error=5.0,
                                         hypotheses=pnp.EPNP_HYPOTHESES, method="epnp", confidence=0.99)
    assert torch.equal(out["pose_init_homo"][:, :3], pose) and torch.equal(out["n_inliers"], n_in)
    P = out["pose_init_homo"].cpu().numpy()
    kd = out["kpt_dist"].cpu().numpy()
    for b in range(B):
        want_kd = _kpt_dist(K_BENCH, P[b, :3], r2[off[b]:off[b + 1]], r3[off[b]:off[b + 1]])
        assert (np.isnan(kd[b]) and np.isnan(want_kd)) or abs(kd[b] - want_kd) <= 1e-9 * abs(want_kd), (b, kd[b], want_kd)
    rot, trans = pnp.pose_errors(out["pose_init_homo"], _dev(ref))
    assert torch.equal(out["rot_dist"], rot) and torch.equal(out["trans_dist"], trans)
    accept = (trans <= flow.ACCEPT_CM) & (rot <= flow.ACCEPT_DEG) & (out["kpt_dist"] < flow.ACCEPT_PX)
    assert torch.equal(out["accept"], accept)
    acc = accept.cpu().numpy()
    assert acc.any() and not acc.all(), acc
    nk = {k: v.cpu().numpy() for k, v in out["kf"].items()}
    for b in range(B):
        if acc[b]:
            assert np.array_equal(nk["image"][b], pairs[b][1]) and int(nk["counts"][b]) == n_tr[b], b
            assert np.array_equal(nk["pts2d"][b], pad2[b]) and np.array_equal(nk["pts3d"][b], pad3[b]), b
        else:
            assert np.array_equal(nk["image"][b], pairs[b][0]) and int(nk["counts"][b]) == counts[b], b
            assert np.array_equal(nk["pts2d"][b], pts[b]) and np.array_equal(nk["pts3d"][b], p3[b]), b
    print(f"flow_track at cap {cap}: n_tracked {n_tr.tolist()}, {int(acc.sum())} of {B} accepted")


# ----------------------------------------------------------------------------- small images, per-pair sizes
@pytest.mark.parametrize("win", SMALL_WINS)
@pytest.mark.parametrize("lev", [0, 2, 4])
def test_small_images(win, lev):
    """Every small size alone as its own H x W call, then all of them as pairs of one 64 x 64 `sizes` batch -- different top
    levels in one launch -- with three entries the device clamps (0, -3 and 69 a side): points and every pyramid level."""
    crit = (3, 10, 0.03)
    S = 64
    clamped = [((0, 5), (1, 5)), ((-3, 40), (1, 40)), ((S + 5, S + 5), (S, S))]
    entries = [(hw, hw) for hw in SMALL_SIZES] + clamped
    slot_p = np.zeros((len(entries), S, S), np.uint8)
    slot_n = np.zeros_like(slot_p)
    pairs, pts, want = [], [], []
    for b, (_, (h, w)) in enumerate(entries):
        a, n = FS.warp_scene(h * 100 + w + b, h, w) if b < len(SMALL_SIZES) else FS.warp_scene(900 + b, S, S)
        slot_p[b, :a.shape[0], :a.shape[1]], slot_n[b, :a.shape[0], :a.shape[1]] = a, n
        a, n = slot_p[b, :h, :w].copy(), slot_n[b, :h, :w].copy()
        p = np.concatenate([FS.scene_points(h + w, h, w, 40, margin=3.0), FS.border_points(h, w, win, L.n_levels(h, w, win, lev))])
        pairs.append((a, n))
        pts.append(p)
        want.append(_model(a, n, p, win, lev, crit))
        if b < len(SMALL_SIZES):                        # alone: the pair is the whole H x W
            ws = torch.full((flow.workspace_bytes(1, h, w, lev),), 0xAB, dtype=torch.uint8, device=DEV)
            got = _lk(_dev(a[None]), _dev(n[None]), p, [len(p)], win, lev, crit, workspace=ws)
            _check(got, want[-1], ("alone", h, w, win, lev))
            _check_pyramid(ws, 1, h, w, lev, win, 0, a, n, ("alone", h, w, win, lev))
            TALLY["configurations"] += 1
    B = len(entries)
    ws = torch.full((flow.workspace_bytes(B, S, S, lev),), 0xAB, dtype=torch.uint8, device=DEV)
    sizes = _dev(np.array([hw for hw, _ in entries], np.int32))
    got = _lk(_dev(slot_p), _dev(slot_n), np.concatenate(pts), [len(p) for p in pts], win, lev, crit, sizes=sizes, workspace=ws)
    _check(got, [np.concatenate(x) for x in zip(*want)], ("sizes batch", win, lev))
    for b, (a, n) in enumerate(pairs):
        _check_pyramid(ws, B, S, S, lev, win, b, a, n, ("sizes batch", entries[b], win, lev))
    TALLY["configurations"] += 1


# ----------------------------------------------------------------------------- layouts
def test_layouts():
    """prev and next as slices of larger tensors with different row and frame pitches (next's the larger), then prev as one
    keyframe expanded over every pair (frame pitch 0); ragged and empty point sets."""
    B, H, W = 6, 96, 128
    win, lev, crit = (15, 15), 2, (3, 10, 0.03)
    pairs = [FS.warp_scene(60 + b, H, W, "affine" if b % 2 else "large") for b in range(B)]
    counts = [0, 300, 17, 0, 250, 1]
    pts = [FS.scene_points(70 + b, H, W, c) for b, c in enumerate(counts)]
    big_p = torch.zeros(B, H + 3, W + 5, dtype=torch.uint8, device=DEV)
    big_n = torch.zeros(B, H + 11, W + 40, dtype=torch.uint8, device=DEV)
    prev_t, next_t = big_p[:, 1:1 + H, 2:2 + W], big_n[:, 4:4 + H, 7:7 + W]
    prev_t.copy_(_dev(np.stack([a for a, _ in pairs])))
    next_t.copy_(_dev(np.stack([n for _, n in pairs])))
    assert prev_t.stride()[:2] != next_t.stride()[:2] and all(x < y for x, y in zip(prev_t.stride()[:2], next_t.stride()[:2]))
    got = _lk(prev_t, next_t, np.concatenate(pts), counts, win, lev, crit)
    _check(got, [np.concatenate(x) for x in zip(*[_model(a, n, p, win, lev, crit) for (a, n), p in zip(pairs, pts)])], "pitches")
    TALLY["configurations"] += 1
    key = big_p[0, 1:1 + H, 2:2 + W]                    # one keyframe shared by every pair, frame pitch 0
    shared = key[None].expand(B, H, W)
    assert shared.stride(0) == 0
    got = _lk(shared, next_t, np.concatenate(pts), counts, win, lev, crit)
    _check(got, [np.concatenate(x) for x in zip(*[_model(pairs[0][0], n, p, win, lev, crit) for (_, n), p in zip(pairs, pts)])],
           "shared keyframe")
    TALLY["configurations"] += 1
    got = _lk(prev_t, next_t, np.zeros((0, 2), np.float32), [0] * B, win, lev, crit)     # no points at all
    assert all(x.shape[0] == 0 for x in got)


# ----------------------------------------------------------------------------- compaction and reprojection
@pytest.mark.parametrize("B", [1, 3, 40])
def test_compact(B):
    """opb_flow_compact for caps around the 1024-row chunk and past it, counts of 0, cap, > cap, negative and random, tracks
    all 0, all 1 and mixed (with a few status values other than 0 and 1); outputs start as NaN / 0x7F sentinels."""
    rs = np.random.RandomState(B)
    for cap in (1, 1023, 1024, 1025, 2000, 3000):
        for r in range(5):
            kinds = [(b + r) % 3 for b in range(B)]     # 0 mixed, 1 all 1, 2 all 0
            status = np.stack([np.where(rs.rand(cap) < 0.6, 1, rs.choice([0, 0, 0, 2, 255], cap)) if k == 0 else np.full(cap, k == 1)
                               for k in kinds]).astype(np.uint8)
            counts = np.array([[cap, int(rs.randint(0, cap + 1)), 0, cap + 5, -7][(b + r) % 5] for b in range(B)], np.int32)
            p2 = rs.randn(B, cap, 2).astype(np.float32)
            p3 = rs.randn(B, cap, 3).astype(np.float32)
            n = B * cap
            out2 = torch.full((n, 2), float("nan"), dtype=torch.float64, device=DEV)
            out3 = torch.full((n, 3), float("nan"), dtype=torch.float64, device=DEV)
            off = torch.full((B + 1,), 0x7F7F7F7F, dtype=torch.int32, device=DEV)
            n_tr = torch.full((B,), 0x7F7F7F7F, dtype=torch.int32, device=DEV)
            pad2 = torch.full((B, cap, 2), float("nan"), device=DEV)
            pad3 = torch.full((B, cap, 3), float("nan"), device=DEV)
            _lib.call(torch.device(DEV), "opb_flow_compact", _dev(status), _dev(p2), _dev(p3), _dev(counts), B, cap, out2, out3, off, n_tr,
                      pad2, pad3)
            w2, w3, woff, wn, wp2, wp3 = _compact_model(status, p2, p3, counts, cap)
            tag = (B, cap, r)
            assert off.cpu().numpy().tolist() == woff.tolist(), tag
            assert n_tr.cpu().numpy().tolist() == wn.tolist(), tag
            total = int(woff[-1])
            assert np.array_equal(out2[:total].cpu().numpy(), w2) and np.array_equal(out3[:total].cpu().numpy(), w3), tag
            assert np.array_equal(pad2.cpu().numpy(), wp2) and np.array_equal(pad3.cpu().numpy(), wp3), tag


def test_reprojection():
    """opb_flow_reprojection for tracks of 0 .. 3000 points against numpy's fp64 row-order sum, to 1e-9 relative."""
    rs = np.random.RandomState(12)
    sizes = [0, 1, 2, 7, 100, 1023, 1024, 1025, 3000, 0, 513]
    B = len(sizes)
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
    K = np.zeros((B, 3, 3))
    K[:, 0, 0], K[:, 1, 1], K[:, 0, 2], K[:, 1, 2], K[:, 2, 2] = rs.uniform(300, 900, B), rs.uniform(300, 900, B), rs.uniform(100, 400, B), \
        rs.uniform(100, 400, B), 1
    pose = np.stack([np.concatenate([FS.rodrigues(rs.uniform(-0.5, 0.5, 3)), [[rs.uniform(-0.05, 0.05)], [rs.uniform(-0.05, 0.05)],
                                                                            [rs.uniform(0.4, 1.0)]]], 1) for _ in range(B)])
    p3 = rs.uniform(-0.08, 0.08, (off[-1], 3))
    p2 = np.concatenate([FS.project(K[b], pose[b], p3[off[b]:off[b + 1]]) for b in range(B)]) + rs.normal(0, 3.0, (off[-1], 2))
    dist = torch.full((B,), 7.0, dtype=torch.float64, device=DEV)
    _lib.call(torch.device(DEV), "opb_flow_reprojection", _dev(K.reshape(B, 9)), _dev(pose.reshape(B, 12)), _dev(p2), _dev(p3), _dev(off), B,
              dist)
    got = dist.cpu().numpy()
    for b in range(B):
        want = _kpt_dist(K[b], pose[b], p2[off[b]:off[b + 1]], p3[off[b]:off[b + 1]])
        if sizes[b] == 0:
            assert np.isnan(got[b]), b
        else:
            assert abs(got[b] - want) <= 1e-9 * want, (b, got[b], want)
