"""Where the arithmetic runs: every GPU entry point on the caller's stream and device, one handle's calls ordered across
streams, several handles and threads at once, and a second device.

Each check compares a call made on a side stream (or another thread, or cuda:1) with the same call made on the default
stream, bit for bit; those single-stream results are pinned against the fp64 references by the other suites, and each group
here also checks one result against the oracle so that the file stands on its own.

The stale-input pattern (group A): on a fresh stream the input buffers are first written with another valid input of the
same shape, then the stream sleeps on the device, then the real input is copied in and the call is made.  A launch on any
other stream runs while the stream sleeps, reads the stale input and returns the other input's result.  Where an entry point
promises no host synchronisation, the stream must still be asleep when the call returns."""
import threading

import numpy as np
import pytest
import torch

from onepose_b200 import GATsSuperGlue, SuperPoint, _lib, features3d, flow, pnp, synthetic
from oracle import gats_spg_oracle as oracle
from oracle import superpoint_oracle as sp_oracle
from tests import flow_scenes as FS
from tests import lk_reference as lk_model

pytestmark = pytest.mark.gpu

SLEEP = 1 << 29              # device cycles of torch.cuda._sleep: about 0.25 s on an H100
B, N, M, M2, L = 4, 192, 320, 257, 8
LENGTHS = [192, 150, 192, 100]
IMG_B, IMG_H, IMG_W, CAP = 2, 96, 128, 256
SP_CONF = {"nms_radius": 3, "max_keypoints": CAP}
N_PNP = 200
CONF_TOL = 1e-4
LK_S, LK_COUNTS, LK_CAP = 128, [200, 90], 60
K_LK = np.array([[300.0, 0, 64.0], [0, 300.0, 64.0], [0, 0, 1]])


# ----------------------------------------------------------------------------- modules and inputs
def _matcher(dev, seed=0):
    m = GATsSuperGlue(dict(synthetic.DEFAULT_HPARAMS)).eval()
    sd = synthetic.make_state_dict(seed)
    m.load_state_dict({k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in sd.items()})
    return m.to(dev), sd


def _extractor(dev, seed=0):
    m = SuperPoint(SP_CONF).eval()
    sd = synthetic.make_superpoint_state_dict(seed, 4.0)
    m.load_state_dict({k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in sd.items()})
    return m.to(dev), sd


def _t(x, dev):
    return torch.from_numpy(np.ascontiguousarray(x)).to(dev)


def _object(i, m, dev):
    d3, d2 = synthetic.make_object(i, m, L)
    return _t(d3, dev), _t(d2, dev)


def _queries(seed, db, dev, n=N):
    return _t(np.stack([synthetic.make_frame(100 * seed + b, db, n)[0] for b in range(B)]), dev)


def _images(seed, dev):
    return _t(np.stack([synthetic.make_image(10 * seed + b, IMG_H, IMG_W) for b in range(IMG_B)]), dev)


def _pnp_frames(seed, dev):
    scenes = [synthetic.make_pnp_scene(50 * seed + b, N_PNP, outlier_frac=0.3) for b in range(B)]
    return {"K": _t(np.stack([s[0] for s in scenes]), dev), "p2": _t(np.concatenate([s[1] for s in scenes]), dev),
            "p3": _t(np.concatenate([s[2] for s in scenes]) * 1000, dev)}


def _matches(seed, dev):
    rs = np.random.RandomState(300 + seed)
    return {"m0": _t(rs.randint(-1, M, size=(B, N)).astype(np.int64), dev),
            "m0b": _t(np.where(np.arange(B)[:, None] % 2 == 0, rs.randint(-1, M, size=(B, N)), rs.randint(-1, M2, size=(B, N))), dev),
            "kp2": _t(rs.rand(B, N, 2).astype(np.float32) * 512, dev), "sc": _t(rs.rand(B, N).astype(np.float32), dev),
            "kp3": _t(0.05 * rs.randn(M, 3).astype(np.float32), dev), "kp3b": _t(0.05 * rs.randn(M2, 3).astype(np.float32), dev)}


class Ctx:
    """The modules of one device, warmed: workspaces sized, weights and objects loaded."""

    def __init__(self, dev):
        self.dev = dev
        self.sp, self.sp_sd = _extractor(dev)
        self.mt, self.sd = _matcher(dev)
        self.d3, self.d2 = _object(1, M, dev)
        self.d3b, self.d2b = _object(2, M2, dev)
        self.db = self.d3.cpu().numpy()
        self.mt.set_object(self.d3, self.d2)
        self.ids = [self.mt.add_object(self.d3, self.d2), self.mt.add_object(self.d3b, self.d2b)]
        self.fwd, _ = _matcher(dev)                           # forward(data): its own current object
        self.obj, _ = _matcher(dev)                           # set_object / add_object cases
        self.obj.set_object(self.d3, self.d2)
        self.q = _queries(0, self.db, dev)
        self.lengths = torch.tensor(LENGTHS, dtype=torch.int32, device=dev)


def _fdata(ctx, q):
    return {"keypoints2d": torch.zeros(B, N, 2, device=ctx.dev), "keypoints3d": torch.zeros(B, M, 3, device=ctx.dev),
            "descriptors2d_query": q, "descriptors3d_db": ctx.d3[None].expand(B, -1, -1),
            "descriptors2d_db": ctx.d2[None].expand(B, -1, -1)}


def _dict_out(d):
    return [d[k] for k in ("matches0", "matches1", "matching_scores0", "matching_scores1", "conf_matrix") if d.get(k) is not None]


def _padded(o):
    c = o["counts"].tolist()
    return [o["counts"]] + [x for b in range(len(c)) for x in (o["keypoints"][b, :c[b]], o["scores"][b, :c[b]], o["descriptors"][b, :, :c[b]])]


def _gathered(g):
    n = int(g["offsets"][-1])
    return [g["offsets"], g["pts2d"][:n], g["pts3d"][:n], g["query_index"][:n]] + ([g["mconf"][:n]] if g["mconf"] is not None else [])


def _posed(p):
    n = int(p["offsets"][-1])
    return [p["pose"], p["pose_homo"], p["n_inliers"], p["inlier_mask"], p["offsets"], p["query_index"][:n]] + \
        ([p["iterations"]] if "iterations" in p else [])


def _add_then_match(ctx, d3, d2, q):
    oid = ctx.obj.add_object(d3, d2)
    out = ctx.obj.match_objects(q, [oid] * B)
    ctx.obj.remove_object(oid)
    return _dict_out(out)


def _leaves(inp):
    np.random.seed(5)                                     # the leaf selection is drawn from numpy's global RNG
    return list(features3d.build_features3d_leaves(inp["obs"], inp["obs_s"], TRACKS, 40, 6))


TRACKS = np.random.RandomState(11).randint(1, 12, size=50)


def _lk_pairs(seed):
    return [FS.warp_scene(70 + 10 * seed + b, LK_S, LK_S) for b in range(IMG_B)]


def _lk_inputs(seed, dev):
    pairs = _lk_pairs(seed)
    return {"prev": _t(np.stack([a for a, _ in pairs]), dev), "next": _t(np.stack([n for _, n in pairs]), dev),
            "pts": _t(np.concatenate([FS.scene_points(seed + b, LK_S, LK_S, n) for b, n in enumerate(LK_COUNTS)]), dev),
            "off": _t(np.array([0, LK_COUNTS[0], sum(LK_COUNTS)], np.int32), dev)}


def _keyframe_inputs(seed, dev):
    """A keyframe state of IMG_B tracks (3D points seen at the 2D ones from [I | 0]), the next crops, and reference poses."""
    rs = np.random.RandomState(500 + seed)
    pairs = _lk_pairs(seed)
    p2 = np.stack([FS.scene_points(seed + b, LK_S, LK_S, LK_CAP, margin=-20.0) for b in range(IMG_B)])
    ray = np.concatenate([p2, np.ones((IMG_B, LK_CAP, 1))], 2) @ np.linalg.inv(K_LK).T
    return {"image": _t(np.stack([a for a, _ in pairs]), dev), "query": _t(np.stack([n for _, n in pairs]), dev), "pts2d": _t(p2, dev),
            "pts3d": _t((ray * rs.uniform(0.4, 0.6, (IMG_B, LK_CAP, 1))).astype(np.float32), dev),
            "counts": _t(np.array([LK_CAP, LK_CAP - 7], np.int32), dev), "K": _t(K_LK, dev), "ref": _t(np.tile(np.eye(4), (IMG_B, 1, 1)), dev)}


def _flow_track(i):
    return flow.flow_track({k: i[k] for k in ("image", "pts2d", "pts3d", "counts")}, i["query"], i["K"], i["ref"])


def _tracked(o):
    return [o[k] for k in ("pose_init_homo", "kpt_dist", "trans_dist", "rot_dist", "n_tracked", "n_inliers", "accept")] + \
        [o["kf"][k] for k in ("image", "pts2d", "pts3d", "counts")]


def _pose_result(seed, dev):
    """A poses_from_matches-style result of IMG_B frames of 50 pairs each (ragged: 50 and 31 used) and its crops."""
    rs = np.random.RandomState(600 + seed)
    n = 50
    return {"offsets": _t(np.array([0, 50, 81], np.int32), dev), "inlier_mask": _t(rs.rand(IMG_B * n) < 0.6, dev),
            "pts2d": _t(rs.rand(IMG_B * n, 2).astype(np.float32).astype(np.float64) * LK_S, dev),
            "pts3d": _t(rs.rand(IMG_B * n, 3).astype(np.float32).astype(np.float64), dev),
            "crops": _t(np.stack([a for a, _ in _lk_pairs(seed)]), dev)}


def _keyframes(i):
    kf = flow.keyframes_from_poses({k: i[k] for k in ("offsets", "inlier_mask", "pts2d", "pts3d")}, i["crops"])
    return [kf[k] for k in ("image", "pts2d", "pts3d", "counts")]


def _sfm(seed, dev):
    rs = np.random.RandomState(400 + seed)
    S = int(TRACKS.sum())
    return {"desc": _t(rs.randn(256, 50).astype(np.float32), dev), "scores": _t(rs.rand(50, 1).astype(np.float32), dev),
            "obs": _t(rs.randn(256, S).astype(np.float32), dev), "obs_s": _t(rs.rand(S, 1).astype(np.float32), dev),
            "tr": _t(rs.randn(S, 256), dev), "tr_s": _t(rs.rand(S, 1), dev)}


# name -> (inputs(ctx, seed), call(ctx, inputs), no host synchronisation promised[, canon(call's result) -> list of tensors: the
# specified parts only; it may read counts to the host, so it runs after the call has been timed])
CASES = {
    "sp_forward_padded": (lambda c, s: {"img": _images(s, c.dev)}, lambda c, i: c.sp.forward_padded(i["img"]), True, _padded),
    "sp_forward": (lambda c, s: {"img": _images(s, c.dev)},
                   lambda c, i: [x for k in ("keypoints", "scores", "descriptors") for x in c.sp(i["img"])[k]], False),
    "match_frames_lengths": (lambda c, s: {"q": _queries(s, c.db, c.dev)},
                             lambda c, i: _dict_out(c.mt.match_frames(i["q"], lengths=c.lengths)), True),
    "match_objects": (lambda c, s: {"q": _queries(s, c.db, c.dev)},
                      lambda c, i: _dict_out(c.mt.match_objects(i["q"], [c.ids[b % 2] for b in range(B)])), True),
    "forward_data": (lambda c, s: {"q": _queries(s, c.db, c.dev)},
                     lambda c, i: (c.fwd(_fdata(c, i["q"])), _dict_out(c.fwd.last_batched))[1], True),
    "set_object": (lambda c, s: dict(zip(("d3", "d2"), _object(10 + s, M, c.dev))),
                   lambda c, i: (c.obj.set_object(i["d3"], i["d2"]), _dict_out(c.obj.match_frames(c.q)))[1], True),
    "add_object": (lambda c, s: dict(zip(("d3", "d2"), _object(20 + s, M, c.dev))),
                   lambda c, i: _add_then_match(c, i["d3"], i["d2"], c.q), False),
    "gather_matches": (lambda c, s: _matches(s, c.dev),
                       lambda c, i: pnp.gather_matches(i["m0"], i["kp2"], i["kp3"], i["sc"]), True, _gathered),
    "gather_matches_objects": (lambda c, s: _matches(s, c.dev),
                               lambda c, i: pnp.gather_matches_objects(i["m0b"], i["kp2"], {0: i["kp3"], 1: i["kp3b"]},
                                                                        [b % 2 for b in range(B)], i["sc"]), True, _gathered),
    "ransac_p3p": (lambda c, s: _pnp_frames(s, c.dev),
                   lambda c, i: list(pnp.ransac_pnp_batch(i["K"], i["p2"], i["p3"], _offsets(c), hypotheses=1024)), True),
    "ransac_epnp": (lambda c, s: _pnp_frames(s, c.dev),
                    lambda c, i: list(pnp.ransac_pnp_batch(i["K"], i["p2"], i["p3"], _offsets(c), method="epnp", hypotheses=1024)), True),
    "ransac_epnp_confidence": (lambda c, s: _pnp_frames(s, c.dev),
                               lambda c, i: list(pnp.ransac_pnp_batch(i["K"], i["p2"], i["p3"], _offsets(c), method="epnp", confidence=0.99)),
                               True),
    "epnp_batch": (lambda c, s: _pnp_frames(s, c.dev), lambda c, i: list(pnp.epnp_batch(i["K"], i["p2"], i["p3"], _offsets(c))), True),
    "poses_from_matches": (lambda c, s: dict(_matches(s, c.dev), K=_pnp_frames(s, c.dev)["K"]),
                           lambda c, i: pnp.poses_from_matches(i["K"], i["kp2"], i["kp3"], i["m0"], i["sc"], hypotheses=512), True, _posed),
    "poses_from_matches_objects": (lambda c, s: dict(_matches(s, c.dev), K=_pnp_frames(s, c.dev)["K"]),
                                   lambda c, i: pnp.poses_from_matches_objects(i["K"], i["kp2"], {0: i["kp3"], 1: i["kp3b"]},
                                                                            [b % 2 for b in range(B)], i["m0b"], i["sc"],
                                                                            method="epnp", confidence=0.99), True, _posed),
    "pad_features3d_random": (lambda c, s: _sfm(s, c.dev), lambda c, i: list(features3d.pad_features3d_random(i["desc"], i["scores"], 64)),
                              False),
    "build_features3d_leaves": (lambda c, s: _sfm(s, c.dev), lambda c, i: _leaves(i), False),
    "mean_descriptors": (lambda c, s: _sfm(s, c.dev), lambda c, i: [features3d.mean_descriptors(i["tr"], TRACKS, device=c.dev)], False),
    "mean_scores": (lambda c, s: _sfm(s, c.dev), lambda c, i: [features3d.mean_scores(i["tr_s"], TRACKS, device=c.dev)], False),
    "lk_batch": (lambda c, s: _lk_inputs(s, c.dev), lambda c, i: list(flow.lk_batch(i["prev"], i["next"], i["pts"], i["off"])), True),
    "flow_track": (lambda c, s: _keyframe_inputs(s, c.dev), lambda c, i: _flow_track(i), True, _tracked),
    "keyframes_from_poses": (lambda c, s: _pose_result(s, c.dev), lambda c, i: _keyframes(i), True),
}


def _offsets(c):
    return torch.arange(0, B * N_PNP + 1, N_PNP, dtype=torch.int32, device=c.dev)


def _same(a, b, tag):
    assert len(a) == len(b), tag
    for i, (x, y) in enumerate(zip(a, b)):
        assert x.dtype == y.dtype and x.shape == y.shape, (tag, i)
        assert x.cpu().numpy().tobytes() == y.cpu().numpy().tobytes(), f"{tag}: output {i} differs"


def _cpu(outs):
    return [x.detach().cpu().clone() for x in outs]


def _canon(name, out):
    case = CASES[name]
    return _cpu(case[3](out) if len(case) > 3 else out)


def _result(ctx, name, seed=0):
    return _canon(name, CASES[name][1](ctx, CASES[name][0](ctx, seed)))


@pytest.fixture(scope="module")
def ctx0():
    return Ctx(torch.device("cuda:0"))


@pytest.fixture(scope="module")
def refs0(ctx0):
    """Every case's result on the default stream (also the warm-up: workspace sizing synchronises by design)."""
    out = {name: _result(ctx0, name) for name in CASES}
    torch.cuda.synchronize()
    return out


def _stale_call(ctx, name):
    """The stale-input pattern on a fresh stream: (outputs, stream still asleep when the call returned)."""
    inputs, call = CASES[name][:2]
    real, stale = inputs(ctx, 0), inputs(ctx, 1)
    buf = {k: torch.empty_like(v) for k, v in real.items()}
    torch.cuda.synchronize(ctx.dev)
    s = torch.cuda.Stream(ctx.dev)
    asleep = torch.cuda.Event()
    with torch.cuda.stream(s):
        for k in buf:
            buf[k].copy_(stale[k])
        torch.cuda._sleep(SLEEP)
        asleep.record(s)
        for k in buf:
            buf[k].copy_(real[k])
        out = call(ctx, buf)
        busy = not asleep.query()
    torch.cuda.synchronize(ctx.dev)
    return _canon(name, out), busy


# ----------------------------------------------------------------------------- A: the caller's stream
@pytest.mark.parametrize("name", list(CASES))
def test_a_entry_point_runs_on_the_callers_stream(ctx0, refs0, name):
    out, busy = _stale_call(ctx0, name)
    _same(out, refs0[name], name)
    if CASES[name][2]:
        assert busy, f"{name} synchronised the host with the caller's stream"


def test_a_match_frames_host_waits_for_the_callers_stream(ctx0):
    """The host input is written by the caller's stream: the library's own copy stream must wait for it."""
    m = ctx0.mt
    real, stale = ctx0.q, _queries(1, ctx0.db, ctx0.dev)
    q_host = torch.empty(real.shape, dtype=torch.float32).pin_memory()
    q_host.copy_(real.cpu())
    ref = {k: v.clone() for k, v in m.match_frames_host(q_host).items()}
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        q_host.copy_(stale, non_blocking=True)
        torch.cuda._sleep(SLEEP)
        q_host.copy_(real, non_blocking=True)
        out = m.match_frames_host(q_host)
    for k in ref:
        assert torch.equal(out[k], ref[k]), k


def test_a_results_against_the_oracles(ctx0, refs0):
    """The single-stream results above are the arithmetic the other suites pin: check two of them here as well."""
    data = {"keypoints2d": np.zeros((B, N, 2), np.float32), "keypoints3d": np.zeros((B, M, 3), np.float32),
            "descriptors2d_query": ctx0.q.cpu().numpy(), "descriptors3d_db": np.repeat(ctx0.db[None], B, 0),
            "descriptors2d_db": np.repeat(ctx0.d2.cpu().numpy()[None], B, 0)}
    ref = oracle.forward(oracle.params_from_numpy(ctx0.sd), data, dict(synthetic.DEFAULT_HPARAMS))
    m0, m1, _, _, conf = refs0["forward_data"]
    assert float((conf - ref["conf_matrix"]).abs().max()) <= CONF_TOL
    assert torch.equal(m0, ref["matches0"]) and torch.equal(m1, ref["matches1"])
    tr = _sfm(0, ctx0.dev)["tr"].cpu().numpy()
    ends = np.cumsum(TRACKS)
    mean = np.stack([tr[e - n:e].mean(axis=0) for e, n in zip(ends, TRACKS)])
    np.testing.assert_allclose(refs0["mean_descriptors"][0].numpy(), mean, rtol=1e-13, atol=1e-15)
    pts = np.concatenate([FS.scene_points(b, LK_S, LK_S, n) for b, n in enumerate(LK_COUNTS)])
    got = [x.numpy() for x in refs0["lk_batch"]]
    for b, (a, n) in enumerate(_lk_pairs(0)):
        rows = slice(sum(LK_COUNTS[:b]), sum(LK_COUNTS[:b + 1]))
        want = lk_model.calc_optical_flow_pyr_lk(a, n, pts[rows], flow.TRACK_WIN, flow.TRACK_LEVELS, flow.TRACK_CRITERIA)
        for g, w in zip(got, want):
            np.testing.assert_array_equal(g[rows], w)


# ----------------------------------------------------------------------------- B: one handle, two streams
def _behind_sleep(s, fn):
    """fn() on stream s behind a device sleep; returns (result, event recorded after it)."""
    done = torch.cuda.Event()
    with torch.cuda.stream(s):
        torch.cuda._sleep(SLEEP)
        out = fn()
        done.record(s)
    return out, done


def test_b_matcher_calls_are_ordered_across_streams(ctx0):
    m = ctx0.mt
    q2 = _queries(2, ctx0.db, ctx0.dev)
    ref_a, ref_b = _cpu(_dict_out(m.match_frames(ctx0.q))), _cpu(_dict_out(m.match_frames(q2)))
    torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    out_a, done_a = _behind_sleep(s1, lambda: m.match_frames(ctx0.q))
    with torch.cuda.stream(s2):
        out_b = m.match_frames(q2)
    s2.synchronize()
    assert done_a.query(), "the call on s2 ran before the handle's earlier call on s1"
    torch.cuda.synchronize()
    _same(_cpu(_dict_out(out_a)), ref_a, "call A")
    _same(_cpu(_dict_out(out_b)), ref_b, "call B")


def test_b_extractor_calls_are_ordered_across_streams(ctx0):
    sp = ctx0.sp
    img_a, img_b = _images(0, ctx0.dev), _images(3, ctx0.dev)
    ref_a, ref_b = _cpu(_padded(sp.forward_padded(img_a))), _cpu(_padded(sp.forward_padded(img_b)))
    torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    out_a, done_a = _behind_sleep(s1, lambda: sp.forward_padded(img_a))
    with torch.cuda.stream(s2):
        out_b = sp.forward_padded(img_b)
    s2.synchronize()
    assert done_a.query(), "the call on s2 ran before the handle's earlier call on s1"
    torch.cuda.synchronize()
    _same(_cpu(_padded(out_a)), ref_a, "call A")
    _same(_cpu(_padded(out_b)), ref_b, "call B")


def test_b_host_call_is_ordered_after_an_async_call(ctx0):
    m = ctx0.mt
    q2 = _queries(2, ctx0.db, ctx0.dev)
    ref_a = _cpu(_dict_out(m.match_frames(ctx0.q)))
    q_host = q2.cpu().pin_memory()
    ref_b = {k: v.clone() for k, v in m.match_frames_host(q_host).items()}
    torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    out_a, done_a = _behind_sleep(s1, lambda: m.match_frames(ctx0.q))
    with torch.cuda.stream(s2):
        out_b = m.match_frames_host(q_host)
    assert done_a.query(), "match_frames_host returned before the handle's earlier call on s1 had run"
    torch.cuda.synchronize()
    _same(_cpu(_dict_out(out_a)), ref_a, "call A")
    for k in ref_b:
        assert torch.equal(out_b[k], ref_b[k]), k


def test_b_object_upload_is_ordered_before_the_next_match(ctx0):
    """set_object on s1 behind a sleep, match_frames on s2: the match must see the new object.  Same M and L as the current
    object, so no buffer grows and no synchronisation hides a missing order."""
    m, _ = _matcher(ctx0.dev)
    d3n, d2n = _object(7, M, ctx0.dev)
    m.set_object(d3n, d2n)
    ref_new = _cpu(_dict_out(m.match_frames(ctx0.q)))
    m.set_object(ctx0.d3, ctx0.d2)
    ref_old = _cpu(_dict_out(m.match_frames(ctx0.q)))
    torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    _behind_sleep(s1, lambda: m.set_object(d3n, d2n))
    with torch.cuda.stream(s2):
        out = m.match_frames(ctx0.q)
    torch.cuda.synchronize()
    out = _cpu(_dict_out(out))
    assert not all(torch.equal(x, y) for x, y in zip(out, ref_old)), "the match read the previous object"
    _same(out, ref_new, "match after set_object")
    # and the new object's result is the oracle's
    data = {"keypoints2d": np.zeros((B, N, 2), np.float32), "keypoints3d": np.zeros((B, M, 3), np.float32),
            "descriptors2d_query": ctx0.q.cpu().numpy(), "descriptors3d_db": np.repeat(d3n.cpu().numpy()[None], B, 0),
            "descriptors2d_db": np.repeat(d2n.cpu().numpy()[None], B, 0)}
    ref = oracle.forward(oracle.params_from_numpy(ctx0.sd), data, dict(synthetic.DEFAULT_HPARAMS))
    assert float((out[4] - ref["conf_matrix"]).abs().max()) <= CONF_TOL
    assert torch.equal(out[0], ref["matches0"]) and torch.equal(out[1], ref["matches1"])


def test_b_range_report_does_not_clear_a_later_calls_flag(ctx0):
    """A range violation reported after a call on s1 resets the device flag; that reset must come before a later call on s2,
    so the later call's own violation still reports count 0 and reaches the host, and a sane call after it is clean."""
    sp, _ = _extractor(ctx0.dev)
    sane = _images(0, ctx0.dev)
    hot = sane * 5e4                                      # conv1a leaves the fp16-split operand range
    ok = _cpu(_padded(sp.forward_padded(sane)))
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    with torch.cuda.stream(s1):
        assert sp.forward_padded(hot)["counts"].tolist() == [0] * IMG_B
        torch.cuda._sleep(SLEEP)                          # s1 stays busy: a reset queued on it lands late
    with torch.cuda.stream(s2):
        with pytest.raises(_lib.OpbError, match="OPB_E_RANGE"):      # the report of the call on s1
            sp.forward_padded(hot)
        out = sp.forward_padded(hot)
    torch.cuda.synchronize()
    assert out["counts"].tolist() == [0] * IMG_B
    with pytest.raises(_lib.OpbError, match="OPB_E_RANGE"):
        sp.check_range()
    with torch.cuda.stream(s2):
        _same(_cpu(_padded(sp.forward_padded(sane))), ok, "sane call after the reports")
    sp.check_range()


# ----------------------------------------------------------------------------- C: several handles and threads at once
def test_c_two_handles_on_two_streams(ctx0):
    dev = ctx0.dev
    ma, sda = _matcher(dev, 0)
    mb, sdb = _matcher(dev, 1)
    ma.set_object(ctx0.d3, ctx0.d2)
    mb.set_object(ctx0.d3b, ctx0.d2b)
    spa, _ = _extractor(dev, 0)
    spb, _ = _extractor(dev, 1)
    qa, qb = ctx0.q, _queries(3, ctx0.d3b.cpu().numpy(), dev)
    img_a, img_b = _images(0, dev), _images(1, dev)
    serial = [_cpu(_dict_out(ma.match_frames(qa))), _cpu(_dict_out(mb.match_frames(qb))), _cpu(_padded(spa.forward_padded(img_a))),
              _cpu(_padded(spb.forward_padded(img_b)))]
    torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    outs = [None] * 4
    for _ in range(2):                                    # interleaved: each stream's work overlaps the other's
        with torch.cuda.stream(s1):
            outs[0] = ma.match_frames(qa)
            outs[2] = spa.forward_padded(img_a)
        with torch.cuda.stream(s2):
            outs[1] = mb.match_frames(qb)
            outs[3] = spb.forward_padded(img_b)
    torch.cuda.synchronize()
    _same(_cpu(_dict_out(outs[0])), serial[0], "matcher a")
    _same(_cpu(_dict_out(outs[1])), serial[1], "matcher b")
    _same(_cpu(_padded(outs[2])), serial[2], "extractor a")
    _same(_cpu(_padded(outs[3])), serial[3], "extractor b")
    data = {"keypoints2d": np.zeros((B, N, 2), np.float32), "keypoints3d": np.zeros((B, M2, 3), np.float32),
            "descriptors2d_query": qb.cpu().numpy(), "descriptors3d_db": np.repeat(ctx0.d3b.cpu().numpy()[None], B, 0),
            "descriptors2d_db": np.repeat(ctx0.d2b.cpu().numpy()[None], B, 0)}
    ref = oracle.forward(oracle.params_from_numpy(sdb), data, dict(synthetic.DEFAULT_HPARAMS))
    assert float((serial[1][4] - ref["conf_matrix"]).abs().max()) <= CONF_TOL
    assert torch.equal(serial[1][0], ref["matches0"])


def _valid_columns(desc, counts):
    """forward_padded's descriptors with the unspecified columns past each frame's count set to 0, on the device."""
    keep = torch.arange(desc.shape[2], device=desc.device)[None] < counts[:, None]
    return torch.where(keep[:, None, :], desc, torch.zeros((), device=desc.device)).contiguous()


class Pipeline:
    """Extractor -> matcher -> poses, with the object built from the extractor's own key points of one image."""

    def __init__(self, dev, seed):
        self.dev = dev
        self.sp, self.sp_sd = _extractor(dev, seed)
        self.mt, _ = _matcher(dev, seed)
        o = self.sp.forward_padded(_images(50 + seed, dev))
        n = int(o["counts"][0])
        d3 = o["descriptors"][0, :, :n].contiguous()
        self.mt.set_object(d3, d3.repeat_interleave(4, dim=1).contiguous())
        self.kp3 = (0.05 * torch.randn(n, 3, generator=torch.Generator().manual_seed(seed))).to(dev)
        self.K = torch.tensor([[600.0, 0, 64], [0, 600.0, 48], [0, 0, 1]], dtype=torch.float64, device=dev)
        self.images = [_images(50 + seed + it, dev) for it in range(3)]

    def step(self, img):
        f = self.sp.forward_padded(img)
        m = self.mt.match_frames(_valid_columns(f["descriptors"], f["counts"]), lengths=f["counts"])
        p = pnp.poses_from_matches(self.K, f["keypoints"], self.kp3, m["matches0"], m["matching_scores0"], hypotheses=512)
        return f, m, p

    @staticmethod
    def canon(r):
        return _cpu(_padded(r[0]) + _dict_out(r[1]) + _posed(r[2]))


def test_c_two_threads_each_with_its_own_pipeline_and_stream(ctx0):
    pipes = [Pipeline(ctx0.dev, 0), Pipeline(ctx0.dev, 1)]
    serial = [[p.canon(p.step(img)) for img in p.images] for p in pipes]
    torch.cuda.synchronize()
    results, errors = [[], []], []

    def run(i):
        try:
            s = torch.cuda.Stream(ctx0.dev)
            with torch.cuda.stream(s):
                for img in pipes[i].images:
                    results[i].append(pipes[i].step(img))
            s.synchronize()
        except Exception as e:                            # surfaced in the main thread
            errors.append(e)

    threads = [threading.Thread(target=run, args=(i,)) for i in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    torch.cuda.synchronize()
    for i in range(2):
        assert len(results[i]) == 3
        for it in range(3):
            _same(Pipeline.canon(results[i][it]), serial[i][it], f"thread {i} iteration {it}")


# ----------------------------------------------------------------------------- D: a second device
two_gpus = pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two visible GPUs")


@pytest.fixture(scope="module")
def ctx1(ctx0, refs0):
    """cuda:1's modules, built while cuda:0 is current and warm (its kernels have their shared-memory limits already)."""
    torch.cuda.set_device(0)
    c = Ctx(torch.device("cuda:1"))
    c.current_device_after_create = torch.cuda.current_device()
    torch.cuda.set_device(0)
    return c


@two_gpus
def test_d_matcher_on_the_second_device(ctx0, refs0, ctx1):
    """The first GEMM and kv-state launches on cuda:1 after cuda:0 is warm; results bit-identical to cuda:0, the caller's device
    untouched, and the result checked against the oracle."""
    assert ctx1.current_device_after_create == 0, "creating cuda:1's handles and objects changed the current device"
    torch.cuda.set_device(0)
    for name in ("match_frames_lengths", "match_objects", "forward_data", "set_object"):
        out = _result(ctx1, name)
        assert torch.cuda.current_device() == 0, name
        _same(out, refs0[name], name)
    q_host = ctx1.q.cpu().pin_memory()
    ref = {k: v.clone() for k, v in ctx0.mt.match_frames_host(q_host).items()}
    out = ctx1.mt.match_frames_host(q_host)
    assert torch.cuda.current_device() == 0
    for k in ref:
        assert torch.equal(out[k], ref[k]), k
    data = {"keypoints2d": np.zeros((B, N, 2), np.float32), "keypoints3d": np.zeros((B, M, 3), np.float32),
            "descriptors2d_query": ctx1.q.cpu().numpy(), "descriptors3d_db": np.repeat(ctx1.db[None], B, 0),
            "descriptors2d_db": np.repeat(ctx1.d2.cpu().numpy()[None], B, 0)}
    ref = oracle.forward(oracle.params_from_numpy(ctx1.sd), data, dict(synthetic.DEFAULT_HPARAMS))
    got = _cpu(CASES["forward_data"][1](ctx1, {"q": ctx1.q}))
    assert float((got[4] - ref["conf_matrix"]).abs().max()) <= CONF_TOL


@two_gpus
def test_d_matcher_refuses_queries_on_another_device(ctx0, ctx1):
    before = ctx1.mt.launch_count()
    with pytest.raises(ValueError, match="cuda:0"):
        ctx1.mt.match_frames(ctx0.q)
    with pytest.raises(ValueError, match="cuda:0"):
        ctx1.mt.match_objects(ctx0.q, [ctx1.ids[0]] * B)
    torch.cuda.synchronize(1)
    assert ctx1.mt.launch_count() == before


@two_gpus
@pytest.mark.parametrize("name", [n for n in CASES if not n.startswith(("match", "forward_data", "set_object"))])
def test_d_entry_point_on_the_second_device(ctx0, refs0, ctx1, name):
    """Extractor (its NMS launch included), pose and feature entry points on cuda:1 while cuda:0 is current."""
    torch.cuda.set_device(0)
    out = _result(ctx1, name)
    assert torch.cuda.current_device() == 0, name
    _same(out, refs0[name], name)


@two_gpus
def test_d_extractor_and_matcher_on_two_devices_in_one_loop(ctx0, ctx1):
    """The pipeline split across GPUs: SuperPoint on cuda:1, the matcher on cuda:0, interleaved; against the one-GPU run and
    the extractor's oracle."""
    torch.cuda.set_device(0)
    sp1 = ctx1.sp
    mt0 = ctx0.mt
    imgs = [_images(60 + i, ctx0.dev) for i in range(3)]
    ref = []
    for img in imgs:
        f = ctx0.sp.forward_padded(img)
        c = f["counts"].clamp(max=N)
        ref.append(_cpu(_padded(f) + _dict_out(mt0.match_frames(_valid_columns(f["descriptors"][:, :, :N], c), lengths=c))))
    torch.cuda.synchronize()
    for img, r in zip(imgs, ref):
        f = sp1.forward_padded(img.to("cuda:1"))
        assert torch.cuda.current_device() == 0
        c = f["counts"].clamp(max=N)
        d = _valid_columns(f["descriptors"][:, :, :N], c).to("cuda:0")
        out = _cpu(_padded(f) + _dict_out(mt0.match_frames(d, lengths=c.to("cuda:0"))))
        assert torch.cuda.current_device() == 0
        _same(out, r, "split pipeline")
    img = imgs[0][:1].cpu().numpy()
    got = sp1(imgs[0][:1].to("cuda:1"))
    sref = sp_oracle.forward(sp_oracle.params_from_numpy(ctx1.sp_sd), img, {"nms_radius": 3, "max_keypoints": CAP})
    d = sp_oracle.compare_keypoints(got["keypoints"][0].cpu().numpy(), got["scores"][0].cpu().numpy(), sref["keypoints"][0].numpy(),
                                    sref["scores"][0].numpy(), 5e-5, CAP)
    assert d["n"] > 0
    assert float((got["descriptors"][0].cpu() - sref["descriptors"][0]).abs().max()) <= 1e-5
