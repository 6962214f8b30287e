"""Frames of different objects in one matcher call (GATsSuperGlue.add_object / match_objects, opb_forward_objects) and the
mixed-object pose hand-off (opb_gather_matches_objects): every frame against the oracle on its own object, the one-object
call against match_frames bit for bit, order independence, agreement with per-object calls, the object registry, and the
pose of planted scenes of several objects solved in one call."""
import ctypes as C

import numpy as np
import pytest
import torch

from onepose_b200 import GATsSuperGlue, _lib, pnp, synthetic
from oracle import gats_spg_oracle as oracle
from tests.gather_oracle import gather_objects_numpy

pytestmark = pytest.mark.gpu

CONF_TOL = 1e-4


def _module(sd, hp):
    m = GATsSuperGlue(dict(hp)).eval()
    m.load_state_dict({k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in sd.items()}, strict=True)
    return m.cuda()


def _add(m, obj_seed, M, L):
    db, leaves = synthetic.make_object(obj_seed, M, L)
    return m.add_object(torch.from_numpy(db).cuda(), torch.from_numpy(leaves).cuda())


def _check_frame(out, b, ref, rb, M, tag):
    """Frame b of a match_objects output against frame rb of an oracle dict on its own object (M columns)."""
    conf = out["conf_matrix"][b, :, :M].cpu()
    rc = ref["conf_matrix"][rb]
    err = float((conf - rc).abs().max())
    assert err <= CONF_TOL, f"{tag}: max|dconf| = {err:.3e}"
    np.testing.assert_array_equal(out["matches0"][b].cpu().numpy(), ref["matches0"][rb].numpy(), err_msg=tag)
    np.testing.assert_array_equal(out["matches1"][b, :M].cpu().numpy(), ref["matches1"][rb].numpy(), err_msg=tag)
    np.testing.assert_allclose(out["matching_scores0"][b].cpu().numpy(), ref["matching_scores0"][rb].numpy(), atol=CONF_TOL)
    np.testing.assert_allclose(out["matching_scores1"][b, :M].cpu().numpy(), ref["matching_scores1"][rb].numpy(), atol=CONF_TOL)
    top2 = rc.topk(2, dim=1).values
    decided = (top2[:, 0] - top2[:, 1]) > 1e-5 * top2[:, 0]
    assert bool((conf.argmax(1) == ref["raw_indices0"][rb])[decided].all()), tag
    # padding past the frame's own M
    assert bool((out["matches1"][b, M:] == -1).all()), tag
    assert bool((out["matching_scores1"][b, M:] == 0).all()), tag
    assert bool((out["conf_matrix"][b, :, M:] == 0).all()), tag
    return err


def _oracle_frames(sd, hp, obj_seed, M, L, frame_ids, N, lengths=None):
    data = synthetic.make_batch(obj_seed, frame_ids, N, M, L)
    if lengths is not None:                    # ragged: the oracle sees each frame's valid columns only
        refs = []
        for j, n in enumerate(lengths):
            d = {k: v[j:j + 1] for k, v in data.items()}
            d["descriptors2d_query"] = d["descriptors2d_query"][:, :, :n]
            d["keypoints2d"] = d["keypoints2d"][:, :n]
            refs.append(oracle.forward(oracle.params_from_numpy(sd), d, hp))
        return data, refs
    return data, oracle.forward(oracle.params_from_numpy(sd), data, hp)


def _mixed_parity(hp, sd, Ms, L, order, N, lengths, chunk, hoist=True):
    """Objects of sizes Ms, frames `order` (object index per frame), ragged `lengths`; each frame against the oracle."""
    m = _module(sd, hp)
    m.set_hoist(hoist)
    m.set_chunk_frames(chunk)
    ids = [_add(m, 300 + k, M, L) for k, M in enumerate(Ms)]
    q = np.zeros((len(order), 256, N), np.float32)
    refs = []
    for b, k in enumerate(order):
        data, r = _oracle_frames(sd, hp, 300 + k, Ms[k], L, [700 + b], N, lengths=[lengths[b]])
        q[b] = data["descriptors2d_query"][0]
        refs.append(r[0])
    lens = torch.tensor(lengths, dtype=torch.int32).cuda()
    out = m.match_objects(torch.from_numpy(q).cuda(), [ids[k] for k in order], lengths=lens)
    assert out["matches1"].shape == (len(order), max(Ms))
    for b, k in enumerate(order):
        n = lengths[b]
        sub = {key: (v[b:b + 1, :n] if key in ("matches0", "matching_scores0") else v[b:b + 1, :n] if key == "conf_matrix" else v[b:b + 1])
               for key, v in out.items()}
        _check_frame(sub, 0, refs[b], 0, Ms[k], f"frame {b} (object {k}, M {Ms[k]})")
        assert bool((out["matches0"][b, n:] == -1).all())
    return m, out, ids


def test_mixed_objects_vs_oracle():
    """Four objects crossing m_pad 256 / 512 / 768, seven frames in interleaved order, ragged lengths, chunks of 3 frames (the
    chunks differ in m_pad)."""
    hp = dict(synthetic.DEFAULT_HPARAMS)
    sd = synthetic.make_state_dict(4)
    _mixed_parity(hp, sd, [100, 256, 300, 700], 8, [3, 0, 2, 1, 0, 3, 2], 200, [200, 150, 77, 200, 1, 199, 120], chunk=3)


@pytest.mark.parametrize("variant", ["L5", "lintrans_additional", "noself", "nohoist"])
def test_mixed_objects_variants_vs_oracle(variant):
    hp = dict(synthetic.DEFAULT_HPARAMS)
    L = 8
    if variant == "L5":
        L = 5
    elif variant == "lintrans_additional":
        hp.update(with_linear_transform=True, additional=True)
    elif variant == "noself":
        hp.update(include_self=False)
    sd = synthetic.make_state_dict(5, hparams=hp)
    _mixed_parity(hp, sd, [60, 300, 130], L, [1, 0, 2, 0, 1], 96, [96, 50, 96, 10, 80], chunk=2, hoist=variant != "nohoist")


def test_hoist_off_matches_hoist_on():
    hp = dict(synthetic.DEFAULT_HPARAMS)
    sd = synthetic.make_state_dict(6)
    a = _mixed_parity(hp, sd, [60, 300, 130], 8, [1, 0, 2, 0, 1], 96, [96, 96, 96, 96, 96], chunk=2, hoist=True)[1]
    b = _mixed_parity(hp, sd, [60, 300, 130], 8, [1, 0, 2, 0, 1], 96, [96, 96, 96, 96, 96], chunk=2, hoist=False)[1]
    err = float((a["conf_matrix"] - b["conf_matrix"]).abs().max())
    assert err <= 2e-6, err


def _q(frame_ids, db, N):
    return torch.from_numpy(np.stack([synthetic.make_frame(f, db, N)[0] for f in frame_ids])).cuda()


def test_one_object_call_equals_match_frames():
    """All frames on one object: match_objects == match_frames bit for bit (same B, N, chunking)."""
    hp = dict(synthetic.DEFAULT_HPARAMS)
    sd = synthetic.make_state_dict(0)
    m = _module(sd, hp)
    m.set_chunk_frames(3)
    db, leaves = synthetic.make_object(11, 700, 8)
    oid = m.add_object(torch.from_numpy(db).cuda(), torch.from_numpy(leaves).cuda())
    m.set_object(torch.from_numpy(db).cuda(), torch.from_numpy(leaves).cuda())
    q = _q(range(50, 57), db, 300)
    lens = torch.tensor([300, 10, 299, 150, 300, 1, 256], dtype=torch.int32).cuda()
    a = m.match_frames(q, lengths=lens)
    b = m.match_objects(q, [oid] * 7, lengths=lens)
    for k in a:
        assert torch.equal(a[k], b[k]), k


def test_frame_order_independence():
    """Within one chunk, permuting the frames permutes the outputs bit for bit."""
    hp = dict(synthetic.DEFAULT_HPARAMS)
    sd = synthetic.make_state_dict(1)
    m = _module(sd, hp)
    Ms = [180, 520, 90]
    ids = [_add(m, 40 + k, M, 8) for k, M in enumerate(Ms)]
    objs = [0, 1, 2, 1, 0, 0, 2, 1, 1, 0, 2, 2, 0, 1, 1, 0, 2, 0, 1, 1]   # 20 frames of three objects in one chunk
    N = 128
    q = torch.stack([_q([900 + b], synthetic.make_object(40 + objs[b], Ms[objs[b]], 8)[0], N)[0] for b in range(len(objs))])
    a = m.match_objects(q, [ids[k] for k in objs])
    perm = np.random.RandomState(3).permutation(len(objs))
    b = m.match_objects(q[torch.from_numpy(perm).cuda()], [ids[objs[p]] for p in perm])
    for k in a:
        assert torch.equal(a[k][torch.from_numpy(perm).cuda()], b[k]), k


def test_agreement_with_per_object_calls():
    """Eight objects with M ~ U[800, 2500], N = 1024, one frame each: one call == eight match_frames calls."""
    hp = dict(synthetic.DEFAULT_HPARAMS)
    sd = synthetic.make_state_dict(0)
    m = _module(sd, hp)
    rs = np.random.RandomState(8)
    Ms = [int(x) for x in rs.randint(800, 2501, size=8)]
    N = 1024
    objs = [synthetic.make_object(60 + k, M, 8) for k, M in enumerate(Ms)]
    ids = [m.add_object(torch.from_numpy(db).cuda(), torch.from_numpy(lv).cuda()) for db, lv in objs]
    q = torch.cat([_q([1200 + k], objs[k][0], N) for k in range(8)])
    mixed = m.match_objects(q, ids)
    max_err = 0.0
    for k, (db, lv) in enumerate(objs):
        m.set_object(torch.from_numpy(db).cuda(), torch.from_numpy(lv).cuda())
        single = m.match_frames(q[k:k + 1])
        M = Ms[k]
        assert torch.equal(mixed["matches0"][k], single["matches0"][0]), k
        assert torch.equal(mixed["matches1"][k, :M], single["matches1"][0]), k
        max_err = max(max_err, float((mixed["conf_matrix"][k, :, :M] - single["conf_matrix"][0]).abs().max()))
    print(f"max |dconf| mixed vs per-object calls: {max_err:.3e}")
    assert max_err <= 1e-5
    for k in (0, 5):                                         # two frames against the oracle as well
        data = synthetic.make_batch(60 + k, [1200 + k], N, Ms[k], 8)
        ref = oracle.forward(oracle.params_from_numpy(sd), data, hp)
        _check_frame(mixed, k, ref, 0, Ms[k], f"frame {k}")


def test_registry_remove_add_reload_and_argument_checks():
    hp = dict(synthetic.DEFAULT_HPARAMS)
    sd = synthetic.make_state_dict(2)
    m = _module(sd, hp)
    N = 64
    a = _add(m, 80, 100, 8)
    b = _add(m, 81, 200, 8)
    q2 = torch.cat([_q([5], synthetic.make_object(80, 100, 8)[0], N), _q([6], synthetic.make_object(81, 200, 8)[0], N)])
    m.match_objects(q2, [a, b])
    m.remove_object(a)
    with pytest.raises(ValueError):
        m.match_objects(q2, [a, b])
    c = _add(m, 82, 900, 8)                                  # larger than anything before: the workspace grows
    q3 = torch.cat([_q([7], synthetic.make_object(82, 900, 8)[0], N), q2[1:]])
    out = m.match_objects(q3, [c, b])
    for k, (seed, M, fid) in enumerate([(82, 900, 7), (81, 200, 6)]):
        ref = oracle.forward(oracle.params_from_numpy(sd), synthetic.make_batch(seed, [fid], N, M, 8), hp)
        _check_frame(out, k, ref, 0, M, f"after add, frame {k}")
    # fixed-width rows: a 2-D out["matches1"] sets M_out; the first 900 columns equal the call's own width, the rest is padding
    wide = m.match_objects(q3, [c, b], out={"matches1": torch.empty(2, 1000, dtype=torch.int64, device="cuda")})
    assert wide["matches1"].shape == (2, 1000) and wide["conf_matrix"].shape == (2, N, 1000)
    for key in out:
        assert torch.equal(wide[key][..., :900], out[key]), key
    assert bool((wide["matches1"][:, 900:] == -1).all()) and bool((wide["matching_scores1"][:, 900:] == 0).all())
    assert bool((wide["conf_matrix"][:, :, 900:] == 0).all())
    with pytest.raises(ValueError):
        m.match_objects(q3, [c, b], out={"matches1": torch.empty(2, 899, dtype=torch.int64, device="cuda")})
    # chunks hold at most 64 frames: larger settings are refused and leave the setting as it was
    with pytest.raises(_lib.OpbError):
        m.set_chunk_frames(65)
    assert m._chunk_frames == 0
    m.set_chunk_frames(64)
    assert torch.equal(m.match_objects(q3, [c, b])["matches0"], out["matches0"])
    m.set_chunk_frames(0)
    # weight reload: registered objects follow the new weights
    sd2 = synthetic.make_state_dict(3)
    m.load_state_dict({k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in sd2.items()}, strict=True)
    out = m.match_objects(q3, [c, b])
    for k, (seed, M, fid) in enumerate([(82, 900, 7), (81, 200, 6)]):
        ref = oracle.forward(oracle.params_from_numpy(sd2), synthetic.make_batch(seed, [fid], N, M, 8), hp)
        _check_frame(out, k, ref, 0, M, f"after reload, frame {k}")
    # argument checks of the C entry point
    lib, h = m._lib, m._handle
    d5 = synthetic.make_object(83, 50, 5)
    l5 = m.add_object(torch.from_numpy(d5[0]).cuda(), torch.from_numpy(d5[1]).cuda())
    o = {k: torch.zeros(2, 900 * N, dtype=t).cuda() for k, t in (("m0", torch.int64), ("m1", torch.int64), ("s0", torch.float32),
                                                                  ("s1", torch.float32))}
    st = torch.cuda.current_stream().cuda_stream

    def call(ids, B=2, Nn=N, M_out=900):
        arr = (C.c_int32 * max(len(ids), 1))(*ids)
        return lib.opb_forward_objects(h, arr, q3.data_ptr(), None, B, Nn, M_out, o["m0"].data_ptr(), o["m1"].data_ptr(), o["s0"].data_ptr(),
                                       o["s1"].data_ptr(), None, st)
    assert call([c, b]) == 0
    assert call([c, 12345]) == -1                            # unknown id
    assert call([a, b]) == -1                                # removed id
    assert call([c, l5]) == -1                               # mixed L
    assert call([c, b], M_out=899) == -1                     # M_out below the largest M
    assert call([c, b], B=0) == -1
    assert call([c, b], Nn=0) == -1
    assert lib.opb_remove_object(h, 12345) == -1
    m.check_range()


def test_current_object_beside_registered_ones():
    """With a current object set next to a registered one: id -1 (the current object's key inside the handle) is an unknown id
    to opb_forward_objects and opb_remove_object, and a weight reload unsets the current object (opb_forward refuses until the
    next opb_set_object) while the registered object gives the same results as before it."""
    hp = dict(synthetic.DEFAULT_HPARAMS)
    sd = synthetic.make_state_dict(2)
    m = _module(sd, hp)
    N = 64
    cur = [torch.from_numpy(t).cuda() for t in synthetic.make_object(84, 150, 8)]
    m.set_object(*cur)
    a = _add(m, 85, 120, 8)
    q = torch.cat([_q([9], synthetic.make_object(84, 150, 8)[0], N), _q([10], synthetic.make_object(85, 120, 8)[0], N)])
    before_cur = {k: v.clone() for k, v in m.match_frames(q).items()}
    before_reg = {k: v.clone() for k, v in m.match_objects(q, [a, a]).items()}
    lib, h = m._lib, m._handle
    o = {k: torch.zeros(2 * 150 * N, dtype=t).cuda() for k, t in (("m0", torch.int64), ("m1", torch.int64), ("s0", torch.float32),
                                                                   ("s1", torch.float32))}
    st = torch.cuda.current_stream().cuda_stream

    def forward_objects(ids):
        arr = (C.c_int32 * 2)(*ids)
        return lib.opb_forward_objects(h, arr, q.data_ptr(), None, 2, N, 150, o["m0"].data_ptr(), o["m1"].data_ptr(), o["s0"].data_ptr(),
                                       o["s1"].data_ptr(), None, st)
    for ids in ([-1, a], [a, -1]):
        assert forward_objects(ids) == -1, ids
        assert b"unknown object id -1" in lib.opb_last_error(h), ids
    assert lib.opb_remove_object(h, -1) == -1
    assert b"unknown object id -1" in lib.opb_last_error(h)
    with pytest.raises(ValueError, match="unknown object id -1"):
        m.match_objects(q, [-1, a])
    assert forward_objects([a, a]) == 0
    # weight reload with the same weights, straight through the C ABI
    assert lib.opb_finalize_weights(h) == 0
    assert lib.opb_forward(h, q.data_ptr(), None, 2, N, o["m0"].data_ptr(), o["m1"].data_ptr(), o["s0"].data_ptr(), o["s1"].data_ptr(),
                           None, st) == -3                  # OPB_E_STATE: no current object
    with pytest.raises(_lib.OpbError, match="OPB_E_STATE"):
        m.match_frames(q)
    after_reg = m.match_objects(q, [a, a])
    for k in before_reg:
        assert torch.equal(after_reg[k], before_reg[k]), k
    assert lib.opb_set_object(h, cur[0].data_ptr(), cur[1].data_ptr(), 150, 8, st) == 0
    after_cur = m.match_frames(q)
    for k in before_cur:
        assert torch.equal(after_cur[k], before_cur[k]), k
    m.check_range()


def test_workspace_fill_does_not_change_bits():
    hp = dict(synthetic.DEFAULT_HPARAMS)
    sd = synthetic.make_state_dict(4)
    lib = _lib.load()

    def run():
        m = _module(sd, hp)
        m.set_chunk_frames(2)
        ids = [_add(m, 90 + k, M, 8) for k, M in enumerate([120, 600, 260])]
        q = torch.cat([_q([30 + b], synthetic.make_object(90 + k, M, 8)[0], 200) for b, (k, M) in enumerate([(2, 260), (0, 120), (1, 600)])])
        out = m.match_objects(q, [ids[2], ids[0], ids[1]], lengths=torch.tensor([200, 31, 170], dtype=torch.int32).cuda())
        torch.cuda.synchronize()
        return {k: v.clone() for k, v in out.items()}
    a = run()
    try:
        assert lib.opb_debug_set_ws_fill(0xFF) == 0
        b = run()
    finally:
        lib.opb_debug_set_ws_fill(-1)
    for k in a:
        assert torch.equal(a[k], b[k]), k


def test_mixed_gather_and_poses_on_planted_scenes():
    """Three planted objects, frames mixed in one call: match_objects -> mixed gather -> poses.  Every frame passes
    1cm@1degree, each pose equals the per-object poses_from_matches route to 1e-12 with the same inliers, and the gather is
    bit-identical to the numpy restatement."""
    hp = dict(synthetic.DEFAULT_HPARAMS)
    m = GATsSuperGlue(hp).eval()
    m.load_state_dict({k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in synthetic.make_state_dict(0).items()})
    m = m.cuda()
    N = 1024
    specs = [(4, 2500, [401, 402, 403]), (5, 1200, [411, 412]), (6, 1800, [421, 422, 423])]
    scenes = [synthetic.make_planted_scene(o, f, N, M) for o, M, f in specs]
    ids = [m.add_object(torch.from_numpy(s["desc3d"]).cuda(), torch.from_numpy(s["desc2d_db"]).cuda()) for s in scenes]
    order = [(0, 0), (1, 0), (2, 0), (0, 1), (2, 1), (1, 1), (0, 2), (2, 2)]     # (scene, frame in scene)
    q = torch.from_numpy(np.stack([scenes[s]["descriptors2d"][f] for s, f in order])).cuda()
    kp2 = torch.from_numpy(np.stack([scenes[s]["keypoints2d"][f] for s, f in order])).cuda()
    K = torch.from_numpy(np.stack([scenes[s]["K"][f] for s, f in order])).cuda()
    gt = torch.from_numpy(np.stack([scenes[s]["pose_gt"][f] for s, f in order])).cuda()
    oids = [ids[s] for s, _ in order]
    kp3 = {ids[s]: torch.from_numpy(scenes[s]["keypoints3d"]).cuda() for s in range(3)}
    out = m.match_objects(q, oids, return_conf=False)
    g = pnp.gather_matches_objects(out["matches0"], kp2, kp3, oids, out["matching_scores0"])
    ref = gather_objects_numpy(out["matches0"].cpu().numpy(), kp2.cpu().numpy(), {k: v.cpu().numpy() for k, v in kp3.items()}, oids,
                               out["matching_scores0"].cpu().numpy())
    off = g["offsets"].cpu().numpy()
    assert np.array_equal(off, ref["offsets"])
    T = int(off[-1])
    for key in ("pts2d", "pts3d", "mconf", "query_index"):
        assert g[key][:T].cpu().numpy().tobytes() == ref[key].tobytes(), key
    res = pnp.poses_from_matches_objects(K, kp2, kp3, oids, out["matches0"], out["matching_scores0"])
    rot, trans = pnp.pose_errors(res["pose"], gt)
    print("rot err deg", rot.cpu().numpy(), "trans err cm", trans.cpu().numpy())
    assert pnp.cm_degree(rot, trans)["1cm@1degree"] == 1.0
    for s in range(3):                                       # the per-object route on the same matches
        rows = [b for b, (ss, _) in enumerate(order) if ss == s]
        r = pnp.poses_from_matches(K[rows], kp2[rows], kp3[ids[s]], out["matches0"][rows], out["matching_scores0"][rows])
        assert float((r["pose"] - res["pose"][rows]).abs().max()) <= 1e-12, s
        assert torch.equal(r["n_inliers"], res["n_inliers"][rows]), s
