"""GPU parity tests (run with -m gpu on an H100): the CUDA path through the module / C ABI
against (a) the golden vectors produced by the reference module and (b) the CPU oracle on
the same seeded inputs.  Contract (BASELINE.json north_star): conf within 1e-4 abs,
match indices bit-exact."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from onepose_b200 import GATsSuperGlue, _lib, features3d, synthetic
from oracle import gats_spg_oracle as oracle
from tests.golden_util import GOLDEN_DIR, RELEASED_CASES, conf_reference_view, load_case, load_dustbin_case

pytestmark = pytest.mark.gpu

CONF_TOL = 1e-4          # north_star tolerance


def _module(sd, hp):
    m = GATsSuperGlue(dict(hp)).eval()
    m.load_state_dict({k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in sd.items()}, strict=True)
    return m.cuda()


def _cuda(data):
    return {k: torch.from_numpy(v).cuda() for k, v in data.items()}


def _check_against(out, ref, tag, frames=None):
    """out: batched dict from the CUDA path (torch, cuda); ref: oracle dict (torch cpu).  frames: rows of `out` that `ref` holds."""
    sel = slice(None) if frames is None else torch.as_tensor(frames)
    conf = out["conf_matrix"][sel].cpu()
    rc = ref["conf_matrix"]
    err = float((conf - rc).abs().max())
    assert err <= CONF_TOL, f"{tag}: max|dconf| = {err:.3e}"
    np.testing.assert_array_equal(out["matches0"][sel].cpu().numpy(), ref["matches0"].numpy(), err_msg=tag)
    np.testing.assert_array_equal(out["matches1"][sel].cpu().numpy(), ref["matches1"].numpy(), err_msg=tag)
    np.testing.assert_allclose(out["matching_scores0"][sel].cpu().numpy(), ref["matching_scores0"].numpy(), atol=CONF_TOL)
    np.testing.assert_allclose(out["matching_scores1"][sel].cpu().numpy(), ref["matching_scores1"].numpy(), atol=CONF_TOL)
    # raw arg-max (before mutual/threshold): must agree wherever the oracle's decision is not a
    # floating-point coin flip (top-1 vs top-2 separated by more than 1e-5 relative)
    top2 = rc.topk(2, dim=2).values
    decided = (top2[..., 0] - top2[..., 1]) > 1e-5 * top2[..., 0]
    mine = conf.argmax(2)
    assert bool((mine == ref["raw_indices0"])[decided].all()), tag
    top2c = rc.topk(2, dim=1).values
    decided_c = (top2c[:, 0] - top2c[:, 1]) > 1e-5 * top2c[:, 0]
    assert bool((conf.argmax(1) == ref["raw_indices1"])[decided_c].all()), tag
    return err


# ----------------------------------------------------------------------------- golden vectors of the reference module
@pytest.mark.parametrize("name", RELEASED_CASES)
def test_golden_reference_outputs(name):
    g, hp, sd, data = load_case(name)
    m = _module(sd, hp)
    pred, conf = m(_cuda(data))
    ref_conf, mine = conf_reference_view(g, conf.cpu().numpy())
    assert np.abs(ref_conf - mine).max() <= CONF_TOL
    assert pred["matches0"].dtype == torch.int64 and pred["matching_scores0"].dtype == torch.float32
    np.testing.assert_array_equal(pred["matches0"].cpu().numpy(), g["matches0"])      # bit-exact
    np.testing.assert_array_equal(pred["matches1"].cpu().numpy(), g["matches1"])
    np.testing.assert_allclose(pred["matching_scores0"].cpu().numpy(), g["matching_scores0"], atol=CONF_TOL)
    np.testing.assert_allclose(pred["matching_scores1"].cpu().numpy(), g["matching_scores1"], atol=CONF_TOL)
    assert tuple(conf.shape) == (len(g["meta_frames"]), int(g["meta_N"]), int(g["meta_M"]))


@pytest.mark.parametrize("name", ["noself_n64_m96", "additional_n64_m96", "lintrans_n64_m96", "noself_lintrans_n64_m96"])
def test_gats_variants_golden(name):
    """Every GraphAttentionLayer branch (GATs.py:48-67): include_self / additional / with_linear_transform."""
    g, hp, sd, data = load_case(name)
    m = _module(sd, hp)
    pred, conf = m(_cuda(data))
    assert np.abs(g["conf_matrix"] - conf.cpu().numpy()).max() <= CONF_TOL
    np.testing.assert_array_equal(pred["matches0"].cpu().numpy(), g["matches0"])
    np.testing.assert_array_equal(pred["matches1"].cpu().numpy(), g["matches1"])


def test_linear_transform_with_additional_vs_oracle():
    """with_linear_transform + additional (GATs.py:56-62) has no golden: compare with the oracle on a batch."""
    hp = dict(synthetic.DEFAULT_HPARAMS, with_linear_transform=True, additional=True)
    sd = synthetic.make_state_dict(5, hparams=hp)
    data = synthetic.make_batch(3, [1, 2, 3], 150, 300, 6)
    ref = oracle.forward(oracle.params_from_numpy(sd), data, hp)
    m = _module(sd, hp)
    m(_cuda(data))
    _check_against(m.last_batched, ref, "lintrans+additional")


def test_dustbin_object_exact_ties():
    """Object built by the reference's feature construction: all-ones dustbin leaves, duplicate all-ones padded 3D points
    (data_utils.py:157,202) -> exactly tied confidences; torch.max keeps the FIRST maximum and so must the packed arg-max."""
    g, hp, sd, data = load_dustbin_case()
    m = _module(sd, hp)
    pred, conf = m(_cuda(data))
    conf = conf.cpu().numpy()
    assert np.abs(conf - g["conf_matrix"]).max() <= CONF_TOL
    np.testing.assert_array_equal(pred["matches0"].cpu().numpy(), g["matches0"])
    np.testing.assert_array_equal(pred["matches1"].cpu().numpy(), g["matches1"])
    n_real = int(g["n_real"])
    assert (conf[0][:, n_real:] == conf[0][:, n_real:n_real + 1]).all()               # the tie is exact here as well
    # rows whose maximum is attained on the tied block: the first tied column wins, like torch.max
    tied_rows = g["raw_indices0"][0] >= n_real
    np.testing.assert_array_equal(conf.argmax(2)[0][tied_rows], g["raw_indices0"][0][tied_rows])


# ----------------------------------------------------------------------------- oracle on seeded inputs
@pytest.mark.parametrize("B,N,M,L,damped", [(3, 300, 700, 8, True), (1, 129, 257, 5, True), (2, 17, 40, 8, False),
                                            (5, 256, 384, 8, True), (2, 203, 333, 8, True), (1, 64, 100, 1, True), (2, 90, 150, 12, True)])
def test_oracle_parity_batched(B, N, M, L, damped):
    hp = dict(synthetic.DEFAULT_HPARAMS)
    sd = synthetic.make_state_dict(4, damped=damped)
    data = synthetic.make_batch(9, list(range(100, 100 + B)), N, M, L)
    ref = oracle.forward(oracle.params_from_numpy(sd), data, hp)
    m = _module(sd, hp)
    m.set_chunk_frames(2)            # exercise the chunk loop (3 = 2 + 1)
    m(_cuda(data))
    _check_against(m.last_batched, ref, f"B{B} N{N} M{M} L{L}")


def test_different_objects_in_one_batch():
    """The reference forward accepts per-element 3D descriptors; the drop-in groups by object."""
    hp = dict(synthetic.DEFAULT_HPARAMS)
    sd = synthetic.make_state_dict(0)
    d1 = synthetic.make_batch(1, [5, 6], 96, 160, 8)
    d2 = synthetic.make_batch(2, [7], 96, 160, 8)
    data = {k: np.concatenate([d1[k], d2[k]], 0) for k in d1}
    ref = oracle.forward(oracle.params_from_numpy(sd), data, hp)
    m = _module(sd, hp)
    pred, conf = m(_cuda(data))
    _check_against(m.last_batched, ref, "mixed objects")


def test_metric_shape_one_frame_vs_oracle():
    """BASELINE metric shape N2D=1024, N3D=7000 (one frame: the oracle needs ~1-2 s of CPU)."""
    hp = dict(synthetic.DEFAULT_HPARAMS)
    sd = synthetic.make_state_dict(0)
    data = synthetic.make_batch(7, [70], 1024, 7000, 8)
    ref = oracle.forward(oracle.params_from_numpy(sd), data, hp)
    m = _module(sd, hp)
    m(_cuda(data))
    err = _check_against(m.last_batched, ref, "metric shape")
    assert int((m.last_batched["matches0"] > -1).sum()) >= 400      # planted correspondences recovered
    print(f"metric-shape max|dconf| = {err:.2e}")


def test_benched_configuration_vs_oracle():
    """The call bench.py times: B=32 frames of one object, chunk 32, N2D=1024, N3D=7000, through match_frames (device) and
    match_frames_host (pinned host in, 16-frame H2D pieces).  Frames 0, 15, 16, 31 (the piece boundaries) meet the oracle."""
    hp = dict(synthetic.DEFAULT_HPARAMS)
    sd = synthetic.make_state_dict(0)
    B, N, M = 32, 1024, 7000
    db, leaves = synthetic.make_object(0, M, 8)
    q = np.stack([synthetic.make_frame(1000 + f, db, N)[0] for f in range(B)], 0)
    frames = [0, 15, 16, 31]
    data = {"keypoints2d": np.zeros((len(frames), N, 2), np.float32), "keypoints3d": np.zeros((len(frames), M, 3), np.float32),
            "descriptors2d_query": q[frames], "descriptors3d_db": np.repeat(db[None], len(frames), 0),
            "descriptors2d_db": np.repeat(leaves[None], len(frames), 0)}
    ref = oracle.forward(oracle.params_from_numpy(sd), data, hp)
    m = _module(sd, hp)
    m.set_object(torch.from_numpy(db).cuda(), torch.from_numpy(leaves).cuda(), reserve=(B, N))
    qt = torch.from_numpy(q)
    dev = m.match_frames(qt.cuda())
    err = _check_against(dev, ref, "bench config (device)", frames)
    host = m.match_frames_host(qt.pin_memory())
    for k in ("matches0", "matches1", "matching_scores0", "matching_scores1"):
        assert torch.equal(host[k], dev[k].cpu()), k
    # return_conf=False (what inference.py:146 needs): same matches, no confidence matrix
    lean = m.match_frames(qt.cuda(), return_conf=False)
    assert lean["conf_matrix"] is None
    for k in ("matches0", "matches1", "matching_scores0", "matching_scores1"):
        assert torch.equal(lean[k], dev[k]), k
    m.check_range()
    print(f"bench-config max|dconf| = {err:.2e}")


def test_dense_stress_shape_vs_oracle():
    """BASELINE configs[3]: N2D=2000, N3D=15000 (dual-softmax + mutual-NN at the largest size the survey names)."""
    hp = dict(synthetic.DEFAULT_HPARAMS)
    sd = synthetic.make_state_dict(0)
    data = synthetic.make_batch(11, [90], 2000, 15000, 8)
    ref = oracle.forward(oracle.params_from_numpy(sd), data, hp)
    m = _module(sd, hp)
    m(_cuda(data))
    err = _check_against(m.last_batched, ref, "dense stress")
    assert int((m.last_batched["matches0"] > -1).sum()) == int((ref["matches0"] > -1).sum()) > 500
    print(f"dense-stress max|dconf| = {err:.2e}")


@pytest.mark.parametrize("N,M", [(4096, 1030), (70, 1001)])
def test_reference_edge_shapes(N, M):
    """N = 4096 (SuperPoint's cap, extract_features.py:19-24); M % 4 != 0 (the confidence matrix leaves through plain
    stores instead of the 3-D tensor map); with and without the confidence matrix."""
    hp = dict(synthetic.DEFAULT_HPARAMS)
    sd = synthetic.make_state_dict(0)
    data = synthetic.make_batch(13, [5, 6], N, M, 8)
    ref = oracle.forward(oracle.params_from_numpy(sd), data, hp)
    m = _module(sd, hp)
    m(_cuda(data))
    _check_against(m.last_batched, ref, f"edge N{N} M{M}")
    lean = m.match_frames(torch.from_numpy(data["descriptors2d_query"]).cuda(), return_conf=False)
    for k in ("matches0", "matches1", "matching_scores0", "matching_scores1"):
        assert torch.equal(lean[k], m.last_batched[k]), k


def test_ragged_query_lengths_in_one_call():
    """Frames with different numbers of query points in ONE call (opb_forward n2d_lengths): every frame equals the oracle run
    on its own valid columns; entries beyond a frame's length are -1 / 0."""
    hp = dict(synthetic.DEFAULT_HPARAMS)
    sd = synthetic.make_state_dict(0)
    M, L, Nmax = 500, 8, 300
    lens = [300, 37, 256, 1, 129]
    db, leaves = synthetic.make_object(3, M, L)
    q = np.zeros((len(lens), 256, Nmax), np.float32)
    refs = []
    for b, n in enumerate(lens):
        qb, _ = synthetic.make_frame(40 + b, db, n)
        q[b, :, :n] = qb
        q[b, :, n:] = 7.0                                   # garbage beyond the length must be ignored
        data = {"keypoints2d": np.zeros((1, n, 2), np.float32), "keypoints3d": np.zeros((1, M, 3), np.float32),
                "descriptors2d_query": qb[None], "descriptors3d_db": db[None], "descriptors2d_db": leaves[None]}
        refs.append(oracle.forward(oracle.params_from_numpy(sd), data, hp))
    m = _module(sd, hp)
    m.set_chunk_frames(2)
    m.set_object(torch.from_numpy(db).cuda(), torch.from_numpy(leaves).cuda())
    out = m.match_frames(torch.from_numpy(q).cuda(), lengths=torch.tensor(lens, dtype=torch.int32))
    for b, n in enumerate(lens):
        ref = refs[b]
        conf = out["conf_matrix"][b].cpu()
        assert float((conf[:n] - ref["conf_matrix"][0]).abs().max()) <= CONF_TOL, b
        assert float(conf[n:].abs().max()) == 0.0 if n < Nmax else True
        np.testing.assert_array_equal(out["matches0"][b, :n].cpu().numpy(), ref["matches0"][0].numpy())
        np.testing.assert_array_equal(out["matches1"][b].cpu().numpy(), ref["matches1"][0].numpy())
        assert bool((out["matches0"][b, n:] == -1).all()) and float(out["matching_scores0"][b, n:].abs().sum()) == 0.0
        np.testing.assert_allclose(out["matching_scores1"][b].cpu().numpy(), ref["matching_scores1"][0].numpy(), atol=CONF_TOL)
    # host-buffer entry point with lengths
    host = m.match_frames_host(torch.from_numpy(q).pin_memory(), lengths=torch.tensor(lens, dtype=torch.int32))
    assert torch.equal(host["matches0"], out["matches0"].cpu()) and torch.equal(host["matches1"], out["matches1"].cpu())


def test_long_lived_handle_ragged_sequence():
    """inference.py's pattern: ONE handle, hundreds of B=1 forward(data) calls with a different N every frame (N % 256 != 0),
    the object tensors re-passed each time.  Padding rows must not accumulate state across calls (a stale pad row would
    eventually leave the operand range), and results must stay equal to the oracle."""
    hp = dict(synthetic.DEFAULT_HPARAMS)
    sd = synthetic.make_state_dict(2, damped=False)        # undamped: residual updates are O(1)
    M, L = 300, 8
    db, leaves = synthetic.make_object(8, M, L)
    m = _module(sd, hp)
    d3 = torch.from_numpy(db)[None].cuda()
    d2 = torch.from_numpy(leaves)[None].cuda()
    k3 = torch.zeros(1, M, 3).cuda()
    rs = np.random.RandomState(0)
    P = oracle.params_from_numpy(sd)
    for it in range(260):
        n = int(rs.randint(30, 520))
        qn, _ = synthetic.make_frame(5000 + it, db, n)
        data = {"keypoints2d": torch.zeros(1, n, 2).cuda(), "keypoints3d": k3, "descriptors2d_query": torch.from_numpy(qn)[None].cuda(),
                "descriptors3d_db": d3, "descriptors2d_db": d2}
        pred, conf = m(data)
        if it % 37 == 0 or it == 259:
            ref = oracle.forward(P, {k: v.cpu().numpy() for k, v in data.items()}, hp)
            _check_against(m.last_batched, ref, f"call {it} N={n}")
    m.check_range()                                         # no call left the operand range


def test_full_size_properties():
    """Size-independent properties at the bench configuration (B=8 frames of one object)."""
    hp = dict(synthetic.DEFAULT_HPARAMS)
    sd = synthetic.make_state_dict(0)
    B, N, M = 8, 1024, 7000
    data = synthetic.make_batch(7, list(range(70, 70 + B)), N, M, 8)
    m = _module(sd, hp)
    m(_cuda(data))
    out = m.last_batched
    conf = out["conf_matrix"]
    # softmax factors: row sums of conf <= max col-softmax <= 1, every entry in [0, 1]
    assert float(conf.min()) >= 0.0 and float(conf.max()) <= 1.0 + 1e-6
    assert float(conf.sum(2).max()) <= 1.0 + 1e-4 and float(conf.sum(1).max()) <= 1.0 + 1e-4
    m0, m1 = out["matches0"], out["matches1"]
    ar = torch.arange(N, device=conf.device)[None].expand(B, N)
    valid = m0 > -1
    # mutual consistency: matches1[matches0[n]] == n for valid n; scores agree with conf
    assert bool((m1.gather(1, m0.clamp_min(0))[valid] == ar[valid]).all())
    picked = conf.gather(2, m0.clamp_min(0)[..., None])[..., 0]
    assert torch.equal(picked[valid], out["matching_scores0"][valid])
    assert bool((out["matching_scores0"][valid] > hp["match_threshold"]).all())
    # frame b of a batch == the same frame run alone (frames are independent)
    solo = _module(sd, hp)
    one = {k: v[3:4] for k, v in data.items()}
    solo(_cuda(one))
    assert torch.equal(solo.last_batched["matches0"][0], m0[3])
    assert float((solo.last_batched["conf_matrix"][0] - conf[3]).abs().max()) <= 1e-6
    # planted correspondences (first N/2 queries) are found
    for b in range(B):
        _, perm = synthetic.make_frame(70 + b, data["descriptors3d_db"][0], N)
        got = m0[b, : N // 2].cpu().numpy()
        assert (got == perm).mean() > 0.95


# ----------------------------------------------------------------------------- kernels in isolation
def test_kv_state_row_groups_are_equivalent():
    """The linear-attention state kernel with 1, 2 and 5 slabs per row group: the per-segment sums agree to fp32 rounding."""
    lib = _lib.load()
    frames, n, m_pts = 2, 300, 1500
    n_pad, m_pad = 512, 1536
    rs = np.random.RandomState(1)
    kvh = np.zeros((frames * (n_pad + m_pad), 512), np.float16)
    for b in range(frames):
        base = b * (n_pad + m_pad)
        kvh[base:base + n] = (rs.rand(n, 512) * 64).astype(np.float16)
        kvh[base + n_pad:base + n_pad + m_pts] = (rs.rand(m_pts, 512) * 64).astype(np.float16)
    kv = torch.from_numpy(kvh).cuda()
    sums = []
    for slabs in (1, 2, 5):
        ng = C.c_int32()
        assert lib.opb_debug_kv_state_h(kv.data_ptr(), frames, n, m_pts, slabs, None, C.byref(ng), None) == 0
        part = torch.zeros(ng.value, 4, 64 * 64 + 64, dtype=torch.float32, device="cuda")
        assert lib.opb_debug_kv_state_h(kv.data_ptr(), frames, n, m_pts, slabs, part.data_ptr(), C.byref(ng), None) == 0
        torch.cuda.synchronize()
        gq, gd = -(-(n_pad // 256) // slabs), -(-(m_pad // 256) // slabs)
        p = part.cpu().double().reshape(frames, gq + gd, 4, -1)
        sums.append(torch.stack([p[:, :gq].sum(1), p[:, gq:].sum(1)], 1))     # [frames, side, head, 4160]
    kf = torch.from_numpy(kvh.astype(np.float64)) / 64.0
    for b in range(frames):
        base = b * (n_pad + m_pad)
        for side, (r0, cnt) in enumerate([(base, n), (base + n_pad, m_pts)]):
            K, V = kf[r0:r0 + cnt, :256], kf[r0:r0 + cnt, 256:]
            for h in range(4):
                ref = torch.cat([(K[:, h * 64:(h + 1) * 64].T @ V[:, h * 64:(h + 1) * 64]).reshape(-1), K[:, h * 64:(h + 1) * 64].sum(0)])
                for s in sums:
                    assert float((s[b, side, h] - ref).abs().max() / ref.abs().max()) < 1e-5
    assert float((sums[0] - sums[1]).abs().max() / sums[0].abs().max()) < 1e-5
    assert float((sums[0] - sums[2]).abs().max() / sums[0].abs().max()) < 1e-5


@pytest.mark.parametrize("name", ["mean_descriptors_m300", "mean_tracks_long_m48"])
def test_segmented_means_match_reference_golden(name):
    """mean_descriptors / mean_scores on the GPU: bit-identical to the reference's numpy results (fp64, numpy's summation order)."""
    g = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    desc, idxs = synthetic.make_tracks(int(g["seed"]), int(g["M"]), max_len=int(g["max_len"]))
    scores = synthetic.make_track_scores(int(g["seed"]), idxs)
    avg = features3d.mean_descriptors(desc, idxs)
    avg_s = features3d.mean_scores(scores, idxs)
    assert avg.dtype == torch.float64 and tuple(avg_s.shape) == (len(idxs), 1)
    np.testing.assert_array_equal(avg.cpu().numpy(), g["avg"])
    np.testing.assert_array_equal(avg_s.cpu().numpy(), g["avg_scores"])


def test_features3d_construction_matches_reference_golden():
    """pad_features3d_random / build_features3d_leaves on the GPU: byte-identical tensors to the imported reference functions
    under the same np.random.seed (data_utils.py:143-205), incl. dustbin fill, truncation and all-ones padding."""
    g = np.load(os.path.join(GOLDEN_DIR, "features3d_n40_l8.npz"))
    obs, obs_scores, idxs, avg, avg_scores = synthetic.make_sfm_features(int(g["seed"]), int(g["n_points"]))
    for tag in ("same", "pad", "trunc"):
        nt = int(g[f"{tag}_n_target"])
        d3, s3 = features3d.pad_features3d_random(avg, avg_scores, nt)
        np.random.seed(int(g["np_seed"]))
        d2, s2 = features3d.build_features3d_leaves(obs, obs_scores, idxs, nt, int(g["num_leaf"]))
        for mine, key in ((d3, "desc3d"), (s3, "scores3d"), (d2, "desc2d"), (s2, "scores2d")):
            ref = g[f"{tag}_{key}"]
            assert mine.is_cuda and mine.dtype == torch.float32 and tuple(mine.shape) == ref.shape, (tag, key)
            assert mine.cpu().numpy().tobytes() == ref.tobytes(), (tag, key)


def test_ransac_pnp_matches_reference_poses():
    """GPU RANSAC-PnP vs the reference's ransac_PnP (cv2.solvePnPRansac EPnP, eval_utils.py:18-42) on seeded scenes with 20-60 %
    outliers: the pose agrees with the reference's and with the ground truth under the reference's own cm-degree metric
    (parity on the pose, not on bits: OpenCV draws its own samples); inlier sets are as large; degenerate inputs give the
    reference's identity / [] result; repeated calls are deterministic."""
    from onepose_b200 import pnp
    from oracle import pnp_oracle
    g = np.load(os.path.join(GOLDEN_DIR, "pnp_scenes.npz"))
    scenes = [(int(s), int(n), float(f)) for s, n, f in g["scenes"]]
    for seed, n, frac in scenes:
        K, uv, P, gt = synthetic.make_pnp_scene(seed, n, frac)
        pose, homo, inliers = pnp.ransac_PnP(K, uv, P, scale=1000)
        ref = g[f"pose_{seed}"]
        if n < 4:
            assert np.array_equal(pose, np.eye(4)[:3]) and len(inliers) == 0 and int(g[f"n_inliers_{seed}"]) == 0
            continue
        r_gt, t_gt = pnp_oracle.pose_error(pose, gt)
        r_ref, t_ref = pnp_oracle.pose_error(pose, ref)
        rr_gt, tr_gt = pnp_oracle.pose_error(ref, gt)
        print(f"pnp scene {seed}: n={n}: ours vs gt {r_gt:.3f} deg {t_gt:.3f} cm | reference vs gt {rr_gt:.3f} deg {tr_gt:.3f} cm | "
              f"inliers {len(inliers)} vs {int(g[f'n_inliers_{seed}'])}")
        if n >= 30:
            assert r_gt < 1.0 and t_gt < 1.0                        # cmd1 of the reference evaluator
            assert r_ref < 0.5 and t_ref < 0.5
        if n >= 100:                                                # enough inliers for the two estimators to be compared
            assert r_gt <= rr_gt + 0.15 and t_gt <= tr_gt + 0.15   # as accurate as the reference's estimate
        assert len(inliers) >= 0.97 * int(g[f"n_inliers_{seed}"])
        assert homo.shape == (4, 4) and np.allclose(homo[3], [0, 0, 0, 1])
    # batched call == per-frame calls, deterministic
    Ks, uvs, Ps, off = [], [], [], [0]
    for seed, n, frac in scenes[:5]:
        K, uv, P, gt = synthetic.make_pnp_scene(seed, n, frac)
        Ks.append(K); uvs.append(uv); Ps.append(P * 1000); off.append(off[-1] + n)
    args = (torch.from_numpy(np.stack(Ks)).cuda(), torch.from_numpy(np.concatenate(uvs)).cuda(), torch.from_numpy(np.concatenate(Ps)).cuda(),
            torch.tensor(off, dtype=torch.int32).cuda())
    pose_a, mask_a, cnt_a = pnp.ransac_pnp_batch(*args)
    pose_b, mask_b, cnt_b = pnp.ransac_pnp_batch(*args)
    assert torch.equal(pose_a, pose_b) and torch.equal(mask_a, mask_b) and torch.equal(cnt_a, cnt_b)
    for i, (seed, n, frac) in enumerate(scenes[:5]):
        single, _, inl = pnp.ransac_PnP(Ks[i], uvs[i], Ps[i] / 1000, scale=1000)
        batched = pose_a[i].cpu().numpy().copy()
        batched[:, 3] /= 1000
        np.testing.assert_allclose(batched, single, atol=1e-12)
        assert int(cnt_a[i]) == len(inl)


# ----------------------------------------------------------------------------- host logic on the device path
def test_object_prologue_hoisting_matches_per_frame_evaluation():
    """Layers 0-1 of the 3D side are frame-invariant: evaluating them once per call (default) must give the
    same answer as evaluating them per frame like the reference (GATs_SuperGlue.py:50-64)."""
    hp = dict(synthetic.DEFAULT_HPARAMS)
    sd = synthetic.make_state_dict(0)
    data = synthetic.make_batch(4, [1, 2, 3], 200, 500, 8)
    ref = oracle.forward(oracle.params_from_numpy(sd), data, hp)
    outs = []
    for hoist in (True, False):
        m = _module(sd, hp)
        m.set_hoist(hoist)
        m.set_chunk_frames(2)
        m(_cuda(data))
        _check_against(m.last_batched, ref, f"hoist={hoist}")
        outs.append(m.last_batched)
    assert float((outs[0]["conf_matrix"] - outs[1]["conf_matrix"]).abs().max()) <= 2e-6
    assert torch.equal(outs[0]["matches0"], outs[1]["matches0"])


def test_results_do_not_depend_on_uninitialised_workspace():
    """Every workspace / object buffer poisoned with 0xFF bytes (NaN patterns) at allocation: same results as the oracle, for
    ragged sizes, growing workspaces and both GATs code paths (only the block-diagonal state operand is required to start zero)."""
    lib = _lib.load()
    hp = dict(synthetic.DEFAULT_HPARAMS)
    sd = synthetic.make_state_dict(1)
    try:
        assert lib.opb_debug_set_ws_fill(0xFF) == 0
        m = _module(sd, hp)
        for obj, (B, N, M, L) in enumerate([(2, 100, 300, 8), (3, 333, 700, 8), (1, 50, 129, 5), (2, 260, 513, 8)]):
            data = synthetic.make_batch(30 + obj, list(range(B)), N, M, L)
            ref = oracle.forward(oracle.params_from_numpy(sd), data, hp)
            m(_cuda(data))
            _check_against(m.last_batched, ref, f"poisoned workspace, object {obj}")
        m.check_range()
    finally:
        lib.opb_debug_set_ws_fill(-1)


def test_programmatic_dependent_launch_is_transparent():
    """PDL on (default) and off give bit-identical results (it only overlaps kernel prologues with the previous kernel's tail)."""
    lib = _lib.load()
    hp = dict(synthetic.DEFAULT_HPARAMS)
    sd = synthetic.make_state_dict(0)
    data = _cuda(synthetic.make_batch(6, [3, 4, 5], 333, 700, 8))
    outs = []
    try:
        for on in (1, 0):
            assert lib.opb_debug_set_pdl(on) == 0
            m = _module(sd, hp)
            m(data)
            m(data)
            outs.append({k: v.clone() for k, v in m.last_batched.items()})
    finally:
        lib.opb_debug_set_pdl(1)
    for k in outs[0]:
        assert torch.equal(outs[0][k], outs[1][k]), k


def test_kv_projection_two_vs_three_passes():
    """The k,v projection runs as A_hi.(B_hi + B_lo) (its output is one fp16 plane; the dropped A_lo term is below that rounding
    and averages out over the segment's rows).  Against the full three-pass product: same matches, conf within 2e-6; both
    meet the oracle -- with the damped fixtures and with undamped weights (O(1) residual updates)."""
    lib = _lib.load()
    hp = dict(synthetic.DEFAULT_HPARAMS)
    for damped, shape in ((True, (2, 300, 900)), (False, (2, 200, 500))):
        sd = synthetic.make_state_dict(3, damped=damped)
        B, N, M = shape
        data = synthetic.make_batch(21, list(range(B)), N, M, 8)
        ref = oracle.forward(oracle.params_from_numpy(sd), data, hp)
        outs = []
        for passes in (2, 3):
            m = _module(sd, hp)
            m._ensure_handle(torch.device("cuda", 0))
            assert lib.opb_debug_set_kv_passes(m._handle, passes) == 0
            m(_cuda(data))
            _check_against(m.last_batched, ref, f"kv passes {passes} damped={damped}")
            outs.append(m.last_batched)
        assert torch.equal(outs[0]["matches0"], outs[1]["matches0"])
        scale = float(outs[1]["conf_matrix"].max())
        assert float((outs[0]["conf_matrix"] - outs[1]["conf_matrix"]).abs().max()) <= 4e-6 * max(scale, 1e-3)


def test_host_buffer_call_equals_device_call():
    """opb_forward_host (pinned host in / host out, chunked H2D on a side stream) == opb_forward on device tensors."""
    hp = dict(synthetic.DEFAULT_HPARAMS)
    sd = synthetic.make_state_dict(0)
    data = synthetic.make_batch(8, list(range(5)), 260, 600, 8)
    m = _module(sd, hp)
    m.set_chunk_frames(2)                       # 3 chunks: 2 + 2 + 1
    m.set_object(torch.from_numpy(data["descriptors3d_db"][0]).cuda(), torch.from_numpy(data["descriptors2d_db"][0]).cuda())
    q = torch.from_numpy(data["descriptors2d_query"])
    dev = m.match_frames(q.cuda())
    for conf_on in (True, False):               # second call reuses the staging buffers / events
        host = m.match_frames_host(q.pin_memory(), materialize_conf=conf_on)
        for k in ("matches0", "matches1", "matching_scores0", "matching_scores1"):
            assert torch.equal(host[k], dev[k].cpu()), k
    ref = oracle.forward(oracle.params_from_numpy(sd), data, hp)
    np.testing.assert_array_equal(host["matches0"].numpy(), ref["matches0"].numpy())


def test_object_cache_follows_tensor_identity_and_content():
    """forward(data) packs the per-object tensors once: same tensors -> no work; a fresh copy with the same content -> no
    re-pack; an in-place change of the SAME tensor (same data_ptr, new version) or a different object -> re-pack."""
    hp = dict(synthetic.DEFAULT_HPARAMS)
    sd = synthetic.make_state_dict(0)
    m = _module(sd, hp)
    packs = []
    orig = m.set_object
    m.set_object = lambda *a, **k: (packs.append(1), orig(*a, **k))[1]
    dA = _cuda(synthetic.make_batch(1, [5], 96, 160, 8))
    dB = synthetic.make_batch(2, [5], 96, 160, 8)
    P = oracle.params_from_numpy(sd)
    refA = oracle.forward(P, {k: v.cpu().numpy() for k, v in dA.items()}, hp)
    refB = oracle.forward(P, dB, hp)
    m(dA); m(dA)
    assert len(packs) == 1
    _check_against(m.last_batched, refA, "object A")
    dA2 = {k: v.clone() for k, v in dA.items()}              # new storage, same content (pack_data's .cuda() every frame)
    m(dA2)
    assert len(packs) == 1
    dA2["descriptors3d_db"].copy_(torch.from_numpy(dB["descriptors3d_db"]).cuda())      # same tensor, new content
    dA2["descriptors2d_db"].copy_(torch.from_numpy(dB["descriptors2d_db"]).cuda())
    dA2["descriptors2d_query"] = torch.from_numpy(dB["descriptors2d_query"]).cuda()
    m(dA2)
    assert len(packs) == 2
    _check_against(m.last_batched, refB, "object B in A's storage")
    m(dA)
    assert len(packs) == 3
    _check_against(m.last_batched, refA, "back to object A")


def test_operand_range_guard_is_lazy_and_poisons_matches():
    """Activations beyond the fp16-split operand range (|x| >= 1023) must be reported, not silently wrong: the call itself
    returns "no match" everywhere without blocking, and the error reaches the host at check_range() / on a later call."""
    hp = dict(synthetic.DEFAULT_HPARAMS)
    sd = synthetic.make_state_dict(0)
    sd = {k: (v * 3e4 if k.endswith("mlp.3.weight") else v) for k, v in sd.items()}     # residual stream explodes
    m = _module(sd, hp)
    data = _cuda(synthetic.make_batch(1, [1], 128, 256, 8))
    pred, _ = m(data)
    assert bool((pred["matches0"] == -1).all()) and bool((pred["matches1"] == -1).all())
    with pytest.raises(_lib.OpbError, match="OPB_E_RANGE"):
        m.check_range()
    m.check_range()                                          # reporting cleared the flag
    m(data)
    torch.cuda.synchronize()
    with pytest.raises(_lib.OpbError, match="OPB_E_RANGE"):   # deferred delivery on the NEXT call
        m(data)
    # a sane model on the same process still works
    ok = _module(synthetic.make_state_dict(0), hp)
    pred, _ = ok(_cuda(synthetic.make_batch(1, [1], 128, 256, 8)))
    assert int((pred["matches0"] > -1).sum()) > 0
    ok.check_range()


def test_match_frames_needs_an_object():
    m = GATsSuperGlue(dict(synthetic.DEFAULT_HPARAMS)).cuda()
    with pytest.raises(RuntimeError, match="set_object"):
        m.match_frames(torch.zeros(1, 256, 8, device="cuda"))


def test_repeat_calls_are_deterministic():
    hp = dict(synthetic.DEFAULT_HPARAMS)
    sd = synthetic.make_state_dict(0)
    data = _cuda(synthetic.make_batch(3, [1, 2], 200, 500, 8))
    m = _module(sd, hp)
    m(data)
    a = {k: v.clone() for k, v in m.last_batched.items()}
    m(data)
    for k, v in m.last_batched.items():
        assert torch.equal(a[k], v), k
