"""The per-object feature producers on the device against numpy and the oracle, byte for byte, and the objects they build run
through the matcher's stage walk.

Means: features3d.mean_descriptors / mean_scores against oracle.mean_descriptors / mean_scores, which run np.mean per slice
as the reference does -- numpy itself, in whatever layout the caller hands over (tests/test_features3d_cpu.py pins numpy's
rule).  NaN exactly where numpy has NaN (a zero-length track), every other value bit-equal.

Gather: pad_features3d_random / build_features3d_leaves against the oracle under the same np.random.seed: byte-identical
tensors, and the global RNG left in the same state.

Producer-built objects: averaged 3D descriptors (norm below 1), random leaf picks and all-ones dustbin leaves (norm 16) for
every track shorter than L -- the objects the reference's inference.py feeds the matcher -- through the stage walk of
tests/test_matcher_stages_gpu.py with its bars unchanged, and an object padded with all-ones points whose tied conf
columns span several of the score GEMM's column tiles."""
import gc
import time
import warnings

import numpy as np
import pytest
import torch

from onepose_b200 import _lib, features3d, synthetic
from oracle import gats_spg_oracle as oracle
from tests import matcher_stage_reference as ref
from tests.test_features3d_cpu import LENGTHS, wide
from tests.test_matcher_config_gpu import _decided_mismatches
from tests.test_matcher_stages_gpu import Stages, _module

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------ means
def _numpy_means(x, idxs):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)         # np.mean of a zero-length track: NaN and a warning
        return oracle.mean_descriptors(x, idxs).reshape(len(idxs), -1)


def _assert_same(got, want, tag):
    got = got.cpu().numpy() if isinstance(got, torch.Tensor) else got
    assert got.dtype == np.float64 and got.shape == want.shape, (tag, got.dtype, got.shape, want.shape)
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan), f"{tag}: NaN at {int((np.isnan(got) != nan).sum())} other places"
    bad = got.view(np.int64)[~nan] != want.view(np.int64)[~nan]
    assert not bad.any(), f"{tag}: {int(bad.sum())} of {bad.size} values differ from numpy"


# name: (view of a base array -> [sum(len), D] of the same values; the same view applies to a CUDA copy of the base)
LAYOUTS = {
    "C": (lambda n, D: (n, D), lambda b, D: b),
    "F": (lambda n, D: (D, n), lambda b, D: b.T),
    "row_strided": (lambda n, D: (2 * n, D), lambda b, D: b[::2]),
    "column_sliced": (lambda n, D: (n, D + 2), lambda b, D: b[:, 1:D + 1]),
    "F_row_strided": (lambda n, D: (D, 2 * n), lambda b, D: b.T[::2]),
}


def _check_means(idxs, D, layout, source, rs, fill=None):
    shape, view = LAYOUTS[layout]
    n = int(np.sum(idxs))
    base = wide(rs, *shape(n, D)) if fill is None else np.full(shape(n, D), fill)
    x = view(base, D)
    want = _numpy_means(x, idxs)
    arg = x if source == "numpy" else view(torch.from_numpy(base).cuda(), D)
    fns = (features3d.mean_descriptors, features3d.mean_scores) if D == 1 else (features3d.mean_descriptors,)
    for fn in fns:
        _assert_same(fn(arg, idxs), want, f"{fn.__name__} {layout} {source} D={D} M={len(idxs)}")


@pytest.mark.parametrize("source", ["numpy", "cuda"])
@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("D", [1, 3, 31, 32, 33, 256, 257])
def test_means_equal_numpy_in_every_layout(D, layout, source):
    """Tracks of 1-17 and 63-65 rows, and zero-length tracks between them."""
    idxs = np.array(list(range(1, 18)) + [0, 63, 64, 0, 65, 0], np.int64)
    _check_means(idxs, D, layout, source, np.random.RandomState(D))


@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("D", [1, 3])
def test_means_equal_numpy_at_long_tracks(D, layout):
    """Lengths where the pairwise split recurses: 127-129, 135-137, 255-257, 1023-1025, 8191-8193, 20000."""
    _check_means(np.array(LENGTHS, np.int64), D, layout, "cuda", np.random.RandomState(7))


@pytest.mark.parametrize("layout", ["C", "F"])
def test_means_at_one_track_and_at_70000(layout):
    """M = 1, and M = 70000 (each thread of the offsets scan sums 69 lengths)."""
    rs = np.random.RandomState(3)
    _check_means(np.array([9], np.int64), 4, layout, "numpy", rs)
    _check_means(rs.randint(0, 7, 70000).astype(np.int64), 3, layout, "numpy", rs)


@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_means_of_negative_zero_tracks_are_positive_zero(layout):
    """All -0.0 tracks of 1-20 and 130 rows: +0.0, as numpy's identity add gives."""
    idxs = np.array(list(range(1, 21)) + [130], np.int64)
    for D in (1, 3):
        _check_means(idxs, D, layout, "numpy", None, fill=-0.0)


def test_mean_scores_of_several_columns_is_numpy_mean():
    """The reference's mean_scores is the same np.mean as mean_descriptors: [sum(len), D] scores give [n_points, D]."""
    idxs = np.array([3, 9, 0, 40], np.int64)
    x = wide(np.random.RandomState(5), int(idxs.sum()), 2)
    _assert_same(features3d.mean_scores(x, idxs), _numpy_means(x, idxs), "mean_scores D=2")


def test_scores_entry_point_is_the_pairwise_one_channel_mean():
    """opb_segmented_mean_scores_f64, called directly: the D = 1 mean."""
    idxs = np.array(LENGTHS, np.int64)
    s = wide(np.random.RandomState(11), int(idxs.sum()))
    dev = torch.device("cuda")
    out = torch.empty(len(idxs), dtype=torch.float64, device=dev)
    lens = torch.from_numpy(idxs).to(dev)
    _lib.call(dev, "opb_segmented_mean_scores_f64", torch.from_numpy(s).to(dev), lens, len(idxs), out)
    _assert_same(out[:, None], _numpy_means(s[:, None], idxs), "opb_segmented_mean_scores_f64")


@pytest.mark.parametrize("make", [lambda: np.ones((9, 3), np.float32), lambda: torch.ones(9, 3, device="cuda"),
                                  lambda: torch.ones(9, 1, device="cuda", dtype=torch.float16)])
def test_means_refuse_fp32_instead_of_widening(make):
    for fn in (features3d.mean_descriptors, features3d.mean_scores):
        with pytest.raises(ValueError, match="fp64"):
            fn(make(), np.array([4, 5]))


# ------------------------------------------------------------------------------------------------ gather
TRACKS = {
    "short": lambda rs, M, L: rs.randint(1, L, M) if L > 1 else np.ones(M, np.int64),
    "long": lambda rs, M, L: rs.randint(L + 1, L + 6, M),
    "exact": lambda rs, M, L: np.full(M, L),
    "with_empty": lambda rs, M, L: rs.randint(0, 2 * L + 2, M) * (rs.rand(M) > 0.3),
    "all_empty": lambda rs, M, L: np.zeros(M, np.int64),
}

FORMS = {
    "numpy32": lambda a: a,
    "numpy64": lambda a: a.astype(np.float64) * (1.0 + 2.0 ** -30),       # fp64 values between fp32 neighbours: rounding counts
    "cpu": lambda a: torch.from_numpy(a),
    "cuda": lambda a: torch.from_numpy(a).cuda(),
    "strided": lambda a: torch.from_numpy(np.repeat(a, 2, axis=1)).cuda()[:, ::2],
}


def _oracle_input(a, form):
    """The array the reference gets: its torch.Tensor(x) turns fp64 numpy input into fp32."""
    return torch.Tensor(FORMS[form](a)).numpy() if form == "numpy64" else a


def _check_gather(dim, M, L, n_target, tracks, form, seed=0):
    rs = np.random.RandomState(seed)
    idxs = TRACKS[tracks](rs, M, L).astype(np.int64)
    n = int(idxs.sum())
    obs, obs_s = rs.randn(dim, n).astype(np.float32), rs.rand(n, 1).astype(np.float32)
    avg, avg_s = rs.randn(dim, M).astype(np.float32), rs.rand(M, 1).astype(np.float32)
    tag = f"dim={dim} M={M} L={L} n_target={n_target} {tracks} {form}"
    cases = [("pad", lambda f: features3d.pad_features3d_random(f(avg), f(avg_s), n_target),
              lambda: oracle.pad_features3d_random(_oracle_input(avg, form), _oracle_input(avg_s, form), n_target))]
    cases.append(("leaves", lambda f: features3d.build_features3d_leaves(f(obs), f(obs_s), idxs, n_target, L),
                  lambda: oracle.build_features3d_leaves(_oracle_input(obs, form), _oracle_input(obs_s, form), idxs, n_target, L)))
    for what, mine_fn, ref_fn in cases:
        np.random.seed(seed + 1)
        mine = mine_fn(FORMS[form])
        after = np.random.rand()
        np.random.seed(seed + 1)
        want = ref_fn()
        assert np.random.rand() == after, f"{what} {tag}: the global RNG was left in another state"
        for got, exp in zip(mine, want):
            assert got.is_cuda and got.dtype == torch.float32 and tuple(got.shape) == exp.shape, (what, tag, tuple(got.shape), exp.shape)
            assert got.cpu().numpy().tobytes() == np.ascontiguousarray(exp).tobytes(), f"{what} {tag}"


@pytest.mark.parametrize("num_leaf", [1, 7, 8, 9, 32])
@pytest.mark.parametrize("tracks", list(TRACKS))
def test_gather_equals_oracle_at_every_track_shape(tracks, num_leaf):
    """n_target below, equal to and above the point count (num_leaf * n_target mostly not a multiple of 256)."""
    for n_target in (29, 40, 41, 300):
        _check_gather(5, 40, num_leaf, n_target, tracks, "numpy32")


@pytest.mark.parametrize("form", list(FORMS))
@pytest.mark.parametrize("dim", [1, 3, 256, 257])
def test_gather_equals_oracle_for_every_input_form(dim, form):
    for n_target in (37, 50, 77):
        _check_gather(dim, 50, 8, n_target, "with_empty", form, seed=dim)


def test_gather_at_15000_points():
    """M = 15000, L = 8: 120000 leaf columns, with 37 points of padding."""
    _check_gather(256, 15000, 8, 15037, "with_empty", "numpy32")


def test_gather_of_zero_points_returns_empty_tensors():
    """n_target_shape = 0: the reference slices to [dim, 0] / [0, 1]; so does the device."""
    _check_gather(4, 10, 8, 0, "with_empty", "numpy32")
    _check_gather(4, 10, 8, 0, "with_empty", "cuda")


def test_gather_refuses_more_channels_than_the_grid_holds():
    """dim > 65535 exceeds gridDim.y: refused with its condition before any launch."""
    with pytest.raises(_lib.OpbError, match="dim <= 65535"):
        features3d.pad_features3d_random(np.ones((65536, 3), np.float32), np.ones((3, 1), np.float32), 4)


# ------------------------------------------------------------------------------------------------ producer-built objects
def sfm_object(seed, M, L, n_target):
    """An object built as inference.py builds it, on the device path: SfM tracks (make_sfm_features, fp64 as the feature files
    hold them, channel-first so the means see F-ordered [sum(len), 256] input), their averages padded to n_target points, and
    L leaves per point picked under np.random.seed(seed), all-ones dustbins for short tracks.
    -> (descriptors3d_db [256, n_target], descriptors2d_db [256, L * n_target]) fp32 numpy, and the dustbin share of the
    real points' leaves."""
    obs, obs_s, idxs, _, _ = synthetic.make_sfm_features(seed, M)
    avg = features3d.mean_descriptors(obs.astype(np.float64).T, idxs)
    avg_s = features3d.mean_scores(obs_s.astype(np.float64), idxs)
    db, _ = features3d.pad_features3d_random(avg.T, avg_s, n_target)
    np.random.seed(seed)
    leaves, _ = features3d.build_features3d_leaves(obs, obs_s, idxs, n_target, L)
    dustbin = float(np.maximum(L - idxs, 0).sum()) / (M * L)
    return db.cpu().numpy(), leaves.cpu().numpy(), dustbin


def _queries(db_real, frame_ids, N):
    """make_frame's queries, planted on the real points' averaged descriptors."""
    return np.ascontiguousarray(np.stack([synthetic.make_frame(f, db_real, N)[0] for f in frame_ids]), np.float32)


def _free():
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _walk(name, seed, M, L, frames, N, hoist, nlen=None):
    _free()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    db, lv, dustbin = sfm_object(seed, M, L, M)
    print(f"\n{name}: {100 * dustbin:.1f} % of the leaves are dustbins, 3D descriptor norms {np.linalg.norm(db, axis=0).min():.3f}-"
          f"{np.linalg.norm(db, axis=0).max():.3f}")
    hp = dict(synthetic.DEFAULT_HPARAMS)
    sd = synthetic.make_state_dict(4)
    queries = _queries(db, frames, N)
    m = _module(sd, hp, hoist)
    st = None
    try:
        m.set_object(torch.from_numpy(db).cuda(), torch.from_numpy(lv).cuda(), reserve=(len(frames), N))
        q = torch.from_numpy(queries).cuda()
        lengths = None if nlen is None else torch.tensor(nlen, dtype=torch.int32).cuda()
        st = Stages(m, lambda: m.match_frames(q, lengths=lengths), oracle.params_from_numpy(sd, torch.float64), hp, queries,
                    [(db, lv)] * len(frames), nlen)
        st.run(hoist)
        torch.cuda.synchronize()
        print(f"{name}: {time.perf_counter() - t0:.1f} s, peak {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB in torch tensors")
        st.report(name)
    finally:
        st = m = q = lengths = None
        _free()


WALKS = {
    # name: (object seed, M, L, frame ids, N, hoist, nlen)
    "ragged": (21, 300, 8, [100, 101, 102, 103], 200, False, [200, 1, 0, 137]),
    "ragged_hoist": (21, 300, 8, [100, 101, 102, 103], 200, True, [200, 0, 1, 137]),
    "ragged_l5": (22, 300, 5, [100, 101, 102, 103], 200, True, [200, 57, 1, 200]),
    "bench": (23, 7000, 8, list(range(100, 132)), 1024, True, None),
}


@pytest.mark.parametrize("name", list(WALKS))
def test_stages_on_producer_built_objects(name):
    seed, M, L, frames, N, hoist, nlen = WALKS[name]
    _walk(name, seed, M, L, frames, N, hoist, nlen)


def test_padded_object_ties_across_column_tiles():
    """6650 real points padded to 7000: the all-ones points fill columns 6650-6999, across three 256-column tiles of the score
    GEMM.  Their conf columns are bit-identical in every frame; a row whose maximum lies among them has its raw arg-max at
    column 6650 (printed: how many rows that is -- the dual softmax splits a row's mass over the 350 ties, so it is rare); two
    frames agree with the fp32 oracle (conf within 1e-4, matches wherever the decision is not a coin flip)."""
    _free()
    M, n_target, B, N = 6650, 7000, 4, 1024
    db, lv, dustbin = sfm_object(24, M, 8, n_target)
    hp = dict(synthetic.DEFAULT_HPARAMS)
    sd = synthetic.make_state_dict(4)
    queries = _queries(db[:, :M], list(range(200, 200 + B)), N)
    m = _module(sd, hp, True)
    try:
        m.set_object(torch.from_numpy(db).cuda(), torch.from_numpy(lv).cuda(), reserve=(B, N))
        q = torch.from_numpy(queries).cuda()
        out = m.match_frames(q)
        m.debug_stop_after(12, 3)
        m.match_frames(q)
        i0, _ = ref.unpack_best(m.debug_read("rowbest"))
        m.debug_stop_after(-1)
        conf = out["conf_matrix"]
        cols = torch.arange(n_target, device=conf.device)
        in_block = 0
        for b in range(B):
            c = conf[b]
            assert torch.equal(c[:, M:], c[:, M:M + 1].expand(-1, n_target - M)), f"frame {b}: padded conf columns differ"
            top = c.max(1, keepdim=True).values
            first = torch.where(c == top, cols, n_target).min(1).values
            rows = first >= M
            in_block += int(rows.sum())
            assert bool((i0[b][rows] == M).all()), f"frame {b}: raw arg-max of a row whose maximum is tied is not column {M}"
        print(f"\npadded object: {100 * dustbin:.1f} % dustbin leaves among the real points, {in_block} of {B * N} rows with their "
              f"maximum in the tied block")
        data = {"descriptors2d_query": queries[:2], "descriptors3d_db": np.repeat(db[None], 2, 0), "descriptors2d_db": np.repeat(lv[None], 2, 0),
                "keypoints2d": np.zeros((2, N, 2), np.float32), "keypoints3d": np.zeros((2, n_target, 3), np.float32)}
        refo = oracle.forward(oracle.params_from_numpy(sd), data, hp)
        err = float((conf[:2].cpu() - refo["conf_matrix"]).abs().max())
        bad, decided, rows = _decided_mismatches({k: out[k][:2] for k in ("matches0", "matches1")}, refo, hp["match_threshold"],
                                                 ref.decided_gap(hp["scale_factor"]))
        print(f"padded object against the oracle: max|dconf| {err:.2e} ({err / 1e-4:.3g} x the bar), {bad} match mismatches among "
              f"{decided} of {rows} decided rows")
        assert err <= 1e-4 and bad == 0
    finally:
        m = q = out = conf = None
        _free()
