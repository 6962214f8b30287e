"""The matcher at the configurations opb_create / set_object accept beyond the released one (scale_factor 0.07, match_threshold
0.2, 8 leaves): scale factors from the smallest accepted value (the fp32 value just above 2 log2(e) / 126, where the tail's
ex2 argument reaches -126 at cos = -1) to 10, thresholds 0, values equal to a produced score, >= 1 and NaN, and 1 to 32 leaves.

  * the stage walk of tests/test_matcher_stages_gpu.py (every step of every layer and of the tail against its fp64 reference)
    at other scales and thresholds, with every bar of that walk; at scale 1 and 10 conf is nearly uniform, so few arg-maxes are
    decided by the fp64 reference and the exact checks (packed arg-max = first maximum of the device's own conf, matches and
    scores = `mutual` of the device's conf bit for bit) are what pins the tail kernels there;
  * end to end against the oracle at the same scales;
  * the two score epilogues driven directly (opb_debug_gemm) on planted extremes: all-antipodal frames (every e at the bottom
    of fp32's normal range at the smallest scale: a cos the score GEMM put below -1 would take ex2's argument below -126 and
    flush e to 0, a NaN conf row; the tensor cores' accumulation toward zero keeps an antipodal cos above -1, and this test
    pins it), exactly aligned and orthogonal rows, duplicate rows and columns across tile edges (equal conf bits, ties won by
    the lowest index on every grid);
  * the threshold's semantics (a strict fp32 comparison) at a produced score and its neighbours, at 0, >= 1 and NaN;
  * the generic GATs aggregation at 2 to 32 leaves, and the refusal of 0 and 33."""
import gc

import numpy as np
import pytest
import torch

from onepose_b200 import _lib, synthetic
from oracle import gats_spg_oracle as oracle
from tests import gemm_core_reference as gr
from tests import matcher_stage_reference as ref
from tests.test_gemm_core_gpu import DEV, GARBAGE, layout_fields, schedules, split
from tests.test_matcher_stages_gpu import CONF_TOL, Stages, _attention_live, _module

pytestmark = pytest.mark.gpu

BOUND = 2.0 * np.log2(np.e) / 126.0                                   # api.cu kMinScaleFactor
SCALE_MIN = float(np.nextafter(np.float32(BOUND), np.float32(1)))     # the smallest scale_factor opb_create accepts


@pytest.fixture(scope="module")
def lib():
    return _lib.load()


def _free():
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _weights(kind, hp=None):
    if kind == "variant":
        return synthetic.make_state_dict(5, hparams=hp)
    sd = synthetic.make_state_dict(4)
    return _attention_live(sd) if kind == "attention_live" else sd


def _walk(name, kind, over, oseed, M, Lf, frames, N, nlen, hoist):
    hp = dict(synthetic.DEFAULT_HPARAMS, **over)
    sd = _weights(kind, hp)
    db, lv = synthetic.make_object(oseed, M, Lf)
    queries = np.stack([synthetic.make_frame(f, db, N)[0] for f in frames])
    if nlen is not None:
        for b, n in enumerate(nlen):
            queries[b, :, n:] = GARBAGE        # the device must ignore everything past each length
    m = _module(sd, hp, hoist)
    try:
        m.set_object(torch.from_numpy(db).cuda(), torch.from_numpy(lv).cuda())
        q = torch.from_numpy(queries).cuda()
        lengths = None if nlen is None else torch.tensor(nlen, dtype=torch.int32).cuda()
        st = Stages(m, lambda: m.match_frames(q, lengths=lengths), oracle.params_from_numpy(sd, torch.float64), hp, queries,
                    [(db, lv)] * len(frames), nlen)
        st.run(hoist)
        st.report(name)
    finally:
        st = m = q = None
        _free()


# ------------------------------------------------------------------------------------------------ a. scales and thresholds
SCALE_CASES = {
    # name: (weights, scale, threshold, frames, N, M, nlen, hoist)
    "bound_ragged": ("fixture", SCALE_MIN, 0.2, [100, 101, 102, 103], 300, 700, [300, 1, 0, 137], False),
    "bound_live_hoist_thr0": ("attention_live", SCALE_MIN, 0.0, [100, 101, 102], 300, 700, [0, 300, 1], True),
    "s0.03_thr0_hoist": ("fixture", 0.03, 0.0, [100, 101], 300, 700, [300, 1], True),
    "s0.05_thr0.9_live": ("attention_live", 0.05, 0.9, [100, 101, 102, 103], 300, 700, [1, 300, 0, 211], False),
    "s0.2_hoist": ("fixture", 0.2, 0.2, [100, 101], 300, 700, None, True),
    "s1_thr0_live": ("attention_live", 1.0, 0.0, [100, 101, 102], 300, 700, [300, 0, 1], False),
    "s10_thr0_hoist": ("fixture", 10.0, 0.0, [100, 101], 300, 700, [1, 300], True),
    "s10_thr0.9_live": ("attention_live", 10.0, 0.9, [100, 101, 102], 300, 700, [257, 1, 300], False),
}


@pytest.mark.parametrize("name", list(SCALE_CASES))
def test_stages_across_scales_and_thresholds(name):
    """The whole stage walk at another scale_factor / match_threshold: every bar of the walk (the tail's scale with 1 / scale),
    arg-max = first maximum of the device's conf, matches = `mutual` of the device's conf at the handle's threshold, zeros past
    N_b / M_b, every conf entry finite.  At scale 1 and 10 the fp64 arg-max check decides few rows: the exact checks carry it."""
    kind, scale, thr, frames, N, M, nlen, hoist = SCALE_CASES[name]
    _walk(name, kind, dict(scale_factor=scale, match_threshold=thr), 9, M, 8, frames, N, nlen, hoist)


def test_stages_at_the_benchmarked_frame_at_the_smallest_scale():
    """One frame of 1024 queries against 7000 points (the benchmarked frame) at the smallest accepted scale."""
    _walk("bench frame at the bound", "fixture", dict(scale_factor=SCALE_MIN), 0, 7000, 8, [100], 1024, None, True)


# ------------------------------------------------------------------------------------------------ b. end to end
E2E_SCALES = [SCALE_MIN, 0.03, 0.05, 0.07, 0.2, 1.0, 10.0]


def _decided_mismatches(out, refo, thr, gap):
    """matches0 / matches1 that differ from the oracle's where its decision is not a floating-point coin flip: the row's and
    its arg-max column's top-1 / top-2 gaps exceed `gap` relative and a mutual score is more than `gap` relative from the
    threshold.  Returns (mismatches, decided rows, valid rows)."""
    rc = refo["conf_matrix"]
    t = rc.topk(2, dim=2).values
    dr = (t[..., 0] - t[..., 1]) > gap * t[..., 0]
    t = rc.topk(2, dim=1).values
    dc = (t[:, 0] - t[:, 1]) > gap * t[:, 0]
    i0, i1 = refo["raw_indices0"], refo["raw_indices1"]
    ms0 = refo["matching_scores0"]
    near = (ms0 > 0) & ((ms0 - thr).abs() <= gap * ms0)        # a mutual score at the threshold (0 is not mutual: no match)
    d0 = dr & dc.gather(1, i0) & ~near
    d1 = dc & d0.gather(1, i1)
    m0, m1 = out["matches0"].cpu(), out["matches1"].cpu()
    bad = int(((m0 != refo["matches0"]) & d0).sum() + ((m1 != refo["matches1"]) & d1).sum())
    return bad, int(d0.sum()), d0.numel()


@pytest.mark.parametrize("scale", E2E_SCALES)
def test_end_to_end_against_oracle_across_scales(scale):
    """The module against the fp32 oracle at the same hparams: max|dconf| within 1e-4 at every scale (measured on an H100:
    4.0e-6 at the smallest scale, 4.7e-6 at 0.07, below 1e-7 from 0.2 up; DESIGN section 2), matches equal wherever decided
    (every row but a handful), scores within 1e-4.  Threshold 0.2 up to scale 0.07, 0 above it (no conf entry reaches 0.2)."""
    thr = 0.2 if scale <= 0.07 else 0.0
    hp = dict(synthetic.DEFAULT_HPARAMS, scale_factor=scale, match_threshold=thr)
    sd = synthetic.make_state_dict(4)
    data = synthetic.make_batch(9, [100, 101], 300, 700, 8)
    refo = oracle.forward(oracle.params_from_numpy(sd), data, hp)
    m = _module(sd, hp, True)
    m({k: torch.from_numpy(v).cuda() for k, v in data.items()})
    m.check_range()
    out = m.last_batched
    conf = out["conf_matrix"].cpu()
    assert bool(torch.isfinite(conf).all())
    err = float((conf - refo["conf_matrix"]).abs().max())
    bad, decided, rows = _decided_mismatches(out, refo, thr, ref.decided_gap(scale))
    n_match = int((out["matches0"] > -1).sum())
    print(f"\nscale {scale:.9g}: max|dconf| = {err:.3e} (bar {CONF_TOL:.0e}), {n_match} matches, {decided}/{rows} rows decided, "
          f"{bad} decided matches differ")
    assert err <= CONF_TOL, f"scale {scale}: max|dconf| = {err:.3e}"
    assert bad == 0
    assert decided >= 0.9 * rows and n_match > 0
    np.testing.assert_allclose(out["matching_scores0"].cpu().numpy(), refo["matching_scores0"].numpy(), atol=CONF_TOL)
    np.testing.assert_allclose(out["matching_scores1"].cpu().numpy(), refo["matching_scores1"].numpy(), atol=CONF_TOL)


# ------------------------------------------------------------------------------------------------ c. planted extremes
PL = ref.Layout(3, 300, 700, 512, 768, nlen=[300, 40, 1], mlen=[700, 600, 1])
DUP_COLS = [0, 255, 256, 511, 699]          # frame 0: one vector in these columns (3D-point tiles of 256)
DUP_ROWS = [0, 127, 128, 299]               # frame 0: one vector in these query rows (row tiles of 128)


def _planted_rows(seed):
    """Unit rows in the score layout: frame 0 random with duplicate rows / columns, aligned (cos = +1) and orthogonal pairs;
    frame 1 every query q and every 3D point -q (all-antipodal: e at its minimum in every entry); frame 2 one query q against
    one point -q.  Pad rows hold GARBAGE."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    L = PL
    pn = torch.nn.functional.normalize(torch.randn(L.rows, 256, device=DEV, generator=g), dim=1)
    basis = torch.linalg.qr(torch.randn(256, 8, device=DEV, dtype=torch.float64, generator=g))[0].T.float()   # orthonormal
    q0, d0 = L.seg_start(0), L.seg_start(1)
    pn[[q0 + r for r in DUP_ROWS]] = basis[0]
    pn[d0 + 3] = basis[0]                   # the duplicate rows are the maxima of column 3: a tie of four rows across row tiles
    pn[[d0 + c for c in DUP_COLS]] = basis[1]
    pn[q0 + 5] = basis[1]                   # row 5's maximum is the tie of the five duplicate columns across column tiles
    pn[q0 + 10], pn[d0 + 20] = basis[2], basis[2]       # aligned: cos = +1
    pn[q0 + 11], pn[d0 + 21] = basis[3], basis[3]       # orthogonal to the pair above
    pn[q0 + 12] = basis[4]                               # orthogonal to both aligned columns
    for b in (1, 2):
        q = basis[4 + b]
        pn[L.seg_rows(2 * b)] = q
        pn[L.seg_rows(2 * b + 1)] = -q
    pn[~L.valid_mask(DEV)] = GARBAGE
    return pn


@pytest.mark.parametrize("scale", [SCALE_MIN, 0.07, 10.0])
def test_score_epilogues_on_planted_extremes(lib, scale):
    """Pass 1: partial sums within 1e-5 + COS_ERR / scale of fp64, and every valid row's and column's partial sum > 0 (no e flushed
    to zero, even where every entry of a frame is antipodal at the smallest scale).  Pass 2 with the fp64 inverse sums: every conf
    entry finite and within its bar, duplicate rows' and columns' conf bit-equal, the packed arg-maxes the first maxima (lowest
    index on the planted ties).  Every output bit-identical on 1, 2, 3, 7, 131, 132 CTAs and the default grid."""
    L = PL
    lf, keep = layout_fields(L)
    p = split(lib, _planted_rows(11))
    base = dict(rows=L.n_pad, n_out=L.m_pad, K1=256, batch=L.B, a_batch_rows=L.R, b_batch_rows=L.R, a1_hi=p[0], a1_lo=p[1],
                a1_ld=256, b1_hi=p[0][L.n_pad:], b1_lo=p[1][L.n_pad:], b1_ld=256, inv_scale=1.0 / scale, **lf)
    n_tiles, m_tiles = L.m_pad // 256, L.n_pad // 128
    sums = schedules(lib, "planted sums", {**base, "epi": _lib.EPI_SCORE_SUMS},
                     {"rowsum_part": torch.empty(L.B, 2 * n_tiles, L.n_pad, device=DEV),
                      "colsum_part": torch.empty(L.B, m_tiles * 4, L.m_pad, device=DEV)})
    rs_ref, cs_ref, cos = gr.score_partials(p[2], L, scale)
    rel = 1e-5 + ref.COS_ERR / scale
    ratios, empty = {}, 0
    for k, r in (("rowsum_part", rs_ref), ("colsum_part", cs_ref)):
        d = sums[k].double()
        z = r == 0
        ratios[k] = max(ref._ratio((d - r).abs()[~z], rel * r[~z]), 0.0 if bool((d[z] == 0).all()) else float("inf"))
        empty += int((d[~z] <= 0).sum())
    assert empty == 0, f"{empty} partial sums with valid entries are not positive: e flushed to zero"
    irs = torch.zeros(L.B, L.n_pad, device=DEV)
    ics = torch.zeros(L.B, L.m_pad, device=DEV)
    for b in range(L.B):
        n, m = L.n_of(b), L.m_of(b)
        e = torch.exp((cos[b][:n, :m] - 1.0) / scale)
        irs[b, :n] = (1.0 / e.sum(1)).float()
        ics[b, :m] = (1.0 / e.sum(0)).float()
    outs = schedules(lib, "planted conf", {**base, "epi": _lib.EPI_SCORE_CONF, "inv_rowsum": irs, "inv_colsum": ics, "conf_ld": 0},
                     {"conf": torch.empty(L.B, L.N, L.M, device=DEV), "rowbest": torch.empty(L.B, L.N, dtype=torch.int64, device=DEV),
                      "colbest": torch.empty(L.B, L.M, dtype=torch.int64, device=DEV)}, zero=("rowbest", "colbest"))
    ratios["conf"], bad_first, bad_zero = 0.0, 0, 0
    for b in range(L.B):
        n, m = L.n_of(b), L.m_of(b)
        conf = outs["conf"][b]
        bad_zero += int((conf[n:] != 0).sum() + (conf[:, m:] != 0).sum())
        c = conf[:n, :m]
        ratios["conf"] = max(ratios["conf"], ref.bar_conf(c, cos[b][:n, :m], irs[b, :n].double(), ics[b, :m].double(), scale))
        i0, v0 = ref.unpack_best(outs["rowbest"][b, :n])
        i1, v1 = ref.unpack_best(outs["colbest"][b, :m])
        bad_first += ref.first_max_mismatches(i0, v0, c, 1) + ref.first_max_mismatches(i1, v1, c, 0)
        if b == 0:
            i0_0, i1_0, c0 = i0, i1, c
        elif b == 1:            # all-antipodal: every entry equal, so every arg-max is index 0
            assert bool((c == c[0, 0]).all()), "all-antipodal frame: conf entries differ"
            assert bool((i0 == 0).all()) and bool((i1 == 0).all())
    report = {k: f"{v:.3f}" for k, v in ratios.items()}
    print(f"\nplanted extremes at scale {scale:.9g}: {report}, all-antipodal conf {float(outs['conf'][1, 0, 0]):.6e} "
          f"(1 / (N M) = {1.0 / (40 * 600):.6e}), single entry {float(outs['conf'][2, 0, 0]):.6e}")
    for k, v in ratios.items():
        assert v <= 1.0, f"{k} at {v:.3g} x its bar"
    assert bad_zero == 0, "conf entries past N_b / M_b are not 0"
    assert bad_first == 0, "packed arg-maxes that are not the first maximum of the device's conf"
    for r in DUP_ROWS[1:]:
        assert torch.equal(c0[r].view(torch.int32), c0[DUP_ROWS[0]].view(torch.int32)), f"duplicate row {r}"
    for col in DUP_COLS[1:]:
        assert torch.equal(c0[:, col].view(torch.int32), c0[:, DUP_COLS[0]].view(torch.int32)), f"duplicate column {col}"
    assert int(i1_0[3]) == DUP_ROWS[0], "the tie of duplicate rows in column 3 is not won by the lowest row"
    assert int(i0_0[5]) == DUP_COLS[0], "the tie of duplicate columns in row 5 is not won by the lowest column"
    assert int(i0_0[10]) == 20 and int(i1_0[20]) == 10, "the aligned pair is not each other's maximum"


# ------------------------------------------------------------------------------------------------ d. threshold semantics
def _run(sd, hp, data):
    m = _module(sd, hp, True)
    m({k: torch.from_numpy(v).cuda() for k, v in data.items()})
    m.check_range()
    return {k: v.clone() for k, v in m.last_batched.items()}


def test_threshold_is_a_strict_fp32_comparison():
    """A score c the matcher produced, used as the threshold (as an fp32 value, as a double that rounds to it, and the fp32 value
    just below it): exactly the first call's matches whose score is > fp32(threshold) survive, conf and scores keep their bits.
    Threshold 0 matches every mutual pair; 1, 1.5 and NaN match nothing.  Each against the oracle at the same hparams."""
    sd = synthetic.make_state_dict(4)
    data = synthetic.make_batch(9, [100, 101], 300, 700, 8)
    hp0 = dict(synthetic.DEFAULT_HPARAMS)
    first = _run(sd, hp0, data)
    s0, m0, s1, m1 = (first[k] for k in ("matching_scores0", "matches0", "matching_scores1", "matches1"))
    vals = torch.sort(s0[m0 > -1]).values
    assert vals.numel() > 20
    c = np.float32(vals[vals.numel() // 2].item())
    assert int((s0 == float(c)).sum()) >= 1
    below = np.nextafter(c, np.float32(0))
    rounds_to_c = float(c) - float(np.spacing(c)) / 4          # a double below c that rounds to c in fp32
    assert np.float32(rounds_to_c) == c and rounds_to_c < float(c)
    for thr, t32 in ((float(c), c), (rounds_to_c, c), (float(below), below)):
        out = _run(sd, dict(hp0, match_threshold=thr), data)
        for k in ("conf_matrix", "matching_scores0", "matching_scores1"):
            assert torch.equal(out[k].view(torch.int32), first[k].view(torch.int32)), (thr, k)
        keep0 = s0 > float(t32)
        keep1 = s1 > float(t32)
        assert torch.equal(out["matches0"], torch.where(keep0, m0, -1)), thr
        assert torch.equal(out["matches1"], torch.where(keep1, m1, -1)), thr
        n_at_c = int(((m0 > -1) & (s0 == float(c))).sum())
        print(f"threshold {thr!r}: {int((out['matches0'] > -1).sum())} matches ({n_at_c} scored exactly fp32(c))")
        assert int((out["matches0"] == -1).sum() - (m0 == -1).sum()) == int(((m0 > -1) & ~keep0).sum())
    for thr in (0.0, 1.0, 1.5, float("nan")):
        hp = dict(hp0, match_threshold=thr)
        out = _run(sd, hp, data)
        refo = oracle.forward(oracle.params_from_numpy(sd), data, hp)
        assert torch.equal(out["conf_matrix"].view(torch.int32), first["conf_matrix"].view(torch.int32)), thr
        for b in range(2):
            r0, r1, rs0, rs1 = ref.mutual(out["conf_matrix"][b], thr)
            assert torch.equal(out["matches0"][b], r0) and torch.equal(out["matches1"][b], r1), thr
            assert torch.equal(out["matching_scores0"][b], rs0) and torch.equal(out["matching_scores1"][b], rs1), thr
        np.testing.assert_array_equal(out["matches0"].cpu().numpy(), refo["matches0"].numpy())
        np.testing.assert_array_equal(out["matches1"].cpu().numpy(), refo["matches1"].numpy())
        n = int((out["matches0"] > -1).sum())
        if thr == 0.0:
            assert torch.equal(out["matches0"] > -1, s0 > 0) and n > int((m0 > -1).sum())
        else:
            assert n == 0 and int((out["matches1"] > -1).sum()) == 0, thr


# ------------------------------------------------------------------------------------------------ e. leaf counts
LEAF_CASES = {
    # name: (weights, hparams overrides, L, frames, N, M, nlen, hoist)
    "l2_ragged": ("fixture", {}, 2, [7, 8, 9], 100, 257, [100, 0, 1], False),
    "l7_hoist": ("fixture", {}, 7, [7, 8], 100, 257, None, True),
    "l9_lintrans": ("variant", dict(with_linear_transform=True), 9, [7, 8], 100, 257, [100, 33], False),
    "l16": ("fixture", {}, 16, [7, 8], 100, 300, None, False),
    "l31_ragged_live": ("attention_live", {}, 31, [7, 8, 9], 100, 257, [1, 100, 64], False),
    "l32_hoist": ("fixture", {}, 32, [7, 8], 100, 513, [100, 99], True),
}


@pytest.mark.parametrize("name", list(LEAF_CASES))
def test_stages_across_leaf_counts(name):
    """The generic GATs aggregation (every leaf count but 8): the stage walk at 2, 7, 9, 16, 31 and 32 leaves (a full warp of leaf
    logits; 2, 7, 9, 31 leave a partial 4-row batch)."""
    kind, over, Lf, frames, N, M, nlen, hoist = LEAF_CASES[name]
    _walk(name, kind, over, 4, M, Lf, frames, N, nlen, hoist)


def test_leaf_counts_outside_1_to_32_are_refused():
    """set_object / add_object refuse 0 and 33 leaves and keep the handle usable."""
    hp = dict(synthetic.DEFAULT_HPARAMS)
    sd = synthetic.make_state_dict(4)
    m = _module(sd, hp, True)
    db, lv = synthetic.make_object(3, 64, 33)
    d3, d2 = torch.from_numpy(db).cuda(), torch.from_numpy(lv).cuda()
    for leaves in (d2[:, :0], d2):
        with pytest.raises(_lib.OpbError, match="num_leaf"):
            m.set_object(d3, leaves)
        with pytest.raises(_lib.OpbError, match="num_leaf"):
            m.add_object(d3, leaves)
    m.set_object(d3, d2[:, :64 * 32])
    q = torch.from_numpy(synthetic.make_frame(1, db, 50)[0][None]).cuda()
    out = m.match_frames(q)
    m.check_range()
    assert int((out["matches0"] > -1).sum()) > 0
