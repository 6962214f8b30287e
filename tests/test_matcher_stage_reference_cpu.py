"""The fp64 stage references of tests/matcher_stage_reference.py, without a GPU.

* Composition: chained over the 12 GNN layers and the tail they equal the oracle's fp64 forward, for ragged query counts,
  frames of objects of different sizes and every GraphAttentionLayer branch -- so a wrong reference cannot hide a wrong kernel.
* Teeth: each planted defect moves its own stage by at least 10x that stage's bar, while the end-to-end conf moves by less
  than the 1e-4 bar of the parity tests (all but InstanceNorm statistics over the pad rows, which the end-to-end bar sees).
  This is why the matcher's attention path is tested stage by stage.
* Tail teeth: conf entries below 1e-4 written as 0, a column using its neighbour's inverse sum, and matching_scores1 taken from
  the wrong row each move the entry-by-entry conf check or the exact mutual check by at least 10x.  Only the last one passes the
  end-to-end bars (conf within 1e-4, decided arg-max); the test asserts each outcome."""
import numpy as np
import pytest
import torch

from onepose_b200 import synthetic
from oracle import gats_spg_oracle as oracle
from tests import matcher_stage_reference as ref

HP = dict(synthetic.DEFAULT_HPARAMS)


def _oracle_frame(P, hp, q, db, leaves):
    data = {"keypoints2d": np.zeros((1, q.shape[1], 2), np.float32), "keypoints3d": np.zeros((1, db.shape[1], 3), np.float32),
            "descriptors2d_query": q[None], "descriptors3d_db": db[None], "descriptors2d_db": leaves[None]}
    return oracle.forward(P, data, hp, torch.float64)


def _compose_vs_oracle(sd, hp, queries, objects, nlen):
    P = oracle.params_from_numpy(sd, torch.float64)
    confs, matches = ref.chain_forward(P, hp, queries, objects, nlen)
    worst = 0.0
    for b in range(len(objects)):
        n = queries.shape[2] if nlen is None else nlen[b]
        o = _oracle_frame(P, hp, queries[b][:, :n], *objects[b])
        worst = max(worst, float((confs[b] - o["conf_matrix"][0]).abs().max()))
        m0, m1, s0, s1 = matches[b]
        assert torch.equal(m0, o["matches0"][0]) and torch.equal(m1, o["matches1"][0]), f"frame {b}"
        assert float((s0 - o["matching_scores0"][0]).abs().max()) <= 1e-10
        assert float((s1 - o["matching_scores1"][0]).abs().max()) <= 1e-10
    assert worst <= 1e-10, worst
    return worst


def test_composition_ragged_queries():
    sd = synthetic.make_state_dict(4)
    data = synthetic.make_batch(9, [100, 101, 102], 200, 300, 8)
    objects = [(data["descriptors3d_db"][b], data["descriptors2d_db"][b]) for b in range(3)]
    _compose_vs_oracle(sd, HP, data["descriptors2d_query"], objects, [200, 1, 137])


def test_composition_objects_of_different_sizes():
    sd = synthetic.make_state_dict(4, damped=False)
    objs = [synthetic.make_object(300 + k, M, 5) for k, M in enumerate([255, 257, 40])]
    order = [0, 2, 1, 0]
    q = np.stack([synthetic.make_frame(50 + b, objs[k][0], 90)[0] for b, k in enumerate(order)])
    _compose_vs_oracle(sd, HP, q, [objs[k] for k in order], [90, 33, 90, 7])


@pytest.mark.parametrize("variant", [dict(include_self=False), dict(additional=True), dict(with_linear_transform=True),
                                     dict(include_self=False, with_linear_transform=True),
                                     dict(with_linear_transform=True, additional=True)])
def test_composition_gats_variants(variant):
    hp = dict(HP, **variant)
    sd = synthetic.make_state_dict(5, hparams=hp)
    data = synthetic.make_batch(3, [1, 2], 64, 96, 6)
    objects = [(data["descriptors3d_db"][b], data["descriptors2d_db"][b]) for b in range(2)]
    _compose_vs_oracle(sd, hp, data["descriptors2d_query"], objects, None)


# ----------------------------------------------------------------------------------------------------------------- teeth
@pytest.fixture(scope="module")
def teeth_setup():
    """The fixture weights (damped, as most parity tests use) on two frames of one object; X entering layers 1 (self) and 2
    (cross) of the clean fp64 chain."""
    sd = synthetic.make_state_dict(4)
    P = oracle.params_from_numpy(sd, torch.float64)
    data = synthetic.make_batch(9, [100, 101], 300, 700, 8)
    objects = [(data["descriptors3d_db"][b], data["descriptors2d_db"][b]) for b in range(2)]
    x, leaves_of, L = ref.assemble(data["descriptors2d_query"], objects)
    x1 = ref.gats_layer(x, leaves_of, P, 0, HP, L)[0]
    x2 = ref.attn_layer(x1, ref.attn_weights(P, 1), L, False)
    clean = ref.chain_forward(P, HP, data["descriptors2d_query"], objects)[0]
    return P, data, objects, L, {1: x1, 2: x2}, clean


DEFECTS = {"msg_scale": ref.Defect(msg_scale=1.01), "rotate_heads": ref.Defect(rotate_heads=True), "own_side": ref.Defect(own_side=True),
           "mean_over_pad": ref.Defect(mean_over_pad=True), "kvt_pad_rows": ref.Defect(kvt_pad_rows=True),
           "in_stats_pad": ref.Defect(in_stats_pad=True)}


def _stage_ratio(name, P, L, xs):
    """Error of the defective stage against the clean one, in multiples of the stage's bar."""
    d = DEFECTS[name]
    layer = 2 if name == "own_side" else 1
    cross = layer == 2
    x, A = xs[layer], ref.attn_weights(P, layer)
    kvt, absprod = ref.kv_proj(x, A, L)
    kmean, bd = ref.kv_state(kvt, L, cross)
    qp = ref.q_proj(x, kmean, A, L, cross)
    G = ref.g_fold(bd, A)
    hid = ref.mlp0(x, qp, G, A, L)
    mu, rstd = ref.in_stats(hid, L)
    if name == "msg_scale":
        return ref.bar_per_segment(ref.g_fold(bd, A, d), G)
    if name == "rotate_heads":
        return ref.bar_rows(ref.q_proj(x, kmean, A, L, cross, d), qp, L.valid_mask())
    if name == "own_side":
        return ref.bar_bd(ref.kv_state(kvt, L, cross, d)[1], bd)
    if name == "mean_over_pad":
        return ref.bar_per_segment(ref.kv_state(kvt, L, cross, d)[0], kmean)
    if name == "kvt_pad_rows":
        return ref.bar_kvt(ref.kv_proj(x, A, L, d)[0], kvt, absprod, L)
    mu_d, rstd_d = ref.in_stats(hid, L, d)
    return max(ref.bar_mu(mu_d, mu, rstd, L), ref.bar_rstd(rstd_d, rstd, L))


@pytest.mark.parametrize("name", list(DEFECTS))
def test_planted_defect_clears_its_stage_bar_but_not_the_end_to_end_bar(teeth_setup, name):
    P, data, objects, L, xs, clean = teeth_setup
    ratio = _stage_ratio(name, P, L, xs)
    confs = ref.chain_forward(P, HP, data["descriptors2d_query"], objects, defect=DEFECTS[name])[0]
    dconf = max(float((c - c0).abs().max()) for c, c0 in zip(confs, clean))
    print(f"{name}: stage error = {ratio:.3g} x its bar, end-to-end max|dconf| = {dconf:.2e}")
    assert ratio >= 10.0, f"{name}: the stage bar would not catch it ({ratio:.3g} x)"
    if name == "in_stats_pad":      # the one defect of the list the end-to-end bar does see (5.6e-2 here)
        assert dconf > 1e-4, f"{name}: no longer visible end to end ({dconf:.2e})"
    else:
        assert dconf < 1e-4, f"{name}: visible end to end ({dconf:.2e})"


# ------------------------------------------------------------------------------------------------------------ tail teeth
TAIL_DEFECTS = {"conf_zero_below_1e-4": ref.Defect(conf_zero_below=1e-4), "conf_neighbour_ics": ref.Defect(conf_neighbour_ics=True),
                "ms1_wrong_row": ref.Defect(ms1_wrong_row=True)}
# whether each defect passes the end-to-end bars: zeroing below 1e-4 keeps max|dconf| under the bar but moves the arg-max of
# columns whose entries all lie below it; the wrong scores row touches neither conf nor the arg-maxes
TAIL_DEFECT_PASSES_END_TO_END = {"conf_zero_below_1e-4": False, "conf_neighbour_ics": False, "ms1_wrong_row": True}


@pytest.fixture(scope="module")
def tail_setup():
    """pn of the clean fp64 chain on two frames of one object (the fixture weights); its inverse sums and conf."""
    sd = synthetic.make_state_dict(4)
    P = oracle.params_from_numpy(sd, torch.float64)
    data = synthetic.make_batch(9, [100, 101], 300, 700, 8)
    objects = [(data["descriptors3d_db"][b], data["descriptors2d_db"][b]) for b in range(2)]
    x, leaves_of, L = ref.assemble(data["descriptors2d_query"], objects)
    pn = ref.final_proj(ref.gnn(x, leaves_of, P, HP, L), P)
    return pn, L


@pytest.mark.parametrize("name", list(TAIL_DEFECTS))
def test_tail_defect_clears_the_conf_or_mutual_bar(tail_setup, name):
    """Each tail defect moves the entry-by-entry conf check or the exact mutual check by at least 10x its bar; the end-to-end
    bars (conf within 1e-4, arg-max where the fp64 decision is clear) are reported alongside."""
    pn, L = tail_setup
    d = TAIL_DEFECTS[name]
    scale, thr = HP["scale_factor"], HP["match_threshold"]
    ratio, dconf, argmax_bad = 0.0, 0.0, 0
    for b in range(L.B):
        cos = pn[L.seg_rows(2 * b)] @ pn[L.seg_rows(2 * b + 1)].T
        e = torch.exp((cos - 1.0) / scale)
        irs, ics = 1.0 / e.sum(1), 1.0 / e.sum(0)
        clean = ref.conf_entries(e, irs, ics)
        bad = ref.conf_entries(e, irs, ics, d).float()       # the device's conf is fp32
        ratio = max(ratio, ref.bar_conf(bad, cos, irs, ics, scale))
        m0, m1, s0, s1 = ref.mutual(bad, thr, d)
        if ref.mutual_mismatches(m0, m1, s0, s1, bad, thr):
            ratio = float("inf")
        dconf = max(dconf, float((bad.double() - clean).abs().max()))
        argmax_bad += ref.argmax_mismatches(bad.argmax(1), clean, 1) + ref.argmax_mismatches(bad.argmax(0), clean, 0)
    e2e = dconf <= 1e-4 and argmax_bad == 0
    print(f"{name}: conf / mutual check = {ratio:.3g} x its bar; end to end max|dconf| = {dconf:.2e}, decided arg-max "
          f"mismatches = {argmax_bad} -> end-to-end bars {'pass' if e2e else 'fail'}")
    assert ratio >= 10.0, f"{name}: the tail checks would not catch it ({ratio:.3g} x)"
    assert e2e == TAIL_DEFECT_PASSES_END_TO_END[name], f"{name}: end-to-end bars {'pass' if e2e else 'fail'}"


def test_clean_tail_meets_the_conf_bar_in_fp32(tail_setup):
    """The clean conf rounded to fp32 (what the epilogue's last product does) stays far inside the per-entry bar, so the bar is
    not met by accident of a loose reference."""
    pn, L = tail_setup
    scale = HP["scale_factor"]
    for b in range(L.B):
        cos = pn[L.seg_rows(2 * b)] @ pn[L.seg_rows(2 * b + 1)].T
        e = torch.exp((cos - 1.0) / scale)
        irs, ics = 1.0 / e.sum(1), 1.0 / e.sum(0)
        assert ref.bar_conf(ref.conf_entries(e, irs, ics).float(), cos, irs, ics, scale) < 0.01


def test_fp16_ulp_equals_numpy_spacing():
    rs = np.random.RandomState(3)
    v = np.concatenate([rs.randn(4000) * 10.0 ** rs.uniform(-9, 4, 4000), [0.0, 2.0 ** -14, 2.0 ** -15, 1.0, 2047.9, 65000.0]])
    want = np.spacing(np.abs(v).astype(np.float16)).astype(np.float64)
    assert np.array_equal(ref.fp16_ulp(torch.from_numpy(v)).numpy(), want)
