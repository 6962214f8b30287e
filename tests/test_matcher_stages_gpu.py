"""Every step of every GNN layer and of the tail against its fp64 stage reference (tests/matcher_stage_reference.py), on the
device's own input to that step: the call is stopped after the step (opb_debug_set_stop) and the buffers are read back
(opb_debug_read).  The end-to-end parity tests cannot see the attention path -- with these weights its message is almost
constant per segment and InstanceNorm removes it (tests/test_matcher_stage_reference_cpu.py measures how blind they are).

Bars, set from the operand formats (fp16-split operands carry ~2^-22 relative down to an absolute 2^-30; 3-pass GEMMs keep
fp32 semantics):
  kvt           one fp16 ulp of fp16(64 ref) / 64 + 2^-11 sum|x||w| (the two-pass projection); pad rows exactly 0
  Kmean, bd     1e-5 of the segment's max; bd's off-diagonal blocks exactly 0
  Q', G, hid    1e-5 of the row's (G: the segment's) max
  mu            1e-6 (|mu| + sigma);   rstd   1e-5 relative
  X after mlp.3 1e-5 max|layer delta| of the segment + 2^-18 |x| + 16 x 2^-30 (the residual through the fp32 accumulator
                and the split); pad rows exactly 0
  X after GATs  1e-5 of the row's max (the rows before W with with_linear_transform likewise); pad rows exactly 0
  pn            unit rows to 1e-6, elements within 1e-5
  inverse sums  1e-5 + 48 x 2^-23 / scale relative (the score GEMM's fp32 accumulation, amplified by 1 / scale)
  arg-max       equal wherever the fp64 top-1 / top-2 gap exceeds 1e-5 relative
Each measured error is printed as a multiple of its bar."""
import numpy as np
import pytest
import torch

from onepose_b200 import GATsSuperGlue, synthetic
from oracle import gats_spg_oracle as oracle
from tests import matcher_stage_reference as ref

pytestmark = pytest.mark.gpu

CONF_TOL = 1e-4


def _module(sd, hp, hoist):
    m = GATsSuperGlue(dict(hp)).eval()
    m.load_state_dict({k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in sd.items()}, strict=True)
    m = m.cuda()
    m.set_hoist(hoist)
    return m


def split_roundtrip(a):
    """fp32 -> the value of its fp16-split planes, (hi + lo) / 64 (common.cuh split_f32)."""
    s = np.asarray(a, np.float32) * np.float32(64)
    hi = s.astype(np.float16)
    lo = (s - hi.astype(np.float32)).astype(np.float16)
    return (hi.astype(np.float32) + lo.astype(np.float32)) / np.float32(64)


def _attention_live(sd):
    """q, k projections x 16: Q' and KVmean far from uniform."""
    sd = dict(sd)
    for i in range(12):
        if i % 3:
            for j in (0, 1):
                sd[f"gnn.layers.{i}.attn.proj.{j}.weight"] = sd[f"gnn.layers.{i}.attn.proj.{j}.weight"] * np.float32(16)
    return sd


def _in_offset(sd):
    """mlp.0 bias + 3: hidden channels with mean / std ~ 100 (the InstanceNorm statistics' hard case)."""
    sd = dict(sd)
    for i in range(12):
        if i % 3:
            sd[f"gnn.layers.{i}.mlp.0.bias"] = sd[f"gnn.layers.{i}.mlp.0.bias"] + np.float32(3)
    return sd


class Stages:
    """Runs a call again and again, stopped after one step each time, and checks that step against its reference."""

    def __init__(self, m, call, P, hp, queries, objects, nlen):
        self.m, self.call, self.P, self.hp = m, call, P, hp
        self.queries, self.objects, self.nlen = queries, objects, nlen
        self.ratios = {}
        # the chunk's inputs as the device holds them (fp16-split planes); leaves stay fp32
        x, self.leaves_of, self.L = ref.assemble(split_roundtrip(queries), [(split_roundtrip(db), lv) for db, lv in objects], nlen)
        self.x0 = x

    def stop(self, layer, step, nlen=None, mlen=None):
        self.m.debug_stop_after(layer, step)
        self.call()
        L = ref.Layout.of(self.m.debug_layout(), nlen, mlen)
        return L, (lambda name: self.m.debug_read(name).cpu().double())

    def record(self, key, ratio):
        self.ratios[key] = ratio

    # ---------------------------------------------------------------- layers
    def gats(self, tag, layer, layer_id, x_in, Lx, leaves_of, nlen, mlen):
        last = 1 if self.hp["with_linear_transform"] else 0
        L, rd = self.stop(layer_id, last, nlen, mlen)
        assert (L.B, L.N, L.M, L.n_pad, L.m_pad) == (Lx.B, Lx.N, Lx.M, Lx.n_pad, Lx.m_pad)
        out, pre = ref.gats_layer(x_in, leaves_of, self.P, layer, self.hp, L)
        x = rd("x")
        self.record((tag, layer, "gats"), ref.bar_gats(x, out, L))
        if last:
            rows = torch.zeros(L.B * L.m_pad, dtype=torch.bool)
            for b in range(L.B):
                rows[b * L.m_pad:b * L.m_pad + L.m_of(b)] = True
            self.record((tag, layer, "gats pre-W"), ref.bar_rows(rd("gats_pre"), pre, rows))
        return x

    def attn(self, tag, layer, layer_id, cross, nlen, mlen, x_prev=None):
        A = ref.attn_weights(self.P, layer)
        L, rd = self.stop(layer_id, 6, nlen, mlen)
        x = rd("x")
        if x_prev is not None:
            assert torch.equal(x, x_prev), f"{tag} layer {layer}: X entering the layer differs between two identical calls"
        kvt, kmean, bd, qp, g, hid, mu, rstd = (rd(n) for n in ("kvt", "kmean", "bd", "qp", "g", "hid", "mu", "rstd"))
        v = L.valid_mask()
        kvt_ref, absprod = ref.kv_proj(x, A, L)
        self.record((tag, layer, "kvt"), ref.bar_kvt(kvt, kvt_ref, absprod, L))
        kmean_ref, bd_ref = ref.kv_state(kvt, L, cross)
        self.record((tag, layer, "kmean"), ref.bar_per_segment(kmean, kmean_ref))
        self.record((tag, layer, "bd"), ref.bar_bd(bd, bd_ref))
        self.record((tag, layer, "Q'"), ref.bar_rows(qp, ref.q_proj(x, kmean, A, L, cross), v))
        self.record((tag, layer, "G"), ref.bar_per_segment(g, ref.g_fold(bd, A)))
        self.record((tag, layer, "hid"), ref.bar_rows(hid, ref.mlp0(x, qp, g, A, L), v))
        mu_ref, rstd_ref = ref.in_stats(hid, L)
        self.record((tag, layer, "mu"), ref.bar_mu(mu, mu_ref, rstd_ref, L))
        self.record((tag, layer, "rstd"), ref.bar_rstd(rstd, rstd_ref, L))
        L7, rd7 = self.stop(layer_id, 7, nlen, mlen)
        out = rd7("x")
        out_ref, delta = ref.mlp3(x, hid, mu, rstd, A, L)
        self.record((tag, layer, "x after mlp.3"), ref.bar_x_out(out, out_ref, delta, L))
        return out

    def tail(self, tag, nlen, mlen):
        L, rd = self.stop(12, 3, nlen, mlen)
        x, pn = rd("x"), rd("pn")
        self.record((tag, 12, "pn"), ref.bar_pn(pn, ref.final_proj(x, self.P), L))
        irs, ics, confs = ref.score_tail(pn, L, self.hp["scale_factor"])
        self.record((tag, 12, "1/rowsum"), ref.bar_inverse_sums(rd("inv_rowsum"), irs, self.hp["scale_factor"]))
        self.record((tag, 12, "1/colsum"), ref.bar_inverse_sums(rd("inv_colsum"), ics, self.hp["scale_factor"]))
        i0, _ = ref.unpack_best(self.m.debug_read("rowbest").cpu())
        i1, _ = ref.unpack_best(self.m.debug_read("colbest").cpu())
        bad = 0
        for b in range(L.B):
            n, mm = L.n_of(b), L.m_of(b)
            if n == 0:
                continue
            bad += ref.argmax_mismatches(i0[b, :n], confs[b], 1) + ref.argmax_mismatches(i1[b, :mm], confs[b], 0)
        self.record((tag, 12, "arg-max"), float("inf") if bad else 0.0)

    # ---------------------------------------------------------------- whole call
    def run(self, hoist):
        L = self.L
        mlen = L.mlen
        x = None
        first = 0
        if hoist:
            db, lv = self.objects[0]
            Lo = ref.Layout(1, 0, db.shape[1], 0, ref.round_up(db.shape[1]))
            xo = torch.zeros(Lo.rows, ref.D, dtype=torch.float64)
            xo[:db.shape[1]] = torch.from_numpy(split_roundtrip(db)).double().T
            leaves = [torch.from_numpy(lv).double().T.reshape(db.shape[1], -1, ref.D)]
            xo = self.gats("prologue", 0, 16, xo, Lo, leaves, None, None)
            self.attn("prologue", 1, 17, False, None, None, xo)
            self.attn("query pass", 1, 1, False, self.nlen, None)
            first = 2
        for layer in range(first, 12):
            if ref.GNN_LAYERS[layer] == "GATs":
                x_in = self.x0 if layer == 0 else x
                x = self.gats("chunk", layer, layer, x_in, L, self.leaves_of, self.nlen, mlen)
            else:
                x = self.attn("chunk", layer, layer, ref.GNN_LAYERS[layer] == "cross", self.nlen, mlen, x)
        self.tail("chunk", self.nlen, mlen)
        self.m.debug_stop_after(-1)

    def report(self, title):
        print(f"\n{title}: measured error / bar")
        for (tag, layer, stage), r in self.ratios.items():
            print(f"  {tag:>10} layer {layer:2d} {stage:>14}: {r:.3g}")
        worst = max(self.ratios.items(), key=lambda kv: kv[1])
        assert worst[1] <= 1.0, f"{title}: {worst[0]} at {worst[1]:.3g} x its bar"


# ------------------------------------------------------------------------------------------------------------- cases
ONE_OBJECT = {
    # name: (weights, hparams overrides, (object seed, M, L), frame ids, N, nlen, hoist)
    "fixture_ragged": ("fixture", {}, (9, 300, 8), [100, 101, 102], 200, [200, 1, 137], False),
    "fixture_ragged_hoist": ("fixture", {}, (9, 300, 8), [100, 101, 102], 200, [200, 1, 137], True),
    "attention_live": ("attention_live", {}, (9, 300, 8), [100, 101], 300, None, False),
    "attention_live_hoist": ("attention_live", {}, (9, 700, 8), [100, 101], 129, [129, 40], True),
    "in_offset": ("in_offset", {}, (9, 300, 8), [100, 101], 300, [300, 57], False),
    "l5_hoist": ("fixture", {}, (4, 257, 5), [7, 8], 100, None, True),
    "noself": ("variant", dict(include_self=False), (3, 96, 6), [1, 2], 64, None, False),
    "additional": ("variant", dict(additional=True), (3, 96, 6), [1, 2], 64, None, True),
    "lintrans": ("variant", dict(with_linear_transform=True), (3, 96, 6), [1, 2], 64, [64, 9], False),
    "noself_lintrans": ("variant", dict(include_self=False, with_linear_transform=True), (3, 96, 6), [1, 2], 64, None, True),
    "lintrans_additional": ("variant", dict(with_linear_transform=True, additional=True), (3, 96, 6), [1, 2], 64, None, True),
}


def _weights(kind, hp):
    if kind == "variant":
        return synthetic.make_state_dict(5, hparams=hp)
    sd = synthetic.make_state_dict(4)
    if kind == "attention_live":
        return _attention_live(sd)
    if kind == "in_offset":
        return _in_offset(sd)
    return sd


@pytest.mark.parametrize("name", list(ONE_OBJECT))
def test_stages_one_object(name):
    kind, over, (oseed, M, Lf), frames, N, nlen, hoist = ONE_OBJECT[name]
    hp = dict(synthetic.DEFAULT_HPARAMS, **over)
    sd = _weights(kind, hp)
    data = synthetic.make_batch(oseed, frames, N, M, Lf)
    m = _module(sd, hp, hoist)
    db, lv = data["descriptors3d_db"][0], data["descriptors2d_db"][0]
    m.set_object(torch.from_numpy(db).cuda(), torch.from_numpy(lv).cuda())
    q = torch.from_numpy(data["descriptors2d_query"]).cuda()
    lengths = None if nlen is None else torch.tensor(nlen, dtype=torch.int32).cuda()
    st = Stages(m, lambda: m.match_frames(q, lengths=lengths), oracle.params_from_numpy(sd, torch.float64), hp,
                data["descriptors2d_query"], [(db, lv)] * len(frames), nlen)
    st.run(hoist)
    st.report(name)


MIXED = {
    # name: (objects (seed, M), L, frame -> object, N, nlen, hoist)
    "objects_255_256_257_700": ([(300, 255), (301, 256), (302, 257), (303, 700)], 8, [0, 3, 1, 2, 3, 0], 150, [150, 1, 99, 150, 64, 7], True),
    "objects_255_256_257_700_no_hoist": ([(300, 255), (301, 256), (302, 257), (303, 700)], 8, [3, 0, 2, 1], 150, [150, 1, 99, 150], False),
    # 17 frames of one object in a row: its GATs group is cut at 16; then interleaved objects
    "l8_group_cut_interleaved": ([(310, 100), (311, 60)], 8, [0] * 17 + [1, 0, 1], 40, None, False),
}


@pytest.mark.parametrize("name", list(MIXED))
def test_stages_objects_of_different_sizes(name):
    objs, Lf, order, N, nlen, hoist = MIXED[name]
    hp = dict(synthetic.DEFAULT_HPARAMS)
    sd = synthetic.make_state_dict(4)
    m = _module(sd, hp, hoist)
    host = [synthetic.make_object(seed, M, Lf) for seed, M in objs]
    ids = [m.add_object(torch.from_numpy(db).cuda(), torch.from_numpy(lv).cuda()) for db, lv in host]
    queries = np.stack([synthetic.make_frame(60 + b, host[k][0], N)[0] for b, k in enumerate(order)])
    q = torch.from_numpy(queries).cuda()
    lengths = None if nlen is None else torch.tensor(nlen, dtype=torch.int32).cuda()
    st = Stages(m, lambda: m.match_objects(q, [ids[k] for k in order], lengths=lengths), oracle.params_from_numpy(sd, torch.float64), hp,
                queries, [host[k] for k in order], nlen)
    st.run(hoist)
    st.report(name)


def test_stopped_call_then_hook_off_is_bit_identical_to_a_fresh_handle():
    """A call stopped inside the object prologue, then one inside the chunk; with the hook off, the next call equals a fresh
    handle's bit for bit (the stopped prologue is redone, nothing of the stopped calls leaks into it)."""
    hp = dict(synthetic.DEFAULT_HPARAMS)
    sd = synthetic.make_state_dict(4)
    data = synthetic.make_batch(9, [100, 101], 200, 300, 8)
    q = torch.from_numpy(data["descriptors2d_query"]).cuda()
    db, lv = (torch.from_numpy(data[k][0]).cuda() for k in ("descriptors3d_db", "descriptors2d_db"))
    lengths = torch.tensor([200, 77], dtype=torch.int32).cuda()
    outs = []
    for stops in ([], [(17, 3), (5, 4)]):
        m = _module(sd, hp, True)
        m.set_object(db, lv)
        for layer, step in stops:
            m.debug_stop_after(layer, step)
            m.match_frames(q, lengths=lengths)
            assert m.debug_layout()["B"] >= 1
        m.debug_stop_after(-1)
        outs.append({k: v.clone() for k, v in m.match_frames(q, lengths=lengths).items()})
        m.check_range()
    for k in outs[0]:
        assert torch.equal(outs[0][k], outs[1][k]), k


@pytest.mark.parametrize("kind", ["attention_live", "in_offset"])
def test_stress_weights_end_to_end_against_oracle(kind):
    """The stage tests' stress weights stay inside the fp16-split operand range and meet the usual end-to-end bars."""
    hp = dict(synthetic.DEFAULT_HPARAMS)
    sd = _weights(kind, hp)
    data = synthetic.make_batch(9, [100, 101], 300, 700, 8)
    refo = oracle.forward(oracle.params_from_numpy(sd), data, hp)
    m = _module(sd, hp, True)
    m({k: torch.from_numpy(v).cuda() for k, v in data.items()})
    m.check_range()
    out = m.last_batched
    err = float((out["conf_matrix"].cpu() - refo["conf_matrix"]).abs().max())
    print(f"{kind}: max|dconf| = {err:.2e}")
    assert err <= CONF_TOL
    np.testing.assert_array_equal(out["matches0"].cpu().numpy(), refo["matches0"].numpy())
    np.testing.assert_array_equal(out["matches1"].cpu().numpy(), refo["matches1"].numpy())
