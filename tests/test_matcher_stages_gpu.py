"""Every step of every GNN layer and of the tail against its fp64 stage reference (tests/matcher_stage_reference.py), on the
device's own input to that step: the call is stopped after the step (opb_debug_set_stop) and the buffers are read back
(opb_debug_read).  The end-to-end parity tests cannot see the attention path -- with these weights its message is almost
constant per segment and InstanceNorm removes it (tests/test_matcher_stage_reference_cpu.py measures how blind they are).

Bars, set from the operand formats (fp16-split operands carry ~2^-22 relative down to an absolute 2^-30; 3-pass GEMMs keep
fp32 semantics):
  kvt           one fp16 ulp of fp16(64 ref) / 64 + 2^-11 sum|x||w| (the two-pass projection); pad rows exactly 0
  Kmean         1e-5 of the segment's max
  bd            1e-5 of the segment's max + (n_pad_src / 16 + 1) x 2^-23 sum|k||v| / n (the state kernel's fp32 accumulation
                over the source segment's rows); off-diagonal blocks exactly 0
  Q', G, hid    1e-5 of the row's (G: the segment's) max
  mu            1e-6 (|mu| + sigma);   rstd   1e-5 relative
  X after mlp.3 1e-5 max|layer delta| of the segment + 2^-18 |x| + 16 x 2^-30 (the residual through the fp32 accumulator
                and the split); pad rows exactly 0
  X after GATs  1e-5 of the row's max (the rows before W with with_linear_transform likewise); pad rows exactly 0
  pn            unit rows to 1e-6, elements within 1e-5
  inverse sums  1e-5 + 48 x 2^-23 / scale relative (the score GEMM's fp32 accumulation, amplified by 1 / scale)
  arg-max       equal wherever the fp64 top-1 / top-2 gap exceeds 1e-5 relative (x 0.07 / scale below scale 0.07)
  conf          per entry against (e . irs)(e . ics) with the device's own inverse sums: 2 x 48 x 2^-23 / scale + the fp32
                argument of ex2, ex2.approx and the three products (ref.conf_rel_bar), + 2^-148 absolute below fp32's normal
                range; every entry finite
Exact checks: the query rows of X as the device first holds them equal the fp16-split value of the caller's queries (zero past
each frame's length); with hoisting, X entering layer 2 equals the query pass's output and each frame's object prologue output
bit for bit; the packed arg-maxes are the first maxima of the device's own conf; matches and scores equal `mutual` of the
device's conf; conf is 0 past each frame's N_b rows and M_b columns.
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
    """Runs a call again and again, stopped after one step each time, and checks that step against its reference.

    chunk / chunk_frames: the chunk of the call to walk (chunk_frames = the handle's frames per chunk); piece / piece_frames: the
    sub-batch of the hoisted query pass whose stages are checked, and the frames per sub-batch (16 for match_frames_host, else
    the chunk).  solo(b): a one-frame call whose frame uses frame b's object (calls of several objects, for their prologues).
    The references run in fp64 on the GPU (ATen, none of the project's kernels)."""

    def __init__(self, m, call, P, hp, queries, objects, nlen, chunk=0, chunk_frames=None, piece=0, piece_frames=None, solo=None):
        self.m, self.call, self.hp, self.solo = m, call, hp, solo
        self.dev = torch.device("cuda", torch.cuda.current_device())
        self.P = {k: v.to(self.dev) for k, v in P.items()}
        B = queries.shape[0]
        cf = chunk_frames or min(B, 32)
        self.chunk, self.f0 = chunk, chunk * cf
        fb = min(cf, B - self.f0)
        self.piece, self.piece_frames = piece, piece_frames or cf
        self.call_objects = objects
        # the chunk's inputs as the device holds them (fp16-split planes; frames of one object share one copy); leaves stay fp32
        rt = {}
        for db, lv in objects:
            if id(db) not in rt:
                rt[id(db)] = (split_roundtrip(db), lv)
        held = [rt[id(db)] for db, _ in objects]
        self.objects = held[self.f0:self.f0 + fb]
        self.q_rt = split_roundtrip(queries[self.f0:self.f0 + fb])
        self.nlen = None if nlen is None else list(nlen[self.f0:self.f0 + fb])
        self.ratios = {}
        self.info = {}          # printed, not asserted: bd against the bar it had before the accumulation term
        x, self.leaves_of, self.L = ref.assemble(self.q_rt, self.objects, self.nlen, self.dev)
        self.x0 = x

    def stop(self, layer, step, nlen=None, mlen=None, piece=0):
        self.m.debug_stop_after(layer, step, self.chunk, piece)
        self.call()
        L = ref.Layout.of(self.m.debug_layout(), nlen, mlen)
        return L, (lambda name: self.m.debug_read(name).double())

    def record(self, key, ratio):
        self.ratios[key] = ratio

    def exact(self, key, same):
        self.record(key, 0.0 if same else float("inf"))

    def invalidate_prologues(self):
        """The next call runs the object prologue of every object again."""
        self.m.debug_invalidate_prologues()

    def query_rows(self, frames, n_pad):
        """The query rows of `frames` (chunk-relative) as the device first holds them [len(frames) * n_pad, 256]: the fp16-split
        value of the caller's queries, zero past each frame's length (whatever the caller left there)."""
        out = torch.zeros(len(frames), n_pad, ref.D, dtype=torch.float64, device=self.dev)
        for i, b in enumerate(frames):
            n = self.q_rt.shape[2] if self.nlen is None else self.nlen[b]
            out[i, :n] = torch.from_numpy(self.q_rt[b][:, :n].T.copy()).to(self.dev, torch.float64)
        return out.view(-1, ref.D)

    # ---------------------------------------------------------------- layers
    def gats(self, tag, layer, layer_id, x_in, Lx, leaves_of, nlen, mlen):
        last = 1 if self.hp["with_linear_transform"] else 0
        L, rd = self.stop(layer_id, last, nlen, mlen)
        assert (L.B, L.N, L.M, L.n_pad, L.m_pad) == (Lx.B, Lx.N, Lx.M, Lx.n_pad, Lx.m_pad)
        out, pre = ref.gats_layer(x_in, leaves_of, self.P, layer, self.hp, L)
        x = rd("x")
        self.record((tag, layer, "gats"), ref.bar_gats(x, out, L))
        if last:
            rows = torch.zeros(L.B * L.m_pad, dtype=torch.bool, device=self.dev)
            for b in range(L.B):
                rows[b * L.m_pad:b * L.m_pad + L.m_of(b)] = True
            self.record((tag, layer, "gats pre-W"), ref.bar_rows(rd("gats_pre"), pre, rows))
        return x

    def attn(self, tag, layer, layer_id, cross, nlen, mlen, x_prev=None, piece=0):
        A = ref.attn_weights(self.P, layer)
        L, rd = self.stop(layer_id, 6, nlen, mlen, piece)
        x = rd("x")
        if x_prev is not None:      # the previous stage's output, or the hand-off the layer starts from
            self.exact((tag, layer, "X in"), torch.equal(x, x_prev))
        v = L.valid_mask(self.dev)
        kvt = rd("kvt")
        kvt_ref, absprod = ref.kv_proj(x, A, L)
        self.record((tag, layer, "kvt"), ref.bar_kvt(kvt, kvt_ref, absprod, L))
        del kvt_ref, absprod
        kmean, bd = rd("kmean"), rd("bd")
        kmean_ref, bd_ref = ref.kv_state(kvt, L, cross)
        absbd = ref.kv_state(kvt.abs(), L, cross)[1]
        del kvt
        self.record((tag, layer, "kmean"), ref.bar_per_segment(kmean, kmean_ref))
        self.record((tag, layer, "bd"), ref.bar_bd(bd, bd_ref, absbd, L, cross))
        self.info[(tag, layer, "bd / 1e-5 of max")] = ref.bar_bd(bd, bd_ref)
        del bd_ref, absbd
        qp = rd("qp")
        self.record((tag, layer, "Q'"), ref.bar_rows(qp, ref.q_proj(x, kmean, A, L, cross), v))
        g = rd("g")
        self.record((tag, layer, "G"), ref.bar_per_segment(g, ref.g_fold(bd, A)))
        del bd
        hid = rd("hid")
        self.record((tag, layer, "hid"), ref.bar_rows(hid, ref.mlp0(x, qp, g, A, L), v))
        del qp, g
        mu, rstd = rd("mu"), rd("rstd")
        mu_ref, rstd_ref = ref.in_stats(hid, L)
        self.record((tag, layer, "mu"), ref.bar_mu(mu, mu_ref, rstd_ref, L))
        self.record((tag, layer, "rstd"), ref.bar_rstd(rstd, rstd_ref, L))
        L7, rd7 = self.stop(layer_id, 7, nlen, mlen, piece)
        out = rd7("x")
        out_ref, delta = ref.mlp3(x, hid, mu, rstd, A, L)
        self.record((tag, layer, "x after mlp.3"), ref.bar_x_out(out, out_ref, delta, L))
        return out

    def tail(self, tag, nlen, mlen):
        """Every stage of the tail on the device's own input, and the call's outputs entry by entry: conf against (e . irs)(e . ics)
        from the device's pn and inverse sums (ref.conf_rel_bar), the packed arg-maxes against the first maximum of the device's
        own conf rows and columns, the matches and scores against `mutual` of the device's conf, and exact zeros past each
        frame's N_b and M_b.  conf and the matches come from an unstopped call (repeat calls are bit-identical)."""
        scale, thr = self.hp["scale_factor"], self.hp["match_threshold"]
        L, rd = self.stop(12, 3, nlen, mlen)
        pn = rd("pn")
        self.record((tag, 12, "pn"), ref.bar_pn(pn, ref.final_proj(rd("x"), self.P), L))
        irs, ics = rd("inv_rowsum"), rd("inv_colsum")
        i0, v0 = ref.unpack_best(self.m.debug_read("rowbest"))
        i1, v1 = ref.unpack_best(self.m.debug_read("colbest"))
        self.m.debug_stop_after(-1)
        out = self.call()
        irs_ref, ics_ref = torch.zeros_like(irs), torch.zeros_like(ics)
        conf_worst, bad_argmax, bad_first, bad_mutual, bad_zero = 0.0, 0, 0, 0, 0
        for b in range(L.B):
            f = self.f0 + b
            n, mm = L.n_of(b), L.m_of(b)
            conf = out["conf_matrix"][f].to(self.dev)
            m0, m1, s0, s1 = (out[k][f].to(self.dev) for k in ("matches0", "matches1", "matching_scores0", "matching_scores1"))
            bad_zero += int((conf[n:] != 0).sum() + (conf[:, mm:] != 0).sum())
            bad_mutual += int((m0[n:] != -1).sum() + (s0[n:] != 0).sum() + (m1[mm:] != -1).sum() + (s1[mm:] != 0).sum())
            if n == 0:          # a frame without queries matches nothing
                bad_mutual += int((m1 != -1).sum() + (s1 != 0).sum())
                continue
            cos = pn[L.seg_rows(2 * b)] @ pn[L.seg_rows(2 * b + 1)].T
            e = torch.exp((cos - 1.0) / scale)
            rs, cs = e.sum(1), e.sum(0)
            irs_ref[b, :n], ics_ref[b, :mm] = 1.0 / rs, 1.0 / cs
            conf64 = e * e / rs[:, None] / cs[None, :]
            del e
            gap = ref.decided_gap(scale)
            bad_argmax += ref.argmax_mismatches(i0[b, :n], conf64, 1, gap) + ref.argmax_mismatches(i1[b, :mm], conf64, 0, gap)
            del conf64
            c = conf[:n, :mm]
            conf_worst = max(conf_worst, ref.bar_conf(c, cos, irs[b, :n], ics[b, :mm], scale))
            bad_first += ref.first_max_mismatches(i0[b, :n], v0[b, :n], c, 1) + ref.first_max_mismatches(i1[b, :mm], v1[b, :mm], c, 0)
            bad_mutual += ref.mutual_mismatches(m0[:n], m1[:mm], s0[:n], s1[:mm], c, thr)
            del cos, c, conf
        self.record((tag, 12, "1/rowsum"), ref.bar_inverse_sums(irs, irs_ref, scale))
        self.record((tag, 12, "1/colsum"), ref.bar_inverse_sums(ics, ics_ref, scale))
        self.exact((tag, 12, "arg-max"), bad_argmax == 0)
        self.record((tag, 12, "conf"), conf_worst)
        self.exact((tag, 12, "conf zero pad"), bad_zero == 0)
        self.exact((tag, 12, "arg-max = first max"), bad_first == 0)
        self.exact((tag, 12, "mutual"), bad_mutual == 0)

    # ---------------------------------------------------------------- hoisting: the hand-off into layer 2
    def prologue_outputs(self, xo_first):
        """X of each object of the chunk after its prologue (stop 17/7), keyed by the chunk frame that first uses it.  The call's
        first frame's object is `xo_first`; the others come from one-frame calls."""
        outs, first_id = {}, id(self.call_objects[0][0])
        for b, (db, _) in enumerate(self.call_objects[self.f0:self.f0 + self.L.B]):
            if id(db) in outs:
                continue
            if id(db) == first_id:
                outs[id(db)] = xo_first
            else:
                self.invalidate_prologues()
                self.m.debug_stop_after(17, 7)
                self.solo(self.f0 + b)
                outs[id(db)] = self.m.debug_read("x").double()
        return [outs[id(db)] for db, _ in self.call_objects[self.f0:self.f0 + self.L.B]]

    # ---------------------------------------------------------------- whole call
    def run(self, hoist):
        L = self.L
        mlen = L.mlen
        x = None
        first = 0
        if hoist:
            self.invalidate_prologues()
            db, lv = self.call_objects[0]
            Lo = ref.Layout(1, 0, db.shape[1], 0, ref.round_up(db.shape[1]))
            xo = torch.zeros(Lo.rows, ref.D, dtype=torch.float64, device=self.dev)
            xo[:db.shape[1]] = torch.from_numpy(split_roundtrip(db)).to(self.dev, torch.float64).T
            leaves = [torch.from_numpy(lv).to(self.dev, torch.float64).T.reshape(db.shape[1], -1, ref.D)]
            xo = self.gats("prologue", 0, 16, xo, Lo, leaves, None, None)
            xo = self.attn("prologue", 1, 17, False, None, None, xo)
            prologue = self.prologue_outputs(xo)
            # the query pass, sub-batch by sub-batch: its input rows, its stages (sub-batch self.piece) and its output
            qpass = []
            for si, p0 in enumerate(range(0, L.B, self.piece_frames)):
                frames = range(p0, min(p0 + self.piece_frames, L.B))
                nl = None if self.nlen is None else self.nlen[p0:frames.stop]
                Lq, rd = self.stop(1, 0, nl, None, si)
                self.exact(("query pass", 1, f"rows in [{si}]"), torch.equal(rd("x"), self.query_rows(frames, L.n_pad)))
                if si == self.piece:
                    qpass.append(self.attn("query pass", 1, 1, False, nl, None, piece=si))
                else:
                    qpass.append(self.stop(1, 7, nl, None, si)[1]("x"))
            # X entering layer 2: each frame's query-pass rows and its object's prologue rows, pad rows zero
            x = torch.zeros(L.rows, ref.D, dtype=torch.float64, device=self.dev)
            q_all = torch.cat(qpass).view(L.B, L.n_pad, ref.D)
            for b in range(L.B):
                x[L.seg_rows(2 * b)] = q_all[b, :L.n_of(b)]
                x[L.seg_rows(2 * b + 1)] = prologue[b][:L.m_of(b)]
            del q_all, qpass, prologue
            first = 2
        for layer in range(first, 12):
            if ref.GNN_LAYERS[layer] == "GATs":
                x_in = self.x0 if layer == 0 else x
                x = self.gats("chunk", layer, layer, x_in, L, self.leaves_of, self.nlen, mlen)
                if layer == 0:      # GATs leaves the query rows alone: they are still the rows the transpose wrote
                    q = x.view(L.B, L.R, ref.D)[:, :L.n_pad].reshape(-1, ref.D)
                    self.exact(("chunk", 0, "query rows in"), torch.equal(q, self.query_rows(range(L.B), L.n_pad)))
            else:
                x = self.attn("chunk", layer, layer, ref.GNN_LAYERS[layer] == "cross", self.nlen, mlen, x)
        del x
        self.tail("chunk", self.nlen, mlen)
        self.m.debug_stop_after(-1)

    def report(self, title):
        print(f"\n{title}: measured error / bar")
        for (tag, layer, stage), r in self.ratios.items():
            print(f"  {tag:>10} layer {layer:2d} {stage:>20}: {r:.3g}")
        if self.info:
            print(f"  worst bd against 1e-5 of the segment's max alone (not asserted): {max(self.info.values()):.3g}")
        worst = max(self.ratios.items(), key=lambda kv: kv[1] if kv[1] == kv[1] else float("inf"))
        assert worst[1] <= 1.0, f"{title}: {worst[0]} at {worst[1]:.3g} x its bar"


# ------------------------------------------------------------------------------------------------------------- cases
ONE_OBJECT = {
    # name: (weights, hparams overrides, (object seed, M, L), frame ids, N, nlen, hoist)
    "fixture_ragged": ("fixture", {}, (9, 300, 8), [100, 101, 102, 103], 200, [200, 1, 0, 137], False),
    "fixture_ragged_hoist": ("fixture", {}, (9, 300, 8), [100, 101, 102, 103], 200, [200, 0, 1, 137], True),
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
                queries, [host[k] for k in order], nlen,
                solo=lambda b: m.match_objects(q[b:b + 1], [ids[order[b]]], lengths=None if lengths is None else lengths[b:b + 1]))
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


def test_stage_reference_on_the_gpu_equals_the_cpu_run():
    """The fp64 stage references allocate on their input's device: the chain on CUDA (ATen) equals the CPU chain to 1e-12, at a
    ragged shape with frames of two objects."""
    hp = dict(synthetic.DEFAULT_HPARAMS)
    sd = synthetic.make_state_dict(4, damped=False)
    objs = [synthetic.make_object(300 + k, M, 5) for k, M in enumerate([257, 40])]
    order = [0, 1, 0]
    q = np.stack([synthetic.make_frame(50 + b, objs[k][0], 90)[0] for b, k in enumerate(order)])
    P = oracle.params_from_numpy(sd, torch.float64)
    outs = [ref.chain_forward({k: v.to(d) for k, v in P.items()}, hp, q, [objs[k] for k in order], [90, 1, 33], device=d)
            for d in ("cpu", "cuda")]
    (c_cpu, m_cpu), (c_gpu, m_gpu) = outs
    for b in range(len(order)):
        err = float(((c_gpu[b].cpu() - c_cpu[b]).abs() / c_cpu[b].abs().clamp_min(1e-300)).max()) if c_cpu[b].numel() else 0.0
        assert err <= 1e-12, (b, err)
        for t_gpu, t_cpu in zip(m_gpu[b], m_cpu[b]):
            if t_cpu.dtype == torch.int64:
                assert torch.equal(t_gpu.cpu(), t_cpu), b
            else:
                assert torch.allclose(t_gpu.cpu(), t_cpu, rtol=1e-12, atol=0), b


@pytest.mark.parametrize("hoist", [True, False])
def test_frame_without_queries_leaves_the_other_frames_intact(hoist):
    """A frame of length 0 is valid input.  In a cross layer its 3D points have no source rows and receive no message; the
    call stays inside the fp16-split range (check_range passes), the empty frame matches nothing, and every other frame equals
    the oracle run on its own queries."""
    hp = dict(synthetic.DEFAULT_HPARAMS)
    sd = synthetic.make_state_dict(0)
    M, N = 300, 160
    lens = [160, 0, 97, 0]
    db, leaves = synthetic.make_object(5, M, 8)
    q = np.full((len(lens), 256, N), 7.0, np.float32)
    refs = {}
    for b, n in enumerate(lens):
        if n:
            q[b, :, :n] = synthetic.make_frame(70 + b, db, n)[0]
            data = {"keypoints2d": np.zeros((1, n, 2), np.float32), "keypoints3d": np.zeros((1, M, 3), np.float32),
                    "descriptors2d_query": q[b:b + 1, :, :n].copy(), "descriptors3d_db": db[None], "descriptors2d_db": leaves[None]}
            refs[b] = oracle.forward(oracle.params_from_numpy(sd), data, hp)
    m = _module(sd, hp, hoist)
    m.set_object(torch.from_numpy(db).cuda(), torch.from_numpy(leaves).cuda())
    out = m.match_frames(torch.from_numpy(q).cuda(), lengths=torch.tensor(lens, dtype=torch.int32).cuda())
    m.check_range()
    for b, n in enumerate(lens):
        conf = out["conf_matrix"][b].cpu()
        if n == 0:
            assert float(conf.abs().max()) == 0.0, b
            assert bool((out["matches0"][b] == -1).all()) and bool((out["matches1"][b] == -1).all()), b
            assert float(out["matching_scores0"][b].abs().sum() + out["matching_scores1"][b].abs().sum()) == 0.0, b
            continue
        r = refs[b]
        assert float((conf[:n] - r["conf_matrix"][0]).abs().max()) <= CONF_TOL, b
        np.testing.assert_array_equal(out["matches0"][b, :n].cpu().numpy(), r["matches0"][0].numpy())
        np.testing.assert_array_equal(out["matches1"][b].cpu().numpy(), r["matches1"][0].numpy())
        assert int((out["matches0"][b] > -1).sum()) > 0, b
