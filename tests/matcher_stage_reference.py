"""fp64 references of the matcher's GNN stages, in the device's layout.

Each function restates one step of the CUDA path (api.cu: run_attn_layer, run_gats, the tail of forward_chunk) on the tensors
the device works on, so that a test can feed it the device's own input to that step (read through opb_debug_read) and compare
the step's output alone.  Conventions of the device layout (DESIGN section 3, common.cuh):
  * activation rows: frame b owns rows [b R, b R + n_pad) (queries, nlen[b] valid) and [b R + n_pad, (b + 1) R) (3D points,
    mlen[b] valid); segment 2 b is the query side, 2 b + 1 the 3D side; pad rows of X are zero;
  * attention channels are head-contiguous: c' = h * 64 + d holds the reference's channel d * 4 + h (GATs_SuperGlue.py:97);
  * bd[s] is indexed by DESTINATION segment s and holds KVmean of its source segment (s itself, or s ^ 1 in a cross layer).
The weights come from the reference-keyed state dict, never from the library's packed weights.  ``chain_forward`` composes the
stages into the whole forward (tests/test_matcher_stage_reference_cpu.py checks it against the oracle), and ``Defect`` plants
the errors the end-to-end suite cannot see.  ``bar_*`` return the error of a device result as a multiple of its bar (<= 1
passes).  Every function allocates on the device of its inputs: the large stage cases run the same fp64 code through ATen on
the GPU (none of the project's kernels), the small ones and the CPU tests on the CPU."""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np
import torch
import torch.nn.functional as F

D, H, DH, SEG = 256, 4, 64, 256
GNN_LAYERS = ["GATs", "self", "cross"] * 4
PERM = torch.tensor([d * H + h for h in range(H) for d in range(DH)])   # head-contiguous c' -> reference channel
TINY = 1e-300


def round_up(x, m=SEG):
    return (x + m - 1) // m * m


@dataclass
class Layout:
    """Python twin of opb::Layout; nlen / mlen: per-frame valid counts (None: N / M everywhere)."""
    B: int
    N: int
    M: int
    n_pad: int
    m_pad: int
    nlen: list | None = None
    mlen: list | None = None
    R: int = field(init=False)

    def __post_init__(self):
        self.R = self.n_pad + self.m_pad

    @classmethod
    def of(cls, d: dict, nlen=None, mlen=None):
        L = cls(d["B"], d["N"], d["M"], d["n_pad"], d["m_pad"], nlen, mlen)
        assert L.R == d["R"] and 2 * L.B == d["S"]
        return L

    @property
    def rows(self):
        return self.B * self.R

    @property
    def S(self):
        return 2 * self.B

    def n_of(self, b):
        return self.N if self.nlen is None else int(self.nlen[b])

    def m_of(self, b):
        return self.M if self.mlen is None else int(self.mlen[b])

    def seg_start(self, s):
        return (s >> 1) * self.R + (self.n_pad if s & 1 else 0)

    def seg_padded(self, s):
        return self.m_pad if s & 1 else self.n_pad

    def seg_valid(self, s):
        return self.m_of(s >> 1) if s & 1 else self.n_of(s >> 1)

    def seg_rows(self, s, padded=False):
        a = self.seg_start(s)
        return slice(a, a + (self.seg_padded(s) if padded else self.seg_valid(s)))

    @staticmethod
    def src_seg(s, cross):
        return s ^ 1 if cross else s

    def valid_mask(self, device="cpu"):
        v = torch.zeros(self.rows, dtype=torch.bool, device=device)
        for s in range(self.S):
            v[self.seg_rows(s)] = True
        return v

    def seg_index(self, device="cpu"):
        """Segment of every row [rows]."""
        r = torch.arange(self.rows, device=device)
        return 2 * (r // self.R) + ((r % self.R) >= self.n_pad).long()


@dataclass
class Defect:
    """Planted errors, one stage each (all off by default)."""
    msg_scale: float = 1.0          # G fold: the message scaled (e.g. a 1 % error in the Q' denominator)
    rotate_heads: bool = False      # q projection: head h's Q' taken from head h + 1
    own_side: bool = False          # state reduce: a cross layer's bd from its own segment
    mean_over_pad: bool = False     # state reduce: Kmean / KVmean divided by the padded row count
    kvt_pad_rows: bool = False      # k,v projection: pad rows not zeroed
    in_stats_pad: bool = False      # InstanceNorm statistics over the padded rows
    conf_zero_below: float = 0.0    # conf epilogue: entries below this written as 0
    conf_neighbour_ics: bool = False  # conf epilogue: column j uses the inverse sum of column j + 1 (within its 32-column chunk)
    ms1_wrong_row: bool = False     # mutual: matching_scores1[m] taken from the row after its arg-max row


NO_DEFECT = Defect()


# ------------------------------------------------------------------------------------------------ weights
def attn_weights(P, i):
    """Layer i's AttentionPropagation weights in the device's channel order (fp64 torch)."""
    p = f"gnn.layers.{i}"
    w = lambda k: P[f"{p}.{k}.weight"][:, :, 0].double()
    b = lambda k: P[f"{p}.{k}.bias"].double()
    W0 = w("mlp.0")
    perm = PERM.to(W0.device)
    return {"Wq": w("attn.proj.0")[perm], "bq": b("attn.proj.0")[perm], "Wk": w("attn.proj.1")[perm], "bk": b("attn.proj.1")[perm],
            "Wv": w("attn.proj.2")[perm], "bv": b("attn.proj.2")[perm], "W0a": W0[:, :D], "W0msg": W0[:, D:],
            "Wm": w("attn.merge"), "bm": b("attn.merge"), "b0": b("mlp.0"), "W1": w("mlp.3"), "b1": b("mlp.3")}


def _elu1(x):
    return F.elu(x) + 1.0


# ------------------------------------------------------------------------------------------------ attention layer stages
def kv_proj(x, A, L: Layout, defect=NO_DEFECT):
    """Step 0: kvt [rows, 512] = [elu(x Wk^T + bk) + 1 | x Wv^T + bv], pad rows zero.  Also the bar's scale sum |x| |W|."""
    k = _elu1(x @ A["Wk"].T + A["bk"])
    v = x @ A["Wv"].T + A["bv"]
    kvt = torch.cat([k, v], 1)
    if not defect.kvt_pad_rows:
        kvt[~L.valid_mask(x.device)] = 0.0
    absprod = x.abs() @ torch.cat([A["Wk"], A["Wv"]], 0).abs().T
    return kvt, absprod


def kv_state(kvt, L: Layout, cross, defect=NO_DEFECT):
    """Steps 1-2: Kmean [S, 256] of each segment and bd [S, 256, 256] = blockdiag(KVmean of the source segment).  The sums run
    over the segment's padded rows (the device's row groups do; the k,v projection leaves its pad rows zero) and divide by the
    valid count."""
    S, dev = L.S, kvt.device
    kmean = torch.zeros(S, D, dtype=torch.float64, device=dev)
    kv = torch.zeros(S, H, DH, DH, dtype=torch.float64, device=dev)
    for s in range(S):
        n = L.seg_padded(s) if defect.mean_over_pad else L.seg_valid(s)
        if n == 0:
            continue
        rows = kvt[L.seg_rows(s, padded=True)]
        k, v = rows[:, :D], rows[:, D:]
        kmean[s] = k.sum(0) / n
        for h in range(H):
            kv[s, h] = k[:, h * DH:(h + 1) * DH].T @ v[:, h * DH:(h + 1) * DH] / n
    bd = torch.zeros(S, D, D, dtype=torch.float64, device=dev)
    for s in range(S):
        src = s if defect.own_side else L.src_seg(s, cross)
        for h in range(H):
            bd[s, h * DH:(h + 1) * DH, h * DH:(h + 1) * DH] = kv[src, h]
    return kmean, bd


def q_proj(x, kmean, A, L: Layout, cross, defect=NO_DEFECT):
    """Step 3: Q' [rows, 256] = elu1(q) / (elu1(q) . Kmean_src + 1e-6 / m_src) per head (GATs_SuperGlue.py:77-80); 0 on the rows
    of a segment whose source has no valid rows (the 3D side of a frame without queries, in a cross layer): no message."""
    q = _elu1(x @ A["Wq"].T + A["bq"])
    seg = L.seg_index(x.device)
    src = seg ^ 1 if cross else seg
    m_src = torch.tensor([max(L.seg_valid(int(s)), 1) for s in range(L.S)], dtype=torch.float64, device=x.device)[src]
    qh = q.view(-1, H, DH)
    den = (qh * kmean[src].view(-1, H, DH)).sum(2) + 1e-6 / m_src[:, None]
    out = qh / den[:, :, None]
    empty_src = torch.tensor([L.seg_valid(int(s)) == 0 for s in range(L.S)], device=x.device)[src]
    out[empty_src] = 0.0            # no source rows (a frame without queries, cross layer): no message
    if defect.rotate_heads:
        out = out.roll(-1, dims=1)
    return out.reshape(-1, D)


def g_fold(bd, A, defect=NO_DEFECT):
    """Step 4: G[s] = W0msg . Wm[:, perm] . bd[s]^T  [S, 512, 256]: merge and the message half of mlp.0 folded into one weight."""
    w0m = A["W0msg"] @ A["Wm"][:, PERM]
    return defect.msg_scale * torch.einsum("ck,sjk->scj", w0m, bd)


def mlp0(x, qp, G, A, L: Layout):
    """Step 5: hid [rows, 512] = x W0a^T + Q' G[seg]^T + b0 + W0msg bm."""
    b0f = A["b0"] + A["W0msg"] @ A["bm"]
    hid = x @ A["W0a"].T + b0f
    for s in range(L.S):
        r = L.seg_rows(s, padded=True)
        hid[r] += qp[r] @ G[s].T
    return hid


def in_stats(hid, L: Layout, defect=NO_DEFECT):
    """Step 6: InstanceNorm1d statistics per segment over its valid rows, two-pass: mu, rstd [S, 512]."""
    mu = torch.zeros(L.S, 2 * D, dtype=torch.float64, device=hid.device)
    rstd = torch.full((L.S, 2 * D), 1.0 / np.sqrt(1e-5), dtype=torch.float64, device=hid.device)
    for s in range(L.S):
        rows = hid[L.seg_rows(s, padded=defect.in_stats_pad)]
        if rows.shape[0] == 0:
            continue
        mu[s] = rows.mean(0)
        rstd[s] = 1.0 / torch.sqrt(((rows - mu[s]) ** 2).mean(0) + 1e-5)
    return mu, rstd


def mlp3(x, hid, mu, rstd, A, L: Layout):
    """Step 7: x + mlp.3(ReLU(IN(hid))), pad rows zero.  Returns (x_out, delta)."""
    seg = L.seg_index(x.device)
    hn = torch.relu((hid - mu[seg]) * rstd[seg])
    delta = hn @ A["W1"].T + A["b1"]
    out = x + delta
    out[~L.valid_mask(x.device)] = 0.0
    return out, delta


def attn_layer(x, A, L: Layout, cross, defect=NO_DEFECT):
    kvt, _ = kv_proj(x, A, L, defect)
    kmean, bd = kv_state(kvt, L, cross, defect)
    qp = q_proj(x, kmean, A, L, cross, defect)
    G = g_fold(bd, A, defect)
    hid = mlp0(x, qp, G, A, L)
    mu, rstd = in_stats(hid, L, defect)
    return mlp3(x, hid, mu, rstd, A, L)[0]


# ------------------------------------------------------------------------------------------------ GATs layer
def gats_rows(h3, leaves, W, a, hp):
    """GraphAttentionLayer (GATs.py:35-88) on one object's valid 3D rows h3 [M, 256] with its leaves [M, Lf, 256].
    Returns (out [M, 256], pre [M, 256]): pre = the aggregated rows before W (with_linear_transform's first step)."""
    W, a = W.double(), a.double()[:, 0]
    s3 = h3 @ (W @ a[D:])
    s2 = leaves @ (W @ a[:D])
    e = F.leaky_relu(s3[:, None] + s2, 0.2)
    if hp["include_self"]:
        e = torch.cat([F.leaky_relu(2 * s3, 0.2)[:, None], e], 1)
    att = torch.softmax(e, 1)
    if hp["include_self"]:
        pre = att[:, :1] * h3 + (att[:, 1:, None] * leaves).sum(1)
    else:
        pre = (att[:, :, None] * leaves).sum(1) / 2 + h3
    if hp["with_linear_transform"]:
        hpre = pre @ W if hp["include_self"] else (att[:, :, None] * leaves).sum(1) / 2 @ W + h3 @ W
        if hp["include_self"] and hp["additional"]:
            hpre = hpre + h3
    else:
        hpre = pre + h3 if (hp["include_self"] and hp["additional"]) else pre
    return F.elu(hpre), pre


def gats_layer(x, leaves_of, P, i, hp, L: Layout):
    """GATs layer i on the 3D segments of x; leaves_of[b] = frame b's leaves [M_b, Lf, 256] (fp64).  Returns (x_out, pre)."""
    out = x.clone()
    pre = torch.zeros(L.B * L.m_pad, D, dtype=torch.float64, device=x.device)
    for b in range(L.B):
        r = L.seg_rows(2 * b + 1)
        o, p = gats_rows(x[r], leaves_of[b], P[f"gnn.layers.{i}.W"], P[f"gnn.layers.{i}.a"], hp)
        out[r] = o
        pre[b * L.m_pad:b * L.m_pad + L.m_of(b)] = p
    return out, pre


# ------------------------------------------------------------------------------------------------ tail
def final_proj(x, P):
    """pn = F.normalize(x Wf^T + bf) per row (GATs_SuperGlue.py:209-213)."""
    y = x @ P["final_proj.weight"][:, :, 0].double().T + P["final_proj.bias"].double()
    return F.normalize(y, p=2, dim=1)


def conf_entries(e, irs, ics, defect=NO_DEFECT):
    """conf = (e / rowsum) (e / colsum) of one frame, as the conf epilogue forms it: (e . irs) . (e . ics)."""
    if defect.conf_neighbour_ics:
        j = torch.arange(ics.shape[0], device=ics.device)
        ics = ics[torch.where((j % 32 != 31) & (j + 1 < ics.shape[0]), j + 1, j)]
    conf = (e * irs[:, None]) * (e * ics[None, :])
    if defect.conf_zero_below:
        conf = torch.where(conf < defect.conf_zero_below, torch.zeros_like(conf), conf)
    return conf


def score_tail(pn, L: Layout, scale, defect=NO_DEFECT):
    """From the unit rows: inverse row / column sums of e = exp((cos - 1) / scale) ([B, n_pad], [B, m_pad], zero past the
    valid counts), conf per frame [N_b, M_b] and the raw arg-maxes (lowest index on ties)."""
    irs = torch.zeros(L.B, L.n_pad, dtype=torch.float64, device=pn.device)
    ics = torch.zeros(L.B, L.m_pad, dtype=torch.float64, device=pn.device)
    confs = []
    for b in range(L.B):
        q, d = pn[L.seg_rows(2 * b)], pn[L.seg_rows(2 * b + 1)]
        e = torch.exp((q @ d.T - 1.0) / scale)
        rs, cs = e.sum(1), e.sum(0)
        irs[b, :len(rs)] = 1.0 / rs
        if q.shape[0]:
            ics[b, :len(cs)] = 1.0 / cs
        confs.append(conf_entries(e, 1.0 / rs, 1.0 / cs, defect))
    return irs, ics, confs


def mutual(conf, thr, defect=NO_DEFECT):
    """Mutual nearest neighbour + threshold (GATs_SuperGlue.py:220-230) of one frame's conf [N_b, M_b]."""
    i0, i1 = conf.argmax(1), conf.argmax(0)
    v0 = conf.max(1).values
    mutual0 = torch.arange(conf.shape[0], device=conf.device) == i1[i0]
    mutual1 = torch.arange(conf.shape[1], device=conf.device) == i0[i1]
    ms0 = torch.where(mutual0, v0, torch.zeros_like(v0))
    src = ms0.roll(-1) if defect.ms1_wrong_row else ms0
    ms1 = torch.where(mutual1, src[i1], torch.zeros_like(ms0[i1]))
    valid0 = mutual0 & (ms0 > thr)
    valid1 = mutual1 & valid0[i1]
    return torch.where(valid0, i0, -1), torch.where(valid1, i1, -1), ms0, ms1


# ------------------------------------------------------------------------------------------------ composition
def assemble(queries, objects, nlen=None, device="cpu"):
    """Device layout of a chunk in fp64: queries [B, 256, N] (columns past nlen[b] ignored), objects[b] = (db [256, M_b],
    leaves [256, M_b * Lf]).  Returns (x [rows, 256], leaves_of, L); frames that share an object share its leaves tensor."""
    B, _, N = queries.shape
    Ms = [o[0].shape[1] for o in objects]
    L = Layout(B, N, max(Ms), round_up(N), round_up(max(Ms)), None if nlen is None else list(nlen),
               None if len(set(Ms)) == 1 else Ms)
    x = torch.zeros(L.rows, D, dtype=torch.float64, device=device)
    leaves_of, seen = [], {}
    for b in range(B):
        n = L.n_of(b)
        x[L.seg_rows(2 * b)] = torch.as_tensor(queries[b][:, :n]).to(device, torch.float64).T
        key = (id(objects[b][0]), id(objects[b][1]))
        if key not in seen:
            db, lv = (torch.as_tensor(t).to(device, torch.float64) for t in objects[b])
            seen[key] = (db.T, lv.T.reshape(db.shape[1], -1, D))
        x[L.seg_rows(2 * b + 1)] = seen[key][0]
        leaves_of.append(seen[key][1])
    return x, leaves_of, L


def gnn(x, leaves_of, P, hp, L: Layout, defect=NO_DEFECT, defect_layers=range(12)):
    for i, kind in enumerate(GNN_LAYERS):
        d = defect if i in defect_layers else NO_DEFECT
        if kind == "GATs":
            x = gats_layer(x, leaves_of, P, i, hp, L)[0]
        else:
            x = attn_layer(x, attn_weights(P, i), L, kind == "cross", d)
    return x


def chain_forward(P, hp, queries, objects, nlen=None, defect=NO_DEFECT, defect_layers=range(12), device="cpu"):
    """The whole forward as the composition of the stages: per frame conf [N_b, M_b] and (matches0, matches1, ms0, ms1).
    P: fp64 parameters on `device`."""
    x, leaves_of, L = assemble(queries, objects, nlen, device)
    x = gnn(x, leaves_of, P, hp, L, defect, defect_layers)
    _, _, confs = score_tail(final_proj(x, P), L, hp["scale_factor"], defect)
    return confs, [mutual(c, hp["match_threshold"], defect) for c in confs]


# ------------------------------------------------------------------------------------------------ bars
def _ratio(err, allowed):
    err = torch.as_tensor(err, dtype=torch.float64)
    allowed = torch.as_tensor(allowed, dtype=torch.float64, device=err.device)
    return float((err / allowed.clamp_min(TINY)).max()) if err.numel() else 0.0


def _pad_ratio(dev, valid_rows):
    """inf when a pad row is not exactly zero."""
    return float("inf") if bool((dev[~valid_rows] != 0).any()) else 0.0


def fp16_ulp(v):
    """Spacing of fp16 at each value of v, after rounding |v| to fp16 (numpy's np.spacing on float16 = IEEE binary16)."""
    a = v.abs().to(torch.float16).double()
    _, ex = torch.frexp(a)
    return torch.where(a < 2.0 ** -14, torch.full_like(a, 2.0 ** -24), torch.ldexp(torch.ones_like(a), ex - 11))


def bar_kvt(dev, ref, absprod, L: Layout):
    """One fp16 ulp of fp16(64 ref) / 64 plus the two-pass GEMM term 2^-11 sum|x||w| (elu' <= 1); pad rows exactly 0."""
    v = L.valid_mask(dev.device)
    allowed = fp16_ulp(64.0 * ref[v]) / 64.0 + 2.0 ** -11 * absprod[v]
    return max(_ratio((dev[v] - ref[v]).abs(), allowed), _pad_ratio(dev, v))


def bar_per_segment(dev, ref, rel=1e-5):
    """<= rel x the segment's max |ref| ([S, ...] tensors)."""
    S = ref.shape[0]
    scale = ref.reshape(S, -1).abs().amax(1)
    return _ratio((dev - ref).reshape(S, -1).abs().amax(1), rel * scale)


def bar_bd(dev, ref, absbd=None, L: Layout | None = None, cross=False):
    """bd: per segment 1e-5 of its max, plus (absbd given) the state kernel's fp32 accumulation, absbd = sum |k||v| / n:
      * the one-plane fp16 products of the source segment's padded rows enter the tensor cores' accumulator one k-block of 16
        rows at a time, each rounding (toward zero) by at most 2^-23 of the running sum <= sum |k||v|: n_pad_src / 16 x 2^-23;
      * kv_state_reduce adds the row groups' partial states in fp32 (at most n_pad_src / 256 groups, one rounding of 2^-24 of a
        partial sum <= sum |k||v| each) and divides by n (one more rounding): (n_pad_src / 256 + 1) x 2^-24.
    Measured on an H100 80GB HBM3 (400 W) against the 1e-5 term alone: 1.24 at 64 frames of N = 2048 (8-slab groups of 2048
    rows), 0.42 at the bench shape, <= 0.14 in the small stage cases; against the whole bar 0.48, 0.23 and <= 0.10.
    Off-diagonal blocks exactly 0."""
    off = torch.ones(D, D, dtype=torch.bool, device=dev.device)
    for h in range(H):
        off[h * DH:(h + 1) * DH, h * DH:(h + 1) * DH] = False
    zero = float("inf") if bool((dev[:, off] != 0).any()) else 0.0
    if absbd is None:
        return max(bar_per_segment(dev, ref), zero)
    S = ref.shape[0]
    n_pad = torch.tensor([L.seg_padded(L.src_seg(s, cross)) for s in range(S)], dtype=torch.float64, device=dev.device)
    acc = n_pad / 16 * 2.0 ** -23 + (n_pad / 256 + 1) * 2.0 ** -24
    allowed = 1e-5 * ref.reshape(S, -1).abs().amax(1)[:, None, None] + acc[:, None, None] * absbd
    return max(_ratio((dev - ref).abs(), allowed), zero)


def bar_rows(dev, ref, rows_mask, rel=1e-5):
    """<= rel x the row's max |ref| on the rows selected."""
    d, r = dev[rows_mask], ref[rows_mask]
    return _ratio((d - r).abs().amax(1), rel * r.abs().amax(1))


def valid_segments(L: Layout, device="cpu"):
    return torch.tensor([L.seg_valid(s) > 0 for s in range(L.S)], device=device)


def bar_mu(dev, ref_mu, ref_rstd, L: Layout):
    """|dmu| <= 1e-6 (|mu| + sigma) on the segments with rows."""
    v = valid_segments(L, dev.device)
    sigma = torch.sqrt((1.0 / ref_rstd[v] ** 2 - 1e-5).clamp_min(0))
    return _ratio((dev[v] - ref_mu[v]).abs(), 1e-6 * (ref_mu[v].abs() + sigma))


def bar_rstd(dev, ref, L: Layout):
    v = valid_segments(L, dev.device)
    return _ratio((dev[v] - ref[v]).abs(), 1e-5 * ref[v].abs())


SPLIT_FLOOR = 2.0 ** -30   # absolute resolution of the fp16-split format: the lo plane's subnormal spacing 2^-24, / 64


def bar_x_out(dev, ref, delta, L: Layout):
    """X after mlp.3: 1e-5 max|layer delta| of the segment, plus the residual's own rounding: it passes through the tensor
    cores' fp32 accumulator as the identity K-block (2^-18.7 |x| measured on an H100 where the layer delta is exactly 0) and is
    split again (|x| < ~2e-3 has a subnormal lo plane, resolution 2^-30): 2^-18 |x| + 16 x 2^-30.  Pad rows exactly 0."""
    v = L.valid_mask(dev.device)
    seg = L.seg_index(dev.device)
    dmax = torch.zeros(L.S, dtype=torch.float64, device=dev.device)
    for s in range(L.S):
        r = delta[L.seg_rows(s)]
        if r.shape[0]:
            dmax[s] = r.abs().max()
    allowed = 1e-5 * dmax[seg][:, None] + 2.0 ** -18 * ref.abs() + 16 * SPLIT_FLOOR
    return max(_ratio((dev - ref).abs()[v], allowed[v]), _pad_ratio(dev, v))


def bar_gats(dev, ref, L: Layout):
    """X after a GATs layer: 1e-5 of the row's max on the 3D rows; every pad row exactly 0."""
    v = L.valid_mask(dev.device)
    three_d = torch.zeros(L.rows, dtype=torch.bool, device=dev.device)
    for b in range(L.B):
        three_d[L.seg_rows(2 * b + 1)] = True
    return max(bar_rows(dev, ref, three_d), _pad_ratio(dev, v))


def bar_pn(dev, ref, L: Layout):
    """Unit rows to 1e-6, and each element within 1e-5 of the fp64 normalized row."""
    v = L.valid_mask(dev.device)
    norm = _ratio((dev[v].norm(dim=1) - 1.0).abs(), torch.full((int(v.sum()),), 1e-6))
    return max(norm, _ratio((dev[v] - ref[v]).abs(), torch.full_like(ref[v], 1e-5)))


COS_ERR = 48 * 2.0 ** -23   # the score GEMM's cos: the fp32 accumulator of the 3-pass K = 256 product rounds once per k-block of 16


def bar_inverse_sums(dev, ref, scale):
    """1e-5 relative, plus the score GEMM's cos error amplified by 1/scale: e = exp((cos - 1) / scale) moves by dcos / scale
    relative, and the fp32 accumulator of the 3-pass K = 256 product rounds (toward zero, with the same sign) once per k-block of
    16: |dcos| <= 48 x 2^-23.  Entries past the valid counts exactly 0 (the reference holds 0 there)."""
    z = ref == 0
    rel = 1e-5 + COS_ERR / scale
    return max(_ratio((dev[~z] - ref[~z]).abs(), rel * ref[~z].abs()), float("inf") if bool((dev[z] != 0).any()) else 0.0)


def conf_rel_bar(cos, scale):
    """Relative bar of each conf entry against (e . irs)(e . ics) in fp64 with the device's own irs, ics, cos from the device's pn,
    e = exp((cos - 1) / scale).  The epilogue computes e = ex2(fma(acc, ea, eb)) once and forms (e . irs)(e . ics):
      * cos: the score GEMM's error |dcos| <= 48 x 2^-23 (bar_inverse_sums) moves e by dcos / scale, e^2 by 2 dcos / scale;
      * the fp32 argument t = log2(e) (cos - 1) / scale, |t| <= 2 log2(e) / scale: the fma rounds once (2^-24 |t|); the factors
        ea and eb share fp32(1 / scale) and fp32(log2 e) (2 x 2^-24 |t|); scale itself is fp32 on the device (2^-24 |t|); ea and
        eb are each rounded once more (2^-24 log2(e) / scale each).  e moves by ln 2 |dt|, e^2 by twice that;
      * ex2.approx: 2^-22 relative, twice for e^2;
      * the three fp32 products: 2^-24 each."""
    log2e = 1.4426950408889634
    t = log2e * (1.0 - cos) / scale
    dt = 4 * 2.0 ** -24 * t + 2 * 2.0 ** -24 * log2e / scale
    return 2 * COS_ERR / scale + 2 * np.log(2.0) * dt + 2 * 2.0 ** -22 + 3 * 2.0 ** -24


CONF_ABS = 2.0 ** -148      # below fp32's normal range each of the three products rounds to 2^-150 absolute (factors <= 1)


def bar_conf(dev, cos, irs, ics, scale):
    """One frame's conf [N_b, M_b] (fp32) against (e . irs)(e . ics) entry by entry (conf_rel_bar, plus CONF_ABS: at scales below
    ~0.05 the smallest entries fall below 2^-126, where fp32 keeps an absolute, not a relative, precision); inf when an entry is
    not finite."""
    if not bool(torch.isfinite(dev).all()):
        return float("inf")
    ref = conf_entries(torch.exp((cos - 1.0) / scale), irs, ics)
    return _ratio((dev.double() - ref).abs(), conf_rel_bar(cos, scale) * ref + CONF_ABS)


def first_max_mismatches(idx, val, conf, dim):
    """Unpacked arg-maxes (idx, value) that are not the first maximum of the device's own conf along `dim`, or whose value bits
    differ from that entry."""
    am = conf.argmax(dim)
    at = conf.gather(dim, am.unsqueeze(dim)).squeeze(dim)
    return int(((idx != am) | (val.float() != at)).sum())


def mutual_mismatches(m0, m1, s0, s1, conf, thr, defect=NO_DEFECT):
    """Entries of the device's matches0 / matches1 / matching_scores0 / matching_scores1 [N_b], [M_b] that differ, bit for bit,
    from `mutual` applied to the device's own conf (fp32)."""
    r0, r1, rs0, rs1 = mutual(conf, thr, defect)
    return int((m0 != r0).sum() + (m1 != r1).sum() + (s0 != rs0).sum() + (s1 != rs1).sum())


def unpack_best(packed):
    """(conf bits << 32) | ~index -> (index, value), on the device of `packed`."""
    idx = 0xFFFFFFFF - (packed & 0xFFFFFFFF)
    val = (packed >> 32).to(torch.int32).view(torch.float32)
    return idx, val.double()


def decided_gap(scale):
    """Relative top-1 / top-2 gap above which an arg-max is decided: 1e-5 at scale >= 0.07, growing as 0.07 / scale below it
    (the cos error enters conf amplified by 1 / scale)."""
    return 1e-5 * max(1.0, 0.07 / scale)


def argmax_mismatches(dev_idx, conf, dim, gap=1e-5):
    """Arg-maxes of conf along `dim` that differ from dev_idx where the fp64 top-1 / top-2 gap exceeds `gap` relative."""
    if conf.shape[dim] < 2:
        decided = torch.ones(conf.shape[1 - dim], dtype=torch.bool, device=conf.device)
    else:
        top2 = conf.topk(2, dim=dim).values
        t0, t1 = (top2[:, 0], top2[:, 1]) if dim == 1 else (top2[0], top2[1])
        decided = (t0 - t1) > gap * t0
    return int(((dev_idx != conf.argmax(dim)) & decided).sum())
