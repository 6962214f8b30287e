"""fp64 references and per-entry bars of the wgmma GEMM core's fused epilogues (csrc/gemm_tc.cu), and an emulation of its
arithmetic.

The core multiplies fp16-split operands, x = (hi + lo) / 64 (common.cuh), in three tensor-core passes into one fp32
accumulator, D += A_hi B_hi + A_hi B_lo + A_lo B_hi, one m64nNk16 MMA per pass and k-step of 16.  Against the exact product of
the values the planes hold, sum_k a_k b_k, an entry moves by at most
  * the dropped A_lo B_lo term: 2^-22 sum_k |a_k| |b_k|  (|lo| <= 2^-11 |hi|);
  * the accumulator: every MMA adds into it and rounds (truncates) once, by at most one fp32 ulp of a running sum that never
    exceeds S = sum_k |a_k| |b_k|: passes x K / 16 x 2^-23 S.
product_bar is that sum; each epilogue adds its own roundings (the fp32 bias add, the output split, ex2.approx, the converter's
FFMA).  ``emulate_product`` restates the accumulation bit for bit in numpy (exact fp16 products, one fp32 rounding per MMA,
round-to-nearest or truncation), so tests/test_gemm_core_reference_cpu.py can show that the bars hold for the emulated
arithmetic and that planted defects exceed them by far.  Every function allocates on the device of its inputs."""
from __future__ import annotations

import numpy as np
import torch

from tests import matcher_stage_reference as ref

SPLIT_FLOOR = ref.SPLIT_FLOOR
F32_OUT = 2.0 ** -23          # the epilogue's fp32 bias add and output: one rounding of the entry (2^-24), with margin
LOG2E = 1.4426950408889634


def plane_value(hi, lo):
    """The value a pair of fp16-split planes holds, fp64."""
    return (hi.double() + lo.double()) / 64.0


def ratio(err, allowed):
    """max(err / allowed); 0 for an empty selection."""
    return ref._ratio(err, allowed)


def product(pairs):
    """sum over (a [rows, k], b [n, k]) of a b^T in fp64, and S = sum |a| |b|^T (the bar's scale)."""
    r = sum(a @ b.T for a, b in pairs)
    S = sum(a.abs() @ b.abs().T for a, b in pairs)
    return r, S


def product_bar(S, K, passes):
    """Per-entry bar of a `passes`-pass split product over K reduction columns (see the module docstring)."""
    return (2.0 ** -22 + passes * ((K + 15) // 16) * 2.0 ** -23) * S


def planes_bar(r):
    """An fp32 epilogue value written as split planes: fma(acc, 2^-6, 64 bias) rounds once (2^-24), the lo plane rounds at
    2^-22 relative or the lo plane's subnormal spacing."""
    return (2.0 ** -22 + 2.0 ** -23) * r.abs() + 2 * SPLIT_FLOOR


def elu1_bar(y, r, ncols):
    """elu1 on the first ncols columns through ex2.approx (2^-22 relative) of the fp32 argument y log2(e) (rounded once: ln 2 x
    2^-24 |y log2 e| relative = 2^-24 |y|)."""
    out = torch.zeros_like(r)
    out[:, :ncols] = (2.0 ** -21 + 2.0 ** -23 * y[:, :ncols].abs()) * r[:, :ncols].abs()
    return out


def qscale_reference(y, dy, kmean, L: ref.Layout, cross):
    """Q' per head from y = acc + bias [rows, 256] (fp64) with the source segment's Kmean, and its per-entry bar from dy (the
    product's bar).  Q_i = u_i / den, u = elu1(y), den = u . k + 1e-6 / m_src:
      |dQ_i| <= du_i / den + |Q_i| (sum_j k_j du_j + 64 x 2^-24 sum_j u_j k_j) / den, du = dy + elu1's own error,
    plus the fp32 products (4 x 2^-24) and the output split."""
    u = ref._elu1(y)
    du = dy + elu1_bar(y, u, 256)
    seg = L.seg_index(y.device)
    src = seg ^ 1 if cross else seg
    m_src = torch.tensor([max(L.seg_valid(int(s)), 1) for s in range(L.S)], dtype=torch.float64, device=y.device)[src]
    uh, duh, kh = u.view(-1, 4, 64), du.view(-1, 4, 64), kmean[src].view(-1, 4, 64)
    den = (uh * kh).sum(2) + 1e-6 / m_src[:, None]
    q = uh / den[:, :, None]
    dden = (kh * duh).sum(2) + 64 * 2.0 ** -24 * (uh * kh).sum(2)
    allowed = duh / den[:, :, None] + q.abs() * (dden / den)[:, :, None] + 4 * 2.0 ** -24 * q.abs()
    allowed = allowed.reshape(-1, 256) + planes_bar(q.reshape(-1, 256))
    return q.reshape(-1, 256), allowed


def mlp3_reference(hid, mu, rstd, x, w1, bias, L: ref.Layout):
    """x_out = [ReLU((h - mu_seg) rstd_seg) | x] . [W1 | I]^T + b, pad rows 0, and its bar.  The converter forms
    64 ReLU(...) as max(fma(h, 64 rstd, -(64 rstd) mu), 0) in fp32: -(64 rstd) mu rounds (2^-24 |mu| rstd), the FMA rounds
    (2^-24 of its result), the split of the result 2^-22; each moves the product by |W1| times that."""
    seg = L.seg_index(hid.device)
    m, s = mu[seg], rstd[seg]
    hn = torch.relu((hid - m) * s)
    eye = torch.eye(x.shape[1], dtype=torch.float64, device=x.device)
    r, S = product([(hn, w1), (x, eye)])
    r = r + bias
    conv = 2.0 ** -23 * m.abs() * s + (2.0 ** -22 + 2.0 ** -23) * hn + SPLIT_FLOOR
    allowed = product_bar(S, hid.shape[1] + x.shape[1], 3) + conv @ w1.abs().T + planes_bar(r)
    r[~L.valid_mask(hid.device)] = 0.0
    return r, allowed


def l2norm_reference(y, dy):
    """F.normalize(y) per row and its bar from dy (the entry's error before the norm): the entry's own error, the norm's (fp32
    sum of 256 squares in four chains: 64 x 2^-24 relative of the square sum, half that of the norm; sqrt, the reciprocal and
    the product: 3 x 2^-24), and the output split."""
    nrm = y.norm(dim=1, keepdim=True)
    out = y / nrm.clamp_min(1e-12)
    dn = (y.abs() * dy).sum(1, keepdim=True) / nrm.clamp_min(1e-300)
    allowed = dy / nrm + out.abs() * (dn / nrm + 40 * 2.0 ** -24) + planes_bar(out)
    return out, allowed


def quarter_stats(c, L: ref.Layout):
    """EPI_F32_STATS partials of every 32-row quarter and column of c [rows, n] (fp64 of the device's fp32 output) over the
    quarter's valid rows: (sum, sum of squared deviations from the quarter's mean), their bars, and the mask of quarters with no
    valid row [rows / 32, n].  Bars of the fp32 two-pass sums over <= 32 rows: sum 32 x 2^-24 sum|x|; deviations from an fp32
    mean off by delta <= 34 x 2^-24 max|x|: 40 x 2^-24 sum d^2 + n delta^2 + 2 delta |sum d|."""
    rows, n = c.shape
    v = L.valid_mask(c.device).view(rows // 32, 32, 1).double()
    cq = c.view(rows // 32, 32, n)
    cnt = v.sum(1)
    s = (cq * v).sum(1)
    mean = s / cnt.clamp_min(1)
    d = (cq - mean[:, None]) * v
    m2 = (d * d).sum(1)
    absum = (cq.abs() * v).sum(1)
    delta = 34 * 2.0 ** -24 * (cq.abs() * v).amax(1)
    s_bar = 32 * 2.0 ** -24 * absum + 1e-300
    m2_bar = 40 * 2.0 ** -24 * m2 + cnt * delta ** 2 + 2 * delta * d.sum(1).abs() + 1e-300
    empty = (cnt == 0).expand(-1, n)
    return s, m2, s_bar, m2_bar, empty


def score_partials(pv, L: ref.Layout, scale):
    """Pass 1 of the score tail from the plane values pv [rows, 256] (fp64): rowsum_part [B, 2 n_tiles, n_pad] (sums over
    128-column tile halves), colsum_part [B, 4 m_tiles, m_pad] (sums over 32-row groups) of e = exp((cos - 1) / scale) on the
    valid entries, 0 elsewhere; and cos [B, n_pad, m_pad]."""
    rs = torch.zeros(L.B, L.m_pad // 128, L.n_pad, dtype=torch.float64, device=pv.device)
    cs = torch.zeros(L.B, L.n_pad // 32, L.m_pad, dtype=torch.float64, device=pv.device)
    cos = torch.zeros(L.B, L.n_pad, L.m_pad, dtype=torch.float64, device=pv.device)
    for b in range(L.B):
        q, d = pv[L.seg_rows(2 * b, padded=True)], pv[L.seg_rows(2 * b + 1, padded=True)]
        cos[b] = q @ d.T
        e = torch.exp((cos[b] - 1.0) / scale)
        e[L.n_of(b):] = 0.0
        e[:, L.m_of(b):] = 0.0
        rs[b] = e.view(L.n_pad, L.m_pad // 128, 128).sum(2).T
        cs[b] = e.view(L.n_pad // 32, 32, L.m_pad).sum(1)
    return rs, cs, cos


# ------------------------------------------------------------------------------------------------ emulation of the core
def f32_round(v, trunc):
    """fp64 -> the nearest fp32 (trunc False) or the fp32 toward zero (trunc True), as fp64."""
    r = v.astype(np.float32)
    if trunc:
        over = np.abs(r.astype(np.float64)) > np.abs(v)
        r = np.where(over, np.nextafter(r, np.float32(0)), r)
    return r.astype(np.float64)


def split_planes(x):
    """numpy fp64 -> the fp16-split planes of common.cuh (as fp64 arrays of fp16 values), pre-scale included."""
    xs = (x * 64.0).astype(np.float32)
    hi = xs.astype(np.float16)
    lo = (xs - hi.astype(np.float32)).astype(np.float16)
    return hi.astype(np.float64), lo.astype(np.float64)


def emulate_product(blocks, trunc, passes=3, acc=None, hook=None):
    """The core's fp32 accumulator over k-blocks of 64 (numpy fp64 arrays of fp16 plane values, pre-scaled):
    blocks = [(a_hi, a_lo, b_hi, b_lo), ...] each [rows, 64] / [n, 64].  Per k-step of 16 the passes A_hi B_hi, A_hi B_lo
    (passes >= 2), A_lo B_hi (passes 3) each add their exact 16-term dot product and round once.  hook(kb, ks, terms) may
    replace a k-step's list of (a, b) pass operands (a planted defect).  Returns the accumulator (pre-scaled by 2^12)."""
    rows, n = blocks[0][0].shape[0], blocks[0][2].shape[0]
    acc = np.zeros((rows, n)) if acc is None else acc
    for kb, (ah, al, bh, bl) in enumerate(blocks):
        for ks in range(ah.shape[1] // 16):
            k = slice(16 * ks, 16 * ks + 16)
            terms = [(ah[:, k], bh[:, k]), (ah[:, k], bl[:, k]), (al[:, k], bh[:, k])][:passes]
            if hook is not None:
                terms = hook(kb, ks, terms, k)
            for a, b in terms:
                acc = f32_round(acc + a @ b.T, trunc)
    return acc
