"""The GEMM core's bars have teeth (no GPU): tests/gemm_core_reference.py's emulation of the core's arithmetic -- exact fp16
products, one fp32 rounding per k16 MMA, to nearest or toward zero -- meets every per-entry bar that tests/test_gemm_core_gpu.py
holds the device to, and each planted defect exceeds its bar by at least 10x.

The operands have one-signed lo planes (every fp16 residual positive), so that a dropped correction pass adds up instead of
averaging out, and the clean truncating accumulator errs in one direction: the worst case the bars are written for."""
from __future__ import annotations

import numpy as np
import pytest
import torch

from tests import gemm_core_reference as gr
from tests import matcher_stage_reference as ref

TEETH = 10.0
GARBAGE = 7.0


def one_signed_planes(rs, rows, cols, lo=0.5, hi=2.0):
    """Positive values as fp16-split planes (x 64) whose lo plane is positive: hi = fp16(64 u), lo = fp16(v ulp(hi) / 2)."""
    h = (64.0 * rs.uniform(lo, hi, (rows, cols))).astype(np.float16)
    l_ = (rs.uniform(0.05, 1.0, (rows, cols)) * np.spacing(h).astype(np.float64) / 2).astype(np.float16)
    return h.astype(np.float64), l_.astype(np.float64)


def blocks_of(ah, al, bh, bl):
    return [(ah[:, k:k + 64], al[:, k:k + 64], bh[:, k:k + 64], bl[:, k:k + 64]) for k in range(0, ah.shape[1], 64)]


def T(x):
    return torch.from_numpy(np.ascontiguousarray(x))


def f32_fma(a, b, c):
    return gr.f32_round(a * b + c, False)


def split_value(v_scaled):
    """Split planes of an fp32 value that is already x 64, as the value they hold."""
    hi = v_scaled.astype(np.float32).astype(np.float16).astype(np.float64)
    lo = (v_scaled - hi).astype(np.float32).astype(np.float16).astype(np.float64)
    return (hi + lo) / 64.0


@pytest.fixture(scope="module")
def prod():
    rs = np.random.RandomState(0)
    rows, n, K = 64, 64, 128
    ah, al = one_signed_planes(rs, rows, K)
    bh, bl = one_signed_planes(rs, n, K, 0.25, 1.0)
    a, b = (ah + al) / 64.0, (bh + bl) / 64.0
    r, S = gr.product([(T(a), T(b))])
    bias = rs.randn(n)
    return dict(ah=ah, al=al, bh=bh, bl=bl, r=r, S=S, K=K, bias=bias)


@pytest.mark.parametrize("trunc", [False, True])
def test_clean_product_meets_bar(prod, trunc):
    """The 3-pass product and the fp32 output with bias, rounded to nearest and truncated: within the bars."""
    acc = gr.emulate_product(blocks_of(prod["ah"], prod["al"], prod["bh"], prod["bl"]), trunc)
    out = acc / 4096.0
    rb = prod["r"] + T(prod["bias"])
    outb = gr.f32_round(out + prod["bias"], False)
    p = gr.ratio((T(out) - prod["r"]).abs(), gr.product_bar(prod["S"], prod["K"], 3))
    pb = gr.ratio((T(outb) - rb).abs(), gr.product_bar(prod["S"], prod["K"], 3) + gr.F32_OUT * rb.abs())
    print(f"clean product ({'truncated' if trunc else 'nearest'}): {p:.3f}, with bias {pb:.3f}")
    assert p <= 1.0 and pb <= 1.0


def _defect_ratio(prod, acc, bias_shift=False):
    bias = np.roll(prod["bias"], -1) if bias_shift else prod["bias"]
    out = gr.f32_round(acc / 4096.0 + bias, False)
    rb = prod["r"] + T(prod["bias"])
    return gr.ratio((T(out) - rb).abs(), gr.product_bar(prod["S"], prod["K"], 3) + gr.F32_OUT * rb.abs())


def test_dropped_lo_pass_is_caught(prod):
    """One k-block's A_lo B_hi pass dropped."""
    drop = lambda kb, ks, terms, k: terms[:2] if kb == 1 else terms   # noqa: E731
    acc = gr.emulate_product(blocks_of(prod["ah"], prod["al"], prod["bh"], prod["bl"]), True, hook=drop)
    r = _defect_ratio(prod, acc)
    print(f"A_lo B_hi of k-block 1 dropped: {r:.1f} x the bar")
    assert r >= TEETH


def test_swapped_k_steps_are_caught(prod):
    """Two k-steps of one k-block swapped in B only."""
    bh, bl = prod["bh"].copy(), prod["bl"].copy()
    for m in (bh, bl):
        m[:, 0:16], m[:, 16:32] = m[:, 16:32].copy(), m[:, 0:16].copy()
    acc = gr.emulate_product(blocks_of(prod["ah"], prod["al"], bh, bl), True)
    r = _defect_ratio(prod, acc)
    print(f"k-steps 0 and 1 of B swapped: {r:.1f} x the bar")
    assert r >= TEETH


def test_neighbour_bias_is_caught(prod):
    """The bias of column c + 1 added to column c."""
    acc = gr.emulate_product(blocks_of(prod["ah"], prod["al"], prod["bh"], prod["bl"]), True)
    r = _defect_ratio(prod, acc, bias_shift=True)
    print(f"bias from column c + 1: {r:.1f} x the bar")
    assert r >= TEETH


# ------------------------------------------------------------------------------------------------ converter + identity (mlp.3)
MLP3_L = ref.Layout(1, 32, 32, 32, 32)       # two 32-row segments, every row valid


def _mlp3(trunc, lose_identity_lo=False, wrong_seg=False):
    rs = np.random.RandomState(1)
    L = MLP3_L
    K1, n = 128, 256
    seg = L.seg_index().numpy()
    mu = np.stack([rs.randn(512) * 20 + 80, rs.randn(512) * 20 - 160]).astype(np.float32).astype(np.float64)
    rstd = (1.0 / (0.5 + rs.rand(2, 512))).astype(np.float32).astype(np.float64)
    hid = (mu[seg][:, :K1] + rs.randn(L.rows, K1) / rstd[seg][:, :K1]).astype(np.float32).astype(np.float64)
    x = rs.randn(L.rows, n) * 4
    xh, xl = gr.split_planes(x)
    wh, wl = gr.split_planes(rs.randn(n, K1) * 0.02)
    bias = rs.randn(n).astype(np.float32).astype(np.float64)
    # the converter: 64 ReLU((h - mu) rstd) = max(fma(h, 64 rstd, -(64 rstd) mu), 0) in fp32, split in place
    sseg = seg.copy()
    if wrong_seg:
        sseg[32:] = 0                                                   # the second tile with the first segment's statistics
    pb = gr.f32_round(64.0 * rstd[sseg][:, :K1], False)
    pa = gr.f32_round(-mu[sseg][:, :K1] * pb, False)
    v = np.maximum(f32_fma(hid, pb, pa), 0.0)
    ah = v.astype(np.float32).astype(np.float16).astype(np.float64)
    al = (v - ah).astype(np.float32).astype(np.float16).astype(np.float64)
    eye_h, eye_l = 64.0 * np.eye(n), np.zeros((n, n))
    blocks = blocks_of(ah, al, wh, wl) + blocks_of(xh, xl, eye_h, eye_l)
    nkb1 = K1 // 64

    def identity_passes(kb, ks, terms, k):
        if kb < nkb1:
            return terms
        return [terms[0]] if lose_identity_lo else [terms[0], terms[2]]   # zero lo plane of I: A_hi I_hi + A_lo I_hi

    acc = gr.emulate_product(blocks, trunc, hook=identity_passes)
    out = split_value(f32_fma(acc, 1.0 / 64.0, bias * 64.0))
    r, allowed = gr.mlp3_reference(T(hid), T(mu[:, :K1]), T(rstd[:, :K1]), T((xh + xl) / 64.0), T((wh + wl) / 64.0), T(bias), L)
    return gr.ratio((T(out) - r).abs(), allowed)


@pytest.mark.parametrize("trunc", [False, True])
def test_clean_converter_meets_bar(trunc):
    r = _mlp3(trunc)
    print(f"clean converter + identity ({'truncated' if trunc else 'nearest'}): {r:.3f}")
    assert r <= 1.0


def test_lost_identity_lo_is_caught():
    """The identity block's A_lo pass lost (the residual keeps its hi plane only)."""
    r = _mlp3(True, lose_identity_lo=True)
    print(f"identity block without its lo plane: {r:.1f} x the bar")
    assert r >= TEETH


def test_neighbour_segment_statistics_are_caught():
    """One row tile converted with the neighbouring segment's mu / rstd."""
    r = _mlp3(True, wrong_seg=True)
    print(f"neighbour segment's mu / rstd for one tile: {r:.1f} x the bar")
    assert r >= TEETH


# ------------------------------------------------------------------------------------------------ InstanceNorm partials
STATS_L = ref.Layout(1, 40, 64, 64, 64)     # query segment: 40 of 64 rows valid (quarter 1 holds 8, the next 2 none)


def _stats(extra_pad_row=False):
    rs = np.random.RandomState(2)
    L = STATS_L
    n = 64
    c = (rs.randn(L.rows, n) * 0.5 + 30.0).astype(np.float32).astype(np.float64)   # large means against the spread
    c[~L.valid_mask().numpy()] = GARBAGE
    nv = L.valid_mask().numpy().reshape(-1, 32).sum(1)
    if extra_pad_row:
        nv[1] += 1                                                  # quarter 1 counts its first pad row
    s = np.zeros((L.rows // 32, n))
    m2 = np.zeros_like(s)
    for qq in range(L.rows // 32):
        rows = c[32 * qq:32 * qq + nv[qq]]
        acc = np.zeros(n)
        for row in rows:
            acc = gr.f32_round(acc + row, False)
        mean = gr.f32_round(acc / nv[qq], False) if nv[qq] else np.zeros(n)
        dd = np.zeros(n)
        for row in rows:
            d = gr.f32_round(row - mean, False)
            dd = f32_fma(d, d, dd)
        s[qq], m2[qq] = acc, dd
    s_ref, m2_ref, s_bar, m2_bar, empty = gr.quarter_stats(T(c), L)
    zero = 0.0 if (s[empty.numpy()] == 0).all() and (m2[empty.numpy()] == 0).all() else float("inf")
    return max(gr.ratio((T(s) - s_ref).abs(), s_bar), gr.ratio((T(m2) - m2_ref).abs(), m2_bar), zero)


def test_clean_stats_meet_bar():
    r = _stats()
    print(f"clean quarter statistics: {r:.3f}")
    assert r <= 1.0


def test_pad_row_in_stats_is_caught():
    r = _stats(extra_pad_row=True)
    print(f"a pad row counted in one quarter: {r:.1f} x the bar")
    assert r >= TEETH


# ------------------------------------------------------------------------------------------------ k,v projection
def _qkv(trunc, elu_on_v_head=False):
    rs = np.random.RandomState(3)
    rows, n, K = 64, 512, 128
    xh, xl = gr.split_planes(rs.randn(rows, K))
    wh, wl = gr.split_planes(rs.randn(n, K) / np.sqrt(K))
    bias = (rs.randn(n) * 0.5).astype(np.float32).astype(np.float64)
    acc = gr.emulate_product(blocks_of(xh, xl, wh, wl), trunc)
    y = f32_fma(acc, 1.0 / 4096.0, bias)
    cols = 320 if elu_on_v_head else 256                        # V head 0 = columns [256, 320)
    yk = y[:, :cols]
    e = np.exp2(gr.f32_round(yk * gr.LOG2E, False)).astype(np.float32).astype(np.float64)
    y[:, :cols] = np.where(yk > 0, gr.f32_round(yk + 1.0, False), e)
    out = (y * 64.0).astype(np.float32).astype(np.float16).astype(np.float64) / 64.0
    r, S = gr.product([(T((xh + xl) / 64.0), T((wh + wl) / 64.0))])
    r = r + T(bias)
    yr = r.clone()
    r[:, :256] = ref._elu1(r[:, :256])
    allowed = ref.fp16_ulp(64.0 * r) / 64.0 + gr.product_bar(S, K, 3) + gr.elu1_bar(yr, r, 256)
    return gr.ratio((T(out) - r).abs(), allowed)


@pytest.mark.parametrize("trunc", [False, True])
def test_clean_qkv_meets_bar(trunc):
    r = _qkv(trunc)
    print(f"clean k,v projection ({'truncated' if trunc else 'nearest'}): {r:.3f}")
    assert r <= 1.0


def test_elu_on_a_v_head_is_caught():
    r = _qkv(True, elu_on_v_head=True)
    print(f"elu1 applied to V head 0: {r:.1f} x the bar")
    assert r >= TEETH
