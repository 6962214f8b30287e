"""The wgmma GEMM core (csrc/gemm_tc.cu) driven directly through opb_debug_gemm: every instantiation the library launches,
against an fp64 reference of its fused epilogue, entry by entry, and bit for bit across tile schedules.

The operands are fp16-split planes (opb_debug_split); every reference works on the values the planes hold, (hi + lo) / 64,
in fp64.  Per-entry bars come from the format (gemm_core_reference.product_bar and the epilogue's own roundings), never from a
matrix's largest entry.  Each case prints its error as a multiple of its bar (<= 1 passes).

Schedules: the core counts k-blocks across all tiles of a CTA, so the ring stage and barrier parity a tile starts on depend
on (tiles done x k-blocks per tile) mod (2 x stages).  Every problem runs with max_ctas in {1, 2, 3, 7, 131, 132} and the
default grid, with k-blocks per tile covering every residue of the ring depth, and the outputs must be bit-identical: a tile's
result does not depend on which CTA computes it.  Outputs are filled with 0xFF before each launch (an entry the kernel never
wrote shows), input rows the epilogue must mask hold finite garbage (7.0)."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest
import torch

from onepose_b200 import _lib
from tests import gemm_core_reference as gr
from tests import matcher_stage_reference as ref

pytestmark = pytest.mark.gpu

CTAS = (1, 2, 3, 7, 131, 132)
GARBAGE = 7.0
DEV = "cuda"


@pytest.fixture(scope="module")
def lib():
    return _lib.load()


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def split(lib, x):
    """fp32 [r, c] (cuda) -> (hi, lo, value): the device's split planes and the fp64 values they hold."""
    x = x.float().contiguous()
    hi, lo = torch.empty_like(x, dtype=torch.float16), torch.empty_like(x, dtype=torch.float16)
    assert lib.opb_debug_split(x.data_ptr(), hi.data_ptr(), lo.data_ptr(), x.numel(), None) == 0
    return hi, lo, gr.plane_value(hi, lo)


def _bytes(t):
    return t.contiguous().view(-1).view(torch.uint8)


def launch(lib, fields, outs, zero=(), **over):
    """One launch: every output filled with 0xFF first (those in `zero`, atomic targets, with 0); returns clones."""
    for k, t in outs.items():
        _bytes(t).fill_(0 if k in zero else 0xFF)
    d = _lib.gemm_desc(**{**fields, **outs, **over})
    rc = lib.opb_debug_gemm(d, None)
    assert rc == 0, (fields.get("epi"), rc)
    torch.cuda.synchronize()
    return {k: t.clone() for k, t in outs.items()}


def schedules(lib, name, fields, outs, zero=()):
    """Default grid twice (repeat), then every max_ctas: all bit-identical.  Returns the default run's outputs."""
    base = launch(lib, fields, outs, zero)
    again = launch(lib, fields, outs, zero)
    for k in outs:
        assert torch.equal(_bytes(base[k]), _bytes(again[k])), f"{name}: {k} differs between two identical calls"
    for ctas in CTAS:
        got = launch(lib, fields, outs, zero, max_ctas=ctas)
        for k in outs:
            assert torch.equal(_bytes(base[k]), _bytes(got[k])), f"{name}: {k} differs with max_ctas = {ctas}"
    return base


def report(name, **ratios):
    print(f"{name}: " + "  ".join(f"{k} {v:.3f}" for k, v in ratios.items()))
    for k, v in ratios.items():
        assert v <= 1.0, f"{name}: {k} = {v:.3f} x its bar"


def layout_fields(L: ref.Layout):
    f = dict(B=L.B, N=L.N, M=L.M, n_pad=L.n_pad, m_pad=L.m_pad)
    keep = []
    if L.nlen is not None:
        t = torch.tensor(L.nlen, dtype=torch.int32, device=DEV)
        keep.append(t)
        f["nlen"] = t
    if L.mlen is not None:
        t = torch.tensor(L.mlen, dtype=torch.int32, device=DEV)
        keep.append(t)
        f["mlen"] = t
    return f, keep


def masked_rows(x, L: ref.Layout):
    """x with GARBAGE in every row past its segment's valid count."""
    x = x.clone()
    x[~L.valid_mask(x.device)] = GARBAGE
    return x


def rand(g, r, c, scale=1.0):
    return torch.randn(r, c, device=DEV, generator=g) * scale


# ------------------------------------------------------------------------------------------------ EPI_F32
# (K1, K2) pairs: k-blocks per tile 1, 7, 4, 7, 6, 8 -> every residue mod 4 (two-stage ring at 256-wide tiles)
F32_256_K = [(64, 0), (448, 0), (192, 64), (320, 128), (128, 256), (256, 256)]
# 128-wide tiles (three-stage ring, no K2 block): 1, 2, 3, 7 k-blocks
F32_128_K = [(64, 0), (128, 0), (192, 0), (448, 0)]


@pytest.mark.parametrize("bn,K1,K2", [(256, k1, k2) for k1, k2 in F32_256_K] + [(128, k1, k2) for k1, k2 in F32_128_K])
def test_f32_product_bias_windows(lib, bn, K1, K2):
    """C = A . B^T + bias with ld > K operand windows and ldc > n_out: every entry within the format's bar, the columns past
    n_out never written."""
    g = _gen(K1 * 7 + K2 + bn)
    rows, n_out = 512, 512 if bn == 256 else 384
    lda1, lda2, ldb1, ldb2, ldc = K1 + 64, K2 + 8, K1 + 8, K2 + 64, n_out + 4
    a1 = split(lib, rand(g, rows, lda1) * torch.exp(rand(g, rows, 1)))
    b1 = split(lib, rand(g, n_out, ldb1, K1 ** -0.5))
    a2 = split(lib, rand(g, rows, max(lda2, 8))) if K2 else None
    b2 = split(lib, rand(g, n_out, max(ldb2, 8), 0.1)) if K2 else None
    bias = rand(g, 1, n_out)[0]
    f = dict(epi=_lib.EPI_F32, bn=0 if bn == 256 else bn, rows=rows, n_out=n_out, K1=K1, K2=K2, a1_hi=a1[0], a1_lo=a1[1],
             a1_ld=lda1, b1_hi=b1[0], b1_lo=b1[1], b1_ld=ldb1, bias=bias, ldc=ldc)
    if K2:
        f.update(a2_hi=a2[0], a2_lo=a2[1], a2_ld=lda2, b2_hi=b2[0], b2_lo=b2[1], b2_ld=ldb2)
    c = torch.empty(rows, ldc, device=DEV)
    out = schedules(lib, f"f32 bn{bn} K1={K1} K2={K2}", f, {"c": c})["c"]
    A = [(a1[2][:, :K1], b1[2][:, :K1])] + ([(a2[2][:, :K2], b2[2][:, :K2])] if K2 else [])
    r, S = gr.product(A)
    r = r + bias.double()
    allowed = gr.product_bar(S, K1 + K2, 3) + gr.F32_OUT * r.abs()
    report(f"f32 bn{bn} K1={K1} K2={K2}", product=gr.ratio((out[:, :n_out].double() - r).abs(), allowed),
           untouched=0.0 if bool((_bytes(out[:, n_out:]) == 0xFF).all()) else float("inf"))


def test_f32_matches_simt_cross_check(lib):
    """The SIMT fp32 backend on the same descriptor: within the same per-entry bar of the fp64 product."""
    g = _gen(3)
    rows, n_out, K = 256, 256, 192
    a, b = split(lib, rand(g, rows, K)), split(lib, rand(g, n_out, K, K ** -0.5))
    f = dict(epi=_lib.EPI_F32, rows=rows, n_out=n_out, K1=K, a1_hi=a[0], a1_lo=a[1], a1_ld=K, b1_hi=b[0], b1_lo=b[1], b1_ld=K,
             ldc=n_out)
    r, S = gr.product([(a[2], b[2])])
    outs = [launch(lib, f, {"c": torch.empty(rows, n_out, device=DEV)}, backend=be)["c"] for be in (0, 1)]
    # the SIMT kernel joins the planes in fp32 and rounds (to nearest) once per FFMA: K x 2^-24 S
    report("f32 wgmma / simt", wgmma=gr.ratio((outs[0].double() - r).abs(), gr.product_bar(S, K, 3)),
           simt=gr.ratio((outs[1].double() - r).abs(), gr.product_bar(S, K, 3) + K * 2.0 ** -24 * S))


def test_gemm_cores_agree_and_match_fp64(lib):
    """wgmma 3-pass fp16-split GEMM vs the SIMT fp32 cross-check vs numpy fp64, same split operands."""
    rs = np.random.RandomState(0)
    for rows, n_out, K in [(256, 256, 64), (256, 256, 256), (512, 768, 256), (256, 512, 512), (1024, 7168, 256)]:
        a = torch.from_numpy((rs.randn(rows, K) * np.exp(rs.randn(rows, 1))).astype(np.float32)).cuda()
        b = torch.from_numpy((rs.randn(n_out, K) / np.sqrt(K)).astype(np.float32)).cuda()
        planes = [torch.empty_like(a, dtype=torch.float16) for _ in range(2)] + [torch.empty_like(b, dtype=torch.float16) for _ in range(2)]
        assert lib.opb_debug_split(a.data_ptr(), planes[0].data_ptr(), planes[1].data_ptr(), a.numel(), None) == 0
        assert lib.opb_debug_split(b.data_ptr(), planes[2].data_ptr(), planes[3].data_ptr(), b.numel(), None) == 0
        outs = []
        for backend in (0, 1):
            c = torch.zeros(rows, n_out, dtype=torch.float32, device="cuda")
            desc = _lib.gemm_desc(epi=_lib.EPI_F32, rows=rows, n_out=n_out, K1=K, a1_hi=planes[0], a1_lo=planes[1], a1_ld=K,
                                  b1_hi=planes[2], b1_lo=planes[3], b1_ld=K, c=c, ldc=n_out, backend=backend)
            rc = lib.opb_debug_gemm(desc, None)
            assert rc == 0, (backend, rc)
            torch.cuda.synchronize()
            outs.append(c.cpu().double())
        ah = (planes[0].cpu().double() + planes[1].cpu().double()) / 64.0
        bh = (planes[2].cpu().double() + planes[3].cpu().double()) / 64.0
        exact = ah @ bh.T
        scale = float(exact.abs().max())
        e_tc = float((outs[0] - exact).abs().max()) / scale
        e_simt = float((outs[1] - exact).abs().max()) / scale
        print(f"gemm {rows}x{n_out}x{K}: rel err wgmma {e_tc:.2e}, simt {e_simt:.2e}")
        # the tensor core truncates (does not round) its fp32 accumulator: ~2^-25 relative per accumulation step
        assert e_simt < 2e-6 and e_tc < 2e-6 + 1.2e-8 * K
        # the split itself represents fp32 to ~2^-22
        assert float((ah.float() - a.cpu()).abs().max() / a.abs().max()) < 2.0 ** -21


@pytest.mark.parametrize("units", [2, 132, 134, 1024])
def test_unit_counts(lib, units):
    """Grids of 2, 132 (one per SM), 134 (uneven over 132) and 1024 tiles: bit-identical on every grid, within the bar."""
    g = _gen(units)
    rows, n_out = {2: (256, 256), 132: (8448, 512), 134: (17152, 256), 1024: (65536, 512)}[units]
    K1 = 64 if units == 1024 else 192
    assert (rows // 128) * (n_out // 256) == units
    a, b = split(lib, rand(g, rows, K1)), split(lib, rand(g, n_out, K1, K1 ** -0.5))
    f = dict(epi=_lib.EPI_F32, rows=rows, n_out=n_out, K1=K1, a1_hi=a[0], a1_lo=a[1], a1_ld=K1, b1_hi=b[0], b1_lo=b[1],
             b1_ld=K1, ldc=n_out)
    out = schedules(lib, f"f32 {units} units", f, {"c": torch.empty(rows, n_out, device=DEV)})["c"]
    r, S = gr.product([(a[2], b[2])])
    report(f"f32 {units} units", product=gr.ratio((out.double() - r).abs(), gr.product_bar(S, K1, 3)))


# ------------------------------------------------------------------------------------------------ EPI_F32_STATS (mlp.0)
STATS_L = ref.Layout(2, 40, 300, 256, 512, nlen=[40, 0], mlen=[300, 77])


@pytest.mark.parametrize("K1,K2", [(64, 256), (128, 256), (128, 64), (256, 256)])
def test_f32_stats(lib, K1, K2):
    """mlp.0: the product with a per-segment B2, and each 32-row quarter's (sum, sum of squared deviations from its mean) over
    its valid rows, from the device's own fp32 output.  A quarter without valid rows gives exact zeros."""
    L = STATS_L
    g = _gen(K1 + K2)
    n_out = 512
    lf, keep = layout_fields(L)
    x = split(lib, masked_rows(rand(g, L.rows, K1), L))
    w = split(lib, rand(g, n_out, K1, K1 ** -0.5))
    q = split(lib, masked_rows(rand(g, L.rows, K2).abs(), L))
    G = split(lib, rand(g, L.S * n_out, K2, K2 ** -0.5) + 3.0)         # offset: channel means large against their spread
    bias = rand(g, 1, n_out)[0]
    f = dict(epi=_lib.EPI_F32_STATS, rows=L.rows, n_out=n_out, K1=K1, K2=K2, a1_hi=x[0], a1_lo=x[1], a1_ld=K1, b1_hi=w[0],
             b1_lo=w[1], b1_ld=K1, a2_hi=q[0], a2_lo=q[1], a2_ld=K2, b2_hi=G[0], b2_lo=G[1], b2_ld=K2, b2_mode=1, bias=bias,
             ldc=n_out, **lf)
    outs = schedules(lib, f"stats K1={K1} K2={K2}", f, {"c": torch.empty(L.rows, n_out, device=DEV),
                                                         "statpart": torch.empty(L.rows // 32, n_out, 2, device=DEV)})
    seg = L.seg_index(DEV)
    Gs = G[2].view(L.S, n_out, K2)
    r = x[2] @ w[2].T + torch.einsum("rk,rnk->rn", q[2], Gs[seg]) + bias.double()
    S = x[2].abs() @ w[2].abs().T + torch.einsum("rk,rnk->rn", q[2].abs(), Gs[seg].abs())
    allowed = gr.product_bar(S, K1 + K2, 3) + gr.F32_OUT * r.abs()
    dev_c = outs["c"].double()
    s_ref, m2_ref, s_bar, m2_bar, empty = gr.quarter_stats(dev_c, L)
    sp = outs["statpart"].double()
    report(f"stats K1={K1} K2={K2}", product=gr.ratio((dev_c - r).abs(), allowed),
           sum=gr.ratio((sp[..., 0] - s_ref).abs(), s_bar), m2=gr.ratio((sp[..., 1] - m2_ref).abs(), m2_bar),
           empty_quarters=0.0 if bool((sp[empty] == 0).all()) else float("inf"))


# ------------------------------------------------------------------------------------------------ EPI_QKV (k,v projection)
QKV_L = ref.Layout(2, 200, 300, 256, 512, nlen=[200, 31], mlen=[300, 129])


@pytest.mark.parametrize("passes", [2, 3])
@pytest.mark.parametrize("K1", [64, 128, 192, 256])
def test_qkv(lib, K1, passes):
    """k,v projection: out.hi = fp16(64 [elu1(K) | V]) with elu1 on the first 256 columns only, pad rows exactly 0.  Two passes
    read A's hi plane only: the reference then takes A = hi / 64."""
    L = QKV_L
    g = _gen(K1 + passes)
    lf, keep = layout_fields(L)
    x = split(lib, masked_rows(rand(g, L.rows, K1), L))
    w = split(lib, rand(g, 512, K1, K1 ** -0.5))
    bias = rand(g, 1, 512)[0] * 0.5
    f = dict(epi=_lib.EPI_QKV, rows=L.rows, n_out=512, K1=K1, a1_hi=x[0], a1_lo=x[1], a1_ld=K1, b1_hi=w[0], b1_lo=w[1],
             b1_ld=K1, a_hi_only=1 if passes == 2 else 0, bias=bias, out_ld=512, **lf)
    out = schedules(lib, f"qkv {passes}-pass K1={K1}", f, {"out_hi": torch.empty(L.rows, 512, dtype=torch.float16, device=DEV)})
    dev = out["out_hi"].double() / 64.0
    a = x[0].double() / 64.0 if passes == 2 else x[2]
    r, S = gr.product([(a, w[2])])
    r = r + bias.double()
    y = r.clone()
    r[:, :256] = ref._elu1(r[:, :256])
    v = L.valid_mask(DEV)
    allowed = ref.fp16_ulp(64.0 * r) / 64.0 + gr.product_bar(S, K1, passes) + gr.elu1_bar(y, r, 256)
    report(f"qkv {passes}-pass K1={K1}", kv=gr.ratio((dev - r).abs()[v], allowed[v]), pad_rows=ref._pad_ratio(dev, v))


# ------------------------------------------------------------------------------------------------ EPI_QSCALE (q projection)
QS_L = ref.Layout(2, 200, 300, 256, 512, nlen=[200, 0], mlen=[300, 77])


@pytest.mark.parametrize("cross", [0, 1])
@pytest.mark.parametrize("K1", [64, 128, 192, 256])
def test_qscale(lib, K1, cross):
    """Q' = elu1(q) / (elu1(q) . Kmean_src + 1e-6 / m_src) per head, with the source segment's Kmean (self / cross).  A segment
    whose source has no valid rows (frame 1 has no queries) gives Q' = 0."""
    L = QS_L
    g = _gen(K1 + 10 * cross)
    lf, keep = layout_fields(L)
    x = split(lib, masked_rows(rand(g, L.rows, K1), L))
    w = split(lib, rand(g, 256, K1, K1 ** -0.5))
    bias = rand(g, 1, 256)[0] * 0.5
    kmean = (0.5 + torch.rand(L.S, 256, device=DEV, generator=g)) / 64.0
    f = dict(epi=_lib.EPI_QSCALE, rows=L.rows, n_out=256, K1=K1, a1_hi=x[0], a1_lo=x[1], a1_ld=K1, b1_hi=w[0], b1_lo=w[1],
             b1_ld=K1, bias=bias, kmean=kmean, cross=cross, out_ld=256, **lf)
    outs = schedules(lib, f"qscale K1={K1} cross={cross}", f, {"out_hi": torch.empty(L.rows, 256, dtype=torch.float16, device=DEV),
                                                               "out_lo": torch.empty(L.rows, 256, dtype=torch.float16, device=DEV)})
    dev = gr.plane_value(outs["out_hi"], outs["out_lo"])
    r, S = gr.product([(x[2], w[2])])
    y = r + bias.double()
    rq, allowed = gr.qscale_reference(y, gr.product_bar(S, K1, 3), kmean.double(), L, cross)
    seg = L.seg_index(DEV)
    empty = torch.tensor([L.seg_valid(L.src_seg(s, cross)) == 0 for s in range(L.S)], device=DEV)[seg]
    report(f"qscale K1={K1} cross={cross}", q=gr.ratio((dev - rq).abs()[~empty], allowed[~empty]),
           no_source=0.0 if bool((dev[empty] == 0).all()) else float("inf"))


# ------------------------------------------------------------------------------------------------ EPI_BIAS_PLANES
@pytest.mark.parametrize("with_bias", [True, False])
@pytest.mark.parametrize("K1", [64, 128, 192, 256])
def test_bias_planes_batched(lib, K1, with_bias):
    """The G fold's form: batched over 4 segments, A shared (a_batch_rows = 0), B per batch; out planes = acc (+ bias)."""
    g = _gen(K1 + with_bias)
    batch, rows = 4, 512
    w = split(lib, rand(g, rows, K1))
    bd = split(lib, rand(g, batch * 256, K1, K1 ** -0.5))
    bias = rand(g, 1, 256)[0] if with_bias else None
    f = dict(epi=_lib.EPI_BIAS_PLANES, rows=rows, n_out=256, K1=K1, batch=batch, a_batch_rows=0, b_batch_rows=256, a1_hi=w[0],
             a1_lo=w[1], a1_ld=K1, b1_hi=bd[0], b1_lo=bd[1], b1_ld=K1, out_ld=256)
    if bias is not None:
        f["bias"] = bias
    name = f"bias planes batched K1={K1} bias={with_bias}"
    outs = schedules(lib, name, f, {"out_hi": torch.empty(batch * rows, 256, dtype=torch.float16, device=DEV),
                                    "out_lo": torch.empty(batch * rows, 256, dtype=torch.float16, device=DEV)})
    dev = gr.plane_value(outs["out_hi"], outs["out_lo"]).view(batch, rows, 256)
    B = bd[2].view(batch, 256, K1)
    r = torch.einsum("rk,znk->zrn", w[2], B) + (bias.double() if bias is not None else 0.0)
    S = torch.einsum("rk,znk->zrn", w[2].abs(), B.abs())
    report(name, planes=gr.ratio((dev - r).abs(), gr.product_bar(S, K1, 3) + gr.planes_bar(r)))


BP_L = ref.Layout(2, 100, 300, 256, 512, nlen=[100, 0], mlen=[300, 45])


@pytest.mark.parametrize("K1,K2", [(64, 0), (192, 0), (320, 0), (256, 64), (128, 128)])
def test_bias_planes_layout(lib, K1, K2):
    """The GATs W form (one batch over the activation layout): rows past their segment's valid count exactly 0; with a shared
    full B2 block."""
    L = BP_L
    g = _gen(K1 + K2 + 1)
    lf, keep = layout_fields(L)
    x = split(lib, masked_rows(rand(g, L.rows, K1), L))
    w = split(lib, rand(g, 256, K1, K1 ** -0.5))
    bias = rand(g, 1, 256)[0]
    f = dict(epi=_lib.EPI_BIAS_PLANES, rows=L.rows, n_out=256, K1=K1, K2=K2, a1_hi=x[0], a1_lo=x[1], a1_ld=K1, b1_hi=w[0],
             b1_lo=w[1], b1_ld=K1, bias=bias, out_ld=256, **lf)
    A = [(x[2], w[2])]
    if K2:
        x2 = split(lib, masked_rows(rand(g, L.rows, K2), L))
        w2 = split(lib, rand(g, 256, K2, K2 ** -0.5))
        f.update(a2_hi=x2[0], a2_lo=x2[1], a2_ld=K2, b2_hi=w2[0], b2_lo=w2[1], b2_ld=K2)
        A.append((x2[2], w2[2]))
    name = f"bias planes layout K1={K1} K2={K2}"
    outs = schedules(lib, name, f, {"out_hi": torch.empty(L.rows, 256, dtype=torch.float16, device=DEV),
                                    "out_lo": torch.empty(L.rows, 256, dtype=torch.float16, device=DEV)})
    dev = gr.plane_value(outs["out_hi"], outs["out_lo"])
    r, S = gr.product(A)
    r = r + bias.double()
    v = L.valid_mask(DEV)
    allowed = gr.product_bar(S, K1 + K2, 3) + gr.planes_bar(r)
    report(name, planes=gr.ratio((dev - r).abs()[v], allowed[v]), pad_rows=ref._pad_ratio(dev, v))


# ------------------------------------------------------------------------------------------------ converter (mlp.3)
CV_L = ref.Layout(2, 150, 300, 256, 512, nlen=[150, 0], mlen=[300, 201])


def _mlp3_problem(lib, K1, seed=0):
    L = CV_L
    g = _gen(K1 + seed)
    lf, keep = layout_fields(L)
    # per segment: channel means far from zero against their spread (|mu| rstd up to ~200), so the converter's
    # fma(h, 64 rstd, -64 mu rstd) rounding matters, and each segment its own statistics
    mu = (torch.randn(L.S, 512, device=DEV, generator=g) * 20.0 + 40.0 * torch.arange(1, L.S + 1, device=DEV)[:, None] *
          torch.tensor([1.0, -1.0], device=DEV).repeat(L.S // 2)[:, None])
    sigma = 0.5 + torch.rand(L.S, 512, device=DEV, generator=g)
    rstd = 1.0 / sigma
    seg = L.seg_index(DEV)
    hid = mu[seg][:, :K1] + sigma[seg][:, :K1] * rand(g, L.rows, K1)
    hid[~L.valid_mask(DEV)] = GARBAGE
    x = split(lib, masked_rows(rand(g, L.rows, 256), L))
    w1 = split(lib, rand(g, 256, K1, K1 ** -0.5))
    eye = split(lib, torch.eye(256, device=DEV))
    bias = rand(g, 1, 256)[0]
    f = dict(epi=_lib.EPI_BIAS_PLANES, rows=L.rows, n_out=256, K1=K1, K2=256, b1_hi=w1[0], b1_lo=w1[1], b1_ld=K1, a2_hi=x[0],
             a2_lo=x[1], a2_ld=256, b2_hi=eye[0], b2_lo=eye[1], b2_ld=256, a_raw=hid, a_raw_ld=K1, mu=mu, rstd=rstd, bias=bias,
             out_ld=256, **lf)
    return L, f, keep, (hid, mu, rstd, x, w1, bias)


@pytest.mark.parametrize("K1", [64, 128, 192, 256, 448])
def test_converter_zero_lo_identity_block(lib, K1):
    """mlp.3: [ReLU((h - mu_seg) rstd_seg) | x] . [W1 | I]^T + b with each segment's own statistics, rows past the valid count
    exactly 0; the identity as a zero-lo block, bit-identical under every tile schedule."""
    L, f, keep, (hid, mu, rstd, x, w1, bias) = _mlp3_problem(lib, K1)
    outs = schedules(lib, f"converter K1={K1}", {**f, "b2_mode": 2},
                     {"out_hi": torch.empty(L.rows, 256, dtype=torch.float16, device=DEV),
                      "out_lo": torch.empty(L.rows, 256, dtype=torch.float16, device=DEV)})
    dev = gr.plane_value(outs["out_hi"], outs["out_lo"])
    r, allowed = gr.mlp3_reference(hid.double(), mu.double()[:, :K1], rstd.double()[:, :K1], x[2], w1[2], bias.double(), L)
    v = L.valid_mask(DEV)
    report(f"converter K1={K1}", x_out=gr.ratio((dev - r).abs()[v], allowed[v]), pad_rows=ref._pad_ratio(dev, v))


# ------------------------------------------------------------------------------------------------ EPI_L2NORM (final_proj)
@pytest.mark.parametrize("K1,zero_bias", [(64, True), (128, False), (192, False), (256, True)])
def test_l2norm(lib, K1, zero_bias):
    """F.normalize(acc + bias) per row; an all-zero row (zero A row, zero bias) hits the 1e-12 clamp and gives 0."""
    g = _gen(K1)
    rows = 768
    a = rand(g, rows, K1)
    a[5] = 0.0
    a[300] = 0.0
    x = split(lib, a)
    w = split(lib, rand(g, 256, K1, K1 ** -0.5))
    bias = torch.zeros(256, device=DEV) if zero_bias else rand(g, 1, 256)[0]
    f = dict(epi=_lib.EPI_L2NORM, rows=rows, n_out=256, K1=K1, a1_hi=x[0], a1_lo=x[1], a1_ld=K1, b1_hi=w[0], b1_lo=w[1],
             b1_ld=K1, bias=bias, out_ld=256)
    name = f"l2norm K1={K1} zero_bias={zero_bias}"
    outs = schedules(lib, name, f, {"out_hi": torch.empty(rows, 256, dtype=torch.float16, device=DEV),
                                    "out_lo": torch.empty(rows, 256, dtype=torch.float16, device=DEV)})
    dev = gr.plane_value(outs["out_hi"], outs["out_lo"])
    r, S = gr.product([(x[2], w[2])])
    y = r + bias.double()
    rn, allowed = gr.l2norm_reference(y, gr.product_bar(S, K1, 3) + gr.F32_OUT * y.abs())
    zero = y.abs().amax(1) == 0
    ratios = dict(rows=gr.ratio((dev - rn).abs()[~zero], allowed[~zero]))
    if zero_bias:
        assert bool(zero[5]) and bool(zero[300])
        ratios["zero_rows"] = 0.0 if bool((dev[zero] == 0).all()) else float("inf")
    report(name, **ratios)


# ------------------------------------------------------------------------------------------------ EPI_SCORE_SUMS / EPI_SCORE_CONF
@pytest.mark.parametrize("conf_ld", [0, 301])
def test_score_tail(lib, conf_ld):
    """The batched score GEMM (one batch = one frame): pass 1's partial row / column sums of e = exp((cos - 1) / scale), then pass
    2's conf = (e irs)(e ics) (through the tensor map when conf_ld % 4 == 0, plain stores otherwise) and the packed arg-maxes.
    Bars of tests/matcher_stage_reference.py; entries past the valid counts exactly 0."""
    L = ref.Layout(3, 200, 300, 256, 512, nlen=[200, 57, 0], mlen=[300, 299, 128])
    scale = 0.1
    g = _gen(conf_ld + 5)
    lf, keep = layout_fields(L)
    pn = torch.nn.functional.normalize(rand(g, L.rows, 256), dim=1)
    pn[~L.valid_mask(DEV)] = GARBAGE
    p = split(lib, pn)
    bview = (p[0][L.n_pad:], p[1][L.n_pad:])
    base = dict(rows=L.n_pad, n_out=L.m_pad, K1=256, batch=L.B, a_batch_rows=L.R, b_batch_rows=L.R, a1_hi=p[0], a1_lo=p[1],
                a1_ld=256, b1_hi=bview[0], b1_lo=bview[1], b1_ld=256, inv_scale=1.0 / scale, **lf)
    n_tiles, m_tiles = L.m_pad // 256, L.n_pad // 128
    sums = schedules(lib, "score sums", {**base, "epi": _lib.EPI_SCORE_SUMS},
                     {"rowsum_part": torch.empty(L.B, 2 * n_tiles, L.n_pad, device=DEV),
                      "colsum_part": torch.empty(L.B, m_tiles * 4, L.m_pad, device=DEV)})
    rs_ref, cs_ref, cos = gr.score_partials(p[2], L, scale)
    rel = 1e-5 + ref.COS_ERR / scale
    ratios = {}
    for k, r in (("rowsum_part", rs_ref), ("colsum_part", cs_ref)):
        d = sums[k].double()
        z = r == 0
        ratios[k] = max(gr.ratio((d - r).abs()[~z], rel * r[~z]), 0.0 if bool((d[z] == 0).all()) else float("inf"))
    report("score sums", **ratios)
    # pass 2 with the fp64 inverse sums as fp32 inputs
    irs = torch.zeros(L.B, L.n_pad, device=DEV)
    ics = torch.zeros(L.B, L.m_pad, device=DEV)
    for b in range(L.B):
        n, m = L.n_of(b), L.m_of(b)
        if n:
            e = torch.exp((cos[b][:n, :m] - 1.0) / scale)
            irs[b, :n] = (1.0 / e.sum(1)).float()
            ics[b, :m] = (1.0 / e.sum(0)).float()
    ld = conf_ld or L.M
    outs = schedules(lib, f"score conf ld={ld}", {**base, "epi": _lib.EPI_SCORE_CONF, "inv_rowsum": irs, "inv_colsum": ics,
                                                  "conf_ld": conf_ld},
                     {"conf": torch.empty(L.B, L.N, ld, device=DEV), "rowbest": torch.empty(L.B, L.N, dtype=torch.int64, device=DEV),
                      "colbest": torch.empty(L.B, L.M, dtype=torch.int64, device=DEV)}, zero=("rowbest", "colbest"))
    ratios = dict(conf=0.0, outside=0.0)
    mism = 0
    for b in range(L.B):
        n, m = L.n_of(b), L.m_of(b)
        conf = outs["conf"][b]
        outside = torch.ones_like(conf, dtype=torch.bool)
        outside[:n, :m] = False
        if bool((conf[outside] != 0).any()):
            ratios["outside"] = float("inf")
        if n == 0:
            mism += int((outs["rowbest"][b] != 0).sum() + (outs["colbest"][b] != 0).sum())
            continue
        c = conf[:n, :m]
        ratios["conf"] = max(ratios["conf"], ref.bar_conf(c, cos[b][:n, :m], irs[b, :n].double(), ics[b, :m].double(), scale))
        i0, v0 = ref.unpack_best(outs["rowbest"][b, :n])
        i1, v1 = ref.unpack_best(outs["colbest"][b, :m])
        mism += ref.first_max_mismatches(i0, v0, c, 1) + ref.first_max_mismatches(i1, v1, c, 0)
        mism += int((outs["rowbest"][b, n:] != 0).sum() + (outs["colbest"][b, m:] != 0).sum())
    report(f"score conf ld={ld}", **ratios)
    assert mism == 0, f"{mism} packed arg-maxes are not the first maximum of the device's conf"


# ------------------------------------------------------------------------------------------------ EPI_CONV
@pytest.mark.parametrize("bn,taps,cin,halo", [(64, 9, 64, 1), (64, 9, 128, 0), (64, 1, 128, 1), (128, 9, 64, 1), (128, 1, 64, 1)])
def test_conv(lib, bn, taps, cin, halo):
    """3x3 / 1x1 convolution over a zero-bordered grid of two 10 x 13 images: out planes = ReLU(conv + bias) on the interior,
    exactly 0 on the border and the padding rows.  3x3 on 64-wide tiles: halo boxes and nine boxes bit-identical with 64 input
    channels, both within the bar with more."""
    g = _gen(bn + taps + cin)
    H, W, ppad, imgs, cout = 10, 13, 256, 2, 128
    w2 = W + 2
    rows = imgs * ppad
    r = torch.arange(rows, device=DEV)
    qpix = r % ppad
    yy, xx = qpix // w2, qpix % w2
    interior = (yy >= 1) & (yy <= H) & (xx >= 1) & (xx <= W)
    act = rand(g, rows, cin).abs() * interior[:, None]           # a valid zero-bordered input grid
    a = split(lib, act)
    offs = [(t // 3 - 1) * w2 + (t % 3 - 1) for t in range(9)] if taps == 9 else [0]
    K1 = taps * cin
    w = split(lib, rand(g, cout, K1, K1 ** -0.5))
    bias = rand(g, 1, cout)[0] * 0.1
    f = dict(epi=_lib.EPI_CONV, bn=bn, rows=rows, n_out=cout, K1=K1, a1_hi=a[0], a1_lo=a[1], a1_ld=cin, b1_hi=w[0], b1_lo=w[1],
             b1_ld=K1, bias=bias, out_ld=cout, taps=taps, kb_per_tap=cin // 64, tap_off=offs, cv_w2=w2, cv_h=H, cv_w=W,
             cv_ppad=ppad, relu=1)
    name = f"conv bn{bn} taps={taps} cin={cin} halo={halo}"
    assert lib.opb_debug_set_conv_halo(halo) == 0
    try:
        outs = schedules(lib, name, f, {"out_hi": torch.empty(rows, cout, dtype=torch.float16, device=DEV),
                                        "out_lo": torch.empty(rows, cout, dtype=torch.float16, device=DEV)})
        other = None
        if bn == 64 and taps == 9:
            assert lib.opb_debug_set_conv_halo(1 - halo) == 0
            other = launch(lib, f, {k: torch.empty_like(v) for k, v in outs.items()})
            if cin == 64:                                       # the same MMAs in the same order
                for k in outs:
                    assert torch.equal(_bytes(outs[k]), _bytes(other[k])), f"{name}: halo and nine-box results differ ({k})"
    finally:
        lib.opb_debug_set_conv_halo(1)
    dev = gr.plane_value(outs["out_hi"], outs["out_lo"])
    zero = torch.zeros(1, cin, dtype=torch.float64, device=DEV)
    y = torch.zeros(rows, cout, dtype=torch.float64, device=DEV)
    S = torch.zeros_like(y)
    for t, o in enumerate(offs):
        src = r + o
        ok = (src >= 0) & (src < rows)
        sh = torch.where(ok[:, None], a[2][src.clamp(0, rows - 1)], zero)
        wt = w[2][:, t * cin:(t + 1) * cin]
        y += sh @ wt.T
        S += sh.abs() @ wt.abs().T
    y = torch.relu(y + bias.double())
    allowed = gr.product_bar(S, K1, 3) + gr.planes_bar(y)
    ratios = dict(interior=gr.ratio((dev - y).abs()[interior], allowed[interior]), border=ref._pad_ratio(dev, interior))
    if other is not None and cin > 64:
        # more than one channel block: the halo form runs (kernel row, channel block, dx), the nine boxes (tap, channel block) --
        # the same products in another accumulation order, each within the bar
        dev2 = gr.plane_value(other["out_hi"], other["out_lo"])
        ratios.update(other_staging=gr.ratio((dev2 - y).abs()[interior], allowed[interior]),
                      other_border=ref._pad_ratio(dev2, interior))
    report(name, **ratios)


# ------------------------------------------------------------------------------------------------ PDL chain
def test_pdl_chain(lib):
    """Launch 1's planes output is launch 2's A operand, back to back on one stream with programmatic dependent launch; the
    same pair with a synchronisation between them, and with PDL off: all three bit-identical."""
    L = BP_L
    g = _gen(77)
    lf, keep = layout_fields(L)
    x = split(lib, masked_rows(rand(g, L.rows, 256), L))
    w1 = split(lib, rand(g, 256, 256, 1 / 16))
    w2 = split(lib, rand(g, 512, 256, 1 / 16))
    bias = rand(g, 1, 256)[0]
    mid = [torch.empty(L.rows, 256, dtype=torch.float16, device=DEV) for _ in range(2)]
    c = torch.empty(L.rows, 512, device=DEV)
    d1 = _lib.gemm_desc(epi=_lib.EPI_BIAS_PLANES, rows=L.rows, n_out=256, K1=256, a1_hi=x[0], a1_lo=x[1], a1_ld=256, b1_hi=w1[0],
                        b1_lo=w1[1], b1_ld=256, bias=bias, out_hi=mid[0], out_lo=mid[1], out_ld=256, **lf)
    d2 = _lib.gemm_desc(epi=_lib.EPI_F32, rows=L.rows, n_out=512, K1=256, a1_hi=mid[0], a1_lo=mid[1], a1_ld=256, b1_hi=w2[0],
                        b1_lo=w2[1], b1_ld=256, c=c, ldc=512)
    stream = torch.cuda.current_stream().cuda_stream

    def pair(sync):
        for t in mid + [c]:
            _bytes(t).fill_(0xFF)
        torch.cuda.synchronize()
        assert lib.opb_debug_gemm(d1, C.c_void_p(stream)) == 0
        if sync:
            torch.cuda.synchronize()
        assert lib.opb_debug_gemm(d2, C.c_void_p(stream)) == 0
        torch.cuda.synchronize()
        return [t.clone() for t in mid + [c]]

    try:
        runs = {"pdl": pair(False), "sync": pair(True)}
        assert lib.opb_debug_set_pdl(0) == 0
        runs["no pdl"] = pair(False)
    finally:
        lib.opb_debug_set_pdl(1)
    for k in ("sync", "no pdl"):
        for a, b in zip(runs["pdl"], runs[k]):
            assert torch.equal(_bytes(a), _bytes(b)), f"PDL chain differs from the {k} run"
    dev = runs["pdl"][2].double()
    r, S = gr.product([(gr.plane_value(runs["pdl"][0], runs["pdl"][1]), w2[2])])
    report("pdl chain", product=gr.ratio((dev - r).abs(), gr.product_bar(S, 256, 3)))


def test_refused_combinations(lib):
    """The converter without an identity block, an identity block without the converter, the SIMT backend on an epilogue and
    an unknown b2_mode are refused (no instantiation exists for them)."""
    L, f, keep, _ = _mlp3_problem(lib, 64)
    outs = {"out_hi": torch.empty(L.rows, 256, dtype=torch.float16, device=DEV),
            "out_lo": torch.empty(L.rows, 256, dtype=torch.float16, device=DEV)}
    INVALID = -1
    assert lib.opb_debug_gemm(_lib.gemm_desc(**{**f, **outs, "b2_mode": 0}), None) == INVALID
    no_conv = {**f, **outs, "b2_mode": 2, "a_raw": 0, "a1_hi": f["a2_hi"], "a1_lo": f["a2_lo"], "a1_ld": 256}
    assert lib.opb_debug_gemm(_lib.gemm_desc(**no_conv), None) == INVALID
    assert lib.opb_debug_gemm(_lib.gemm_desc(**{**f, **outs, "b2_mode": 2, "backend": 1}), None) == INVALID
    assert lib.opb_debug_gemm(_lib.gemm_desc(**{**f, **outs, "b2_mode": 3}), None) == INVALID
