"""The GEMM core's ping-pong schedule (csrc/gemm_tc.cu, PP): 128 x 128 tiles, the CTA's units alternating between the two
consumer warpgroups, one warpgroup's epilogue under the other's main loop.

A unit's ring position is (units done by the CTA) x (k-blocks per tile) + k-block, and which warpgroup runs it is the unit's
parity in the CTA, so the schedule is exercised by: CTAs with one unit (warpgroup 1 idle), two, and odd and even counts
above that; k-blocks per tile in every residue mod (3 ring stages x 2 warpgroups) = 6.  Every case is held to its fp64 bar
and must be bit-identical across grids (the result of a tile does not depend on the CTA or warpgroup that computes it)."""
from __future__ import annotations

import pytest
import torch

from onepose_b200 import _lib
from tests import gemm_core_reference as gr
from tests import matcher_stage_reference as ref
from tests.test_gemm_core_gpu import DEV, _bytes, _gen, launch, layout_fields, masked_rows, rand, report, split

pytestmark = pytest.mark.gpu

# 768 x 256 -> 12 units of 128 x 128: 1 CTA = 12 units, 2 = 6 each, 5 = 3, 3, 2, 2, 2, 7 = 2 x 5 + 1 x 2, 12 = 1 each
ROWS, N_OUT = 768, 256
PP_CTAS = (1, 2, 5, 7, 12, 132)


@pytest.fixture(scope="module")
def lib():
    return _lib.load()


def grids(lib, name, fields, outs):
    """Default grid, then every max_ctas of PP_CTAS: all bit-identical.  Returns the default run's outputs."""
    base = launch(lib, fields, outs)
    for ctas in PP_CTAS:
        got = launch(lib, fields, outs, max_ctas=ctas)
        for k in outs:
            assert torch.equal(_bytes(base[k]), _bytes(got[k])), f"{name}: {k} differs with max_ctas = {ctas}"
    return base


# k-blocks per tile 1 .. 7 (every residue mod 6), the last three with a K2 block
PP_K = [(64, 0), (128, 0), (192, 0), (256, 0), (192, 128), (256, 128), (320, 128)]


@pytest.mark.parametrize("K1,K2", PP_K)
def test_pingpong_f32(lib, K1, K2):
    g = _gen(100 + K1 + K2)
    a1 = split(lib, rand(g, ROWS, K1) * torch.exp(rand(g, ROWS, 1)))
    b1 = split(lib, rand(g, N_OUT, K1, K1 ** -0.5))
    f = dict(epi=_lib.EPI_F32, rows=ROWS, n_out=N_OUT, K1=K1, K2=K2, a1_hi=a1[0], a1_lo=a1[1], a1_ld=K1, b1_hi=b1[0],
             b1_lo=b1[1], b1_ld=K1, ldc=N_OUT)
    A = [(a1[2], b1[2])]
    if K2:
        a2, b2 = split(lib, rand(g, ROWS, K2)), split(lib, rand(g, N_OUT, K2, 0.1))
        f.update(a2_hi=a2[0], a2_lo=a2[1], a2_ld=K2, b2_hi=b2[0], b2_lo=b2[1], b2_ld=K2)
        A.append((a2[2], b2[2]))
    out = grids(lib, f"pp f32 K1={K1} K2={K2}", f, {"c": torch.empty(ROWS, N_OUT, device=DEV)})["c"]
    r, S = gr.product(A)
    report(f"pp f32 K1={K1} K2={K2}", product=gr.ratio((out.double() - r).abs(), gr.product_bar(S, K1 + K2, 3) + gr.F32_OUT * r.abs()))


# ragged segments: 3 frames, one without queries; 256-row aligned segments -> 18 row tiles x 4 column tiles = 72 units
PP_STATS_L = ref.Layout(3, 200, 300, 256, 512, nlen=[200, 0, 77], mlen=[300, 129, 1])


@pytest.mark.parametrize("K1,K2", [(64, 64), (128, 192), (256, 256)])
def test_pingpong_f32_stats(lib, K1, K2):
    """mlp.0's epilogue under the ping-pong schedule: product and the per-quarter InstanceNorm partials over ragged segments."""
    L = PP_STATS_L
    g = _gen(200 + K1 + K2)
    n_out = 512
    lf, keep = layout_fields(L)
    x = split(lib, masked_rows(rand(g, L.rows, K1), L))
    w = split(lib, rand(g, n_out, K1, K1 ** -0.5))
    q = split(lib, masked_rows(rand(g, L.rows, K2).abs(), L))
    G = split(lib, rand(g, L.S * n_out, K2, K2 ** -0.5) + 3.0)
    bias = rand(g, 1, n_out)[0]
    f = dict(epi=_lib.EPI_F32_STATS, rows=L.rows, n_out=n_out, K1=K1, K2=K2, a1_hi=x[0], a1_lo=x[1], a1_ld=K1, b1_hi=w[0],
             b1_lo=w[1], b1_ld=K1, a2_hi=q[0], a2_lo=q[1], a2_ld=K2, b2_hi=G[0], b2_lo=G[1], b2_ld=K2, b2_mode=1, bias=bias,
             ldc=n_out, **lf)
    outs = grids(lib, f"pp stats K1={K1} K2={K2}", f, {"c": torch.empty(L.rows, n_out, device=DEV),
                                                        "statpart": torch.empty(L.rows // 32, n_out, 2, device=DEV)})
    seg = L.seg_index(DEV)
    Gs = G[2].view(L.S, n_out, K2)
    r = x[2] @ w[2].T + torch.einsum("rk,rnk->rn", q[2], Gs[seg]) + bias.double()
    S = x[2].abs() @ w[2].abs().T + torch.einsum("rk,rnk->rn", q[2].abs(), Gs[seg].abs())
    dev_c = outs["c"].double()
    s_ref, m2_ref, s_bar, m2_bar, empty = gr.quarter_stats(dev_c, L)
    sp = outs["statpart"].double()
    report(f"pp stats K1={K1} K2={K2}", product=gr.ratio((dev_c - r).abs(), gr.product_bar(S, K1 + K2, 3) + gr.F32_OUT * r.abs()),
           sum=gr.ratio((sp[..., 0] - s_ref).abs(), s_bar), m2=gr.ratio((sp[..., 1] - m2_ref).abs(), m2_bar),
           empty_quarters=0.0 if bool((sp[empty] == 0).all()) else float("inf"))
