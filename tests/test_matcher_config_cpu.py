"""The matcher's configuration edges without a GPU: what the reference's threshold comparison does, and the tail's exponential
near the smallest scale_factor opb_create accepts.

* Threshold: the reference compares `mscores0 > match_threshold` with mscores0 an fp32 tensor and the threshold a Python float.
  PyTorch casts a Python scalar to the tensor's dtype, so the comparison is in fp32.  The device stores fp32(match_threshold) and
  compares fp32 scores to it, so the oracle and the device agree for every double, by construction.
* The bound: the score epilogues compute e = ex2(fma(acc, ea, eb)) with ex2.approx.ftz, which flushes results below 2^-126 to 0.
  opb_create refuses scale_factor < 2 log2(e) / 126, so that e stays normal for every cos >= -1.  The bar on the score GEMM's
  cos allows COS_ERR = 48 x 2^-23 either way, and just above the bound a cos of -1 - COS_ERR would take the argument below
  -126: a row whose every entry is there would sum to 0, its inverse sum would be inf and its conf 0 x inf = NaN.  The device
  does not get there: its fp32 accumulator rounds toward zero (tests/gemm_core_reference.py), so the 3-pass product of a unit
  row with its own negation, which also drops the lo x lo term, lands above -1, and the argument stays above -126 at every
  accepted scale.  tests/test_matcher_config_gpu.py plants such rows on the device at the smallest scale."""
import numpy as np
import torch

from onepose_b200 import synthetic
from oracle import gats_spg_oracle as oracle
from tests import gemm_core_reference as gr
from tests import matcher_stage_reference as ref

F32 = np.float32
LOG2E = F32(1.4426950408889634)
BOUND = 2.0 * np.log2(np.e) / 126.0
SCALE_MIN = np.nextafter(F32(BOUND), F32(1))        # the smallest scale_factor opb_create accepts


# ------------------------------------------------------------------------------------------------ threshold
def test_threshold_comparison_is_in_fp32():
    """A double just below an fp32 score c that rounds to c does not let c pass, in torch (the reference) or in the stage
    reference's `mutual`; fp32(c)'s predecessor does.  In fp64 the double would let it pass."""
    c = F32(0.6180339)
    below = float(c) - float(np.spacing(c)) / 4
    assert F32(below) == c and float(c) > below
    t = torch.tensor([c], dtype=torch.float32)
    assert not bool((t > below)[0])                                  # fp32: fp32(below) == c
    assert bool((t.double() > below)[0])                             # an fp64 comparison would differ
    assert bool((t > float(np.nextafter(c, F32(0))))[0])
    conf = torch.tensor([[c, 0.1, 0.05], [0.2, 0.01, 0.3]], dtype=torch.float32)
    for thr, n in ((below, 0), (float(c), 0), (float(np.nextafter(c, F32(0))), 1), (0.0, 2), (1.0, 0), (float("nan"), 0)):
        m0, m1, s0, _ = ref.mutual(conf, thr)
        assert int((m0 > -1).sum()) == n and int((m1 > -1).sum()) == n, thr
        assert float(s0[0]) == float(c)                               # the scores do not depend on the threshold


def test_oracle_threshold_at_a_produced_score():
    """The oracle at a threshold equal to one of its own mutual scores (as fp32, and as a double just below it that rounds to
    it): that match is dropped, the same matches as at fp32(threshold); at the predecessor of the score it is kept."""
    sd = synthetic.make_state_dict(4)
    data = synthetic.make_batch(9, [100], 64, 96, 8)
    P = oracle.params_from_numpy(sd)
    hp = dict(synthetic.DEFAULT_HPARAMS)
    first = oracle.forward(P, data, hp)
    s0, m0 = first["matching_scores0"][0], first["matches0"][0]
    vals = torch.sort(s0[m0 > -1]).values
    assert vals.numel() >= 5
    c = F32(vals[vals.numel() // 2].item())
    below = float(c) - float(np.spacing(c)) / 4
    outs = {thr: oracle.forward(P, data, dict(hp, match_threshold=thr))["matches0"][0]
            for thr in (float(c), below, float(np.nextafter(c, F32(0))))}
    assert torch.equal(outs[float(c)], outs[below])
    assert torch.equal(outs[float(c)], torch.where(s0 > float(c), m0, -1))
    kept = outs[float(np.nextafter(c, F32(0)))]
    assert torch.equal(kept, torch.where(s0 >= float(c), m0, -1))
    assert int((kept > -1).sum()) > int((outs[float(c)] > -1).sum())


# ------------------------------------------------------------------------------------------------ the bound window
def _ex2_ftz(x):
    """ex2.approx.ftz.f32 on its range: 2^x, and +0 where the result would be below 2^-126."""
    x = np.asarray(x, np.float64)
    return np.where(x < -126.0, 0.0, np.exp2(np.maximum(x, -126.0)))


def _argument(cos, scale):
    """The epilogue's fp32 argument: acc = cos x 2^12 (the fp16-split product's pre-scale), inv_scale = 1.f / scale (api.cu),
    ea = 2^-12 inv_scale log2(e), eb = -inv_scale log2(e) (each product rounded to fp32), t = fma(acc, ea, eb)."""
    inv = F32(1) / F32(scale)
    ea = F32(F32(F32(2.0 ** -12) * inv) * LOG2E)
    eb = F32(-inv * LOG2E)
    acc = np.asarray(F32(np.asarray(cos, np.float64) * 4096.0), np.float64)
    t = (acc * np.float64(ea) + np.float64(eb)).astype(F32)            # acc * ea is exact in fp64; one rounding to fp32
    return t


def _scales_above_bound(n):
    """The first n fp32 scale factors opb_create accepts."""
    s = [SCALE_MIN]
    for _ in range(n - 1):
        s.append(np.nextafter(s[-1], F32(1)))
    return np.array(s, F32)


def test_a_cosine_below_minus_one_flushes_just_above_the_bound():
    """At the smallest accepted scales an all-antipodal row with cos = -1 - COS_ERR would sum to 0 (every e flushed) and its
    conf would be NaN; that window ends within about COS_ERR / 2 relative of the bound, and cos = -1 itself never enters it."""
    cos = -1.0 - ref.COS_ERR
    scales = _scales_above_bound(400)
    flushed = np.array([_ex2_ftz(_argument(cos, s)) == 0.0 for s in scales])
    assert flushed[0], "nextafter(bound) is inside the window"
    last = int(np.nonzero(flushed)[0].max())
    assert 10 <= last < 200 and not flushed[last + 1:].any()
    rel = float(scales[last]) / BOUND - 1.0
    assert rel < ref.COS_ERR / 2 * 1.05, rel
    print(f"{last + 1} fp32 scale factors above the bound flush cos = -1 - COS_ERR (up to {rel:.2e} relative)")
    assert all(_ex2_ftz(_argument(-1.0, s)) > 0 for s in scales)
    # the chain the flush starts: row sum 0 -> inverse inf -> conf 0 x inf = NaN
    with np.errstate(divide="ignore", invalid="ignore"):
        e = F32(_ex2_ftz(_argument(cos, scales[0])))
        irs = F32(1) / (e * F32(700))
        assert np.isinf(irs) and np.isnan((e * irs) * (e * F32(1)))


def test_the_device_cos_of_antipodal_unit_rows_stays_above_minus_one():
    """The score GEMM's accumulation as the device runs it (fp16-split planes, three passes, the fp32 accumulator rounded toward
    zero once per pass and k-step of 16; gemm_core_reference.emulate_product) on unit rows against their negation: cos lands
    in (-1, -1 + COS_ERR], never below -1, so ex2's argument stays at or above -126 at the smallest accepted scale.  Rounding
    to nearest instead could put it below -1 by up to COS_ERR."""
    rs = np.random.RandomState(0)
    q = rs.randn(64, 256)
    q = (q / np.linalg.norm(q, axis=1, keepdims=True)).astype(F32).astype(np.float64)
    hi, lo = gr.split_planes(q)
    blocks = [(hi[:, k:k + 64], lo[:, k:k + 64], -hi[:, k:k + 64], -lo[:, k:k + 64]) for k in range(0, 256, 64)]
    cos = np.diag(gr.emulate_product(blocks, True)) / 4096.0
    assert (cos > -1.0).all() and (cos <= -1.0 + ref.COS_ERR).all(), (cos.min(), cos.max())
    assert (_argument(cos, SCALE_MIN) >= -126.0).all()
    print(f"emulated antipodal cos + 1 in [{cos.min() + 1:.2e}, {cos.max() + 1:.2e}]")
