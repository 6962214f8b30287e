"""CPU checks of the pose hand-off: the reference's pose metric (pnp.pose_errors / pnp.cm_degree against what the unmodified
reference computed, tests/golden/pnp_pose_metrics.npz), the numpy restatement of the matcher -> PnP gather against the
reference's masking expression, and the argument checks of opb_gather_matches (they run before any CUDA call)."""
import ctypes as C
import os

import numpy as np
import torch

from onepose_b200 import _lib, pnp
from tests.gather_oracle import gather_matches
from tests.golden_util import GOLDEN_DIR


def _golden():
    return dict(np.load(os.path.join(GOLDEN_DIR, "pnp_pose_metrics.npz"), allow_pickle=False))


def _acos_slack_deg(ref_deg, delta=1e-15):
    """How far the angle can move when (trace - 1) / 2 moves by a few units in the last place: acos has an unbounded slope at
    0 and 180 degrees, so there numpy's BLAS product (which may fuse multiply-adds) and an unfused sum differ by ~1e-6 degree."""
    c = np.cos(np.deg2rad(ref_deg))
    a = np.arccos(c)
    return np.rad2deg(np.maximum(np.abs(np.arccos(np.clip(c + delta, -1, 1)) - a), np.abs(np.arccos(np.clip(c - delta, -1, 1)) - a)))


def _check_errors(g, rot, trans):
    for i, tag in enumerate(g["tags"]):
        r_ref, t_ref = g["rot_err_deg"][i], g["trans_err_cm"][i]
        if np.isnan(r_ref):             # the trace rounded below -1: NaN, or 180 degrees where the trace rounds to -1
            assert np.isnan(rot[i]) or abs(rot[i] - 180.0) <= 1e-6, (tag, rot[i])
        else:
            assert abs(rot[i] - r_ref) <= 1e-9 + _acos_slack_deg(r_ref), (tag, rot[i], r_ref)
        if np.isnan(t_ref):
            assert np.isnan(trans[i]), tag
        else:
            assert abs(trans[i] - t_ref) <= 1e-9, (tag, trans[i], t_ref)


def test_pose_errors_match_reference_query_pose_error():
    """Per pair with the shapes the reference was called with (3x4 / 4x4 mixes), and as one batch of 4x4 poses."""
    g = _golden()
    rot, trans = [], []
    for p, q, pr, gr in zip(g["pose_pred"], g["pose_gt"], g["pred_rows"], g["gt_rows"]):
        r, t = pnp.pose_errors(torch.from_numpy(p[:pr])[None], torch.from_numpy(q[:gr])[None])
        assert r.dtype == torch.float64 and r.shape == (1,) and t.shape == (1,)
        rot.append(float(r[0]))
        trans.append(float(t[0]))
    _check_errors(g, np.array(rot), np.array(trans))
    rb, tb = pnp.pose_errors(torch.from_numpy(g["pose_pred"]), torch.from_numpy(g["pose_gt"]))
    np.testing.assert_array_equal(rb.numpy(), np.array(rot))
    np.testing.assert_array_equal(tb.numpy(), np.array(trans))
    rb3, tb3 = pnp.pose_errors(torch.from_numpy(g["pose_pred"][:, :3]), torch.from_numpy(g["pose_gt"]))
    np.testing.assert_array_equal(rb3.numpy(), rb.numpy())
    np.testing.assert_array_equal(tb3.numpy(), tb.numpy())


def test_cm_degree_matches_aggregate_metrics_and_evaluator():
    g = _golden()
    agg = dict(zip((str(k) for k in g["aggregate_keys"]), g["aggregate_vals"]))
    summ = dict(zip((str(k) for k in g["summarize_keys"]), g["summarize_vals"]))
    rot, trans = pnp.pose_errors(torch.from_numpy(g["pose_pred"]), torch.from_numpy(g["pose_gt"]))
    for errs in ((rot, trans), (torch.from_numpy(g["rot_err_deg"]), torch.from_numpy(g["trans_err_cm"]))):
        got = pnp.cm_degree(*errs)
        assert list(got) == list(agg), (list(got), list(agg))
        for thr, key in zip((1, 3, 5), agg):
            assert got[key] == agg[key] == summ[f"cmd{thr}"], (key, got[key], agg[key])
    assert list(pnp.cm_degree(rot, trans, thresholds=(2,))) == ["2cm@2degree"]


def test_gather_oracle_matches_reference_masking():
    """The restatement equals inference.py:147-152 (valid = matches > -1; kpts2d[valid]; kpts3d[matches[valid]]; conf[valid])
    frame by frame, on matches in the reference's own domain [-1, M)."""
    rs = np.random.RandomState(3)
    for B, N, M in ((1, 1, 1), (3, 37, 50), (4, 500, 7000), (2, 0, 5)):
        m0 = np.where(rs.rand(B, N) < 0.4, rs.randint(0, M, size=(B, N)), -1).astype(np.int64)
        if B > 1:
            m0[0] = -1
            m0[1] = rs.randint(0, M, size=N)
        kp2 = rs.randn(B, N, 2).astype(np.float32)
        kp3 = rs.randn(M, 3).astype(np.float32)
        sc = rs.rand(B, N).astype(np.float32)
        g = gather_matches(m0, kp2, kp3, sc)
        for b in range(B):
            matches, kpts2d, confidence = m0[b], kp2[b], sc[b]
            valid = matches > -1
            mkpts2d, mkpts3d, mconf = kpts2d[valid], kp3[matches[valid]], confidence[valid]
            o0, o1 = g["offsets"][b], g["offsets"][b + 1]
            assert np.array_equal(g["pts2d"][o0:o1], mkpts2d.astype(np.float64))
            assert np.array_equal(g["pts3d"][o0:o1], mkpts3d.astype(np.float64))
            assert np.array_equal(g["mconf"][o0:o1], mconf)
            assert np.array_equal(g["query_index"][o0:o1], np.nonzero(valid)[0])
        assert g["offsets"][0] == 0 and g["offsets"][-1] == len(g["pts2d"])


def test_gather_matches_rejects_bad_arguments():
    lib = _lib.load()
    buf = C.c_void_p(16)     # never dereferenced: every call below fails its argument check first

    def call(m0=buf, sc=None, kp2=buf, kp3=buf, B=2, N=4, M=3, p2=buf, p3=buf, mconf=None, qi=None, off=buf):
        return lib.opb_gather_matches(m0, sc, kp2, kp3, B, N, M, p2, p3, mconf, qi, off, None)

    for kw in (dict(B=0), dict(B=-1), dict(N=-1), dict(M=0), dict(off=None), dict(kp3=None), dict(m0=None), dict(kp2=None),
               dict(p2=None), dict(p3=None), dict(mconf=buf), dict(B=1 << 16, N=1 << 16)):
        assert call(**kw) == -1, kw
