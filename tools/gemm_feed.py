#!/usr/bin/env python
"""Where the matcher's GEMM time goes: the wgmma core's main-loop rate and per-tile cost, and the per-launch profile of a step.

    python tools/gemm_feed.py [--lib PATH] [--window 0.5]

(a) opb_debug_gemm (tensor-core backend, fp16-split planes, 128 x 256 tiles, EPI_F32) at rows = 262144, n_out = 512 and
    K = 256 / 512 / 1024 / 2048, each timed with CUDA events over >= --window seconds of back-to-back launches.  A least-squares
    line of time against K: the slope is the main loop's cost per k-block, the intercept the per-launch fixed cost (epilogue,
    ring refills, launch).  The slope is reported as executed TFLOP/s (three fp16 passes per product), as the shared-memory
    fill per SM (96 KB land in a CTA's ring per k-block: A hi/lo + B hi/lo) and as that fill summed over the SMs.
(b) the mlp.3-shaped GEMM (converter variant: A = ReLU(IN(hid)) formed from raw fp32 in the core, plus the identity K-block)
    at rows = 262144 (32 frames of 1024 + 7168 rows), n_out = 256 and K1 = 256 / 512 / 768 / 1024.  The same line fit; the
    slope counts the three passes of the K1 part only, the identity block is in the intercept.  Both (a) and (b) go through
    opb_debug_gemm's problem descriptor.
(c) the benchmarked call (match_frames, B = 32, N2D = 1024, N3D = 7000) with the profiling hook on: ms per step and share of
    the step for every GEMM and the large helper kernels.

--lib loads another build of the library (A/B between builds in one process).  Needs a GPU; there is no CPU path.
"""
from __future__ import annotations

import argparse
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ROWS, N_OUT, KS = 262144, 512, (256, 512, 1024, 2048)
BM, BN, BK = 128, 256, 64
STAGE_BYTES = 2 * BM * BK * 2 + 2 * BN * BK * 2          # A hi/lo + B hi/lo of one k-block
DENSE_FLOP_PER_CLK_SM = 4096                             # fp16 wgmma, dense
MLP3_FRAMES, MLP3_NPAD, MLP3_MPAD, MLP3_K1S = 32, 1024, 7168, (256, 512, 768, 1024)
PROFILE_PREFIXES = [("gemm epi9 ", "k,v projection (EPI_QKV)"), ("gemm epi2 ", "q projection (EPI_QSCALE)"),
                    ("gemm epi10 n256 k256 ", "G fold (EPI_BIAS_PLANES)"), ("gemm epi1 ", "mlp.0 (EPI_F32_STATS)"),
                    ("gemm epi10 n256 k768 ", "mlp.3 + residual (EPI_BIAS_PLANES, ACV_NORM_RELU)"),
                    ("gemm epi5 ", "final_proj (EPI_L2NORM)"), ("gemm epi6 ", "score pass 1 (EPI_SCORE_SUMS)"),
                    ("gemm epi7 ", "score pass 2 (EPI_SCORE_CONF)"), ("gemm epi0 ", "fp32 out (EPI_F32)"),
                    ("kv_state_h", ""), ("gats_aggregate", ""), ("in_stats_final", ""), ("score_sums_finalize", ""),
                    ("mutual_match", "")]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[torch.cuda.current_device()]
    except (OSError, subprocess.SubprocessError, IndexError):
        return "nvidia-smi unavailable"


def time_launches(launch, window):
    """(ms per launch, launches) over >= window seconds of back-to-back launches, after a warm-up."""
    for _ in range(3):
        launch()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        launch()
    e1.record()
    torch.cuda.synchronize()
    n = max(10, int(np.ceil(window / (e0.elapsed_time(e1) * 1e-3 / 5))))
    e0.record()
    for _ in range(n):
        launch()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n, n


def gemm_slope(lib, window):
    from onepose_b200 import _lib
    dev = torch.device("cuda")
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    kmax = max(KS)
    g = torch.Generator(device=dev).manual_seed(0)
    a = [torch.randn(ROWS, kmax, device=dev, generator=g).half() for _ in range(2)]
    b = [torch.randn(N_OUT, kmax, device=dev, generator=g).half() for _ in range(2)]
    c = torch.empty(ROWS, N_OUT, device=dev)
    rows = []
    for K in KS:
        # K-major planes of width K: the first K columns of contiguous copies
        ak = [x[:, :K].contiguous() for x in a]
        bk = [x[:, :K].contiguous() for x in b]
        desc = _lib.gemm_desc(epi=_lib.EPI_F32, rows=ROWS, n_out=N_OUT, K1=K, a1_hi=ak[0], a1_lo=ak[1], a1_ld=K,
                              b1_hi=bk[0], b1_lo=bk[1], b1_ld=K, c=c, ldc=N_OUT)

        def launch():
            rc = lib.opb_debug_gemm(desc, None)
            if rc != 0:
                raise RuntimeError(f"opb_debug_gemm rc={rc}")

        rows.append((K,) + time_launches(launch, window))
        del ak, bk
    Ks = np.array([r[0] for r in rows], float)
    ts = np.array([r[1] for r in rows], float)
    slope, icept = np.polyfit(Ks, ts, 1)                    # ms per unit of K, ms
    tiles = (ROWS // BM) * (N_OUT // BN)
    kb_per_k = 1.0 / BK
    exec_flop_per_k = 3 * 2.0 * ROWS * N_OUT              # three fp16 passes
    tflops = exec_flop_per_k / (slope * 1e-3) / 1e12
    fill_tbs = tiles * kb_per_k * STAGE_BYTES / (slope * 1e-3) / 1e12
    print("(a) opb_debug_gemm, tensor-core backend, rows=%d n_out=%d, %d tiles of %dx%d, %d SMs" % (ROWS, N_OUT, tiles, BM, BN, sms))
    for K, ms, n in rows:
        print(f"    K={K:5d}  {ms:8.3f} ms/launch  ({n} launches)  {exec_flop_per_k * K / (ms * 1e-3) / 1e12:6.1f} TFLOP/s executed")
    resid = ts - (slope * Ks + icept)
    print(f"    slope      {slope * BK * 1e3:8.2f} us per k-block of the whole launch ({tiles} tiles); fit residual max {np.abs(resid).max():.4f} ms")
    print(f"    main loop  {tflops:6.1f} TFLOP/s executed   shared-memory fill {fill_tbs * 1e3 / sms:6.1f} GB/s per SM = "
          f"{fill_tbs:5.2f} TB/s over {sms} SMs ({STAGE_BYTES // 1024} KB per tile and k-block)")
    print(f"    intercept  {icept:8.3f} ms per launch = {icept * 1e3 / (tiles / sms):6.2f} us per tile wave")
    return {"slope_tflops_executed": tflops, "fill_tbs": fill_tbs, "fill_gbs_per_sm": fill_tbs * 1e3 / sms, "intercept_ms": icept,
            "points": [{"K": K, "ms": ms} for K, ms, _ in rows]}


def mlp3_slope(lib, window):
    from onepose_b200 import _lib
    dev = torch.device("cuda")
    rows = MLP3_FRAMES * (MLP3_NPAD + MLP3_MPAD)
    segs = 2 * MLP3_FRAMES
    g = torch.Generator(device=dev).manual_seed(0)
    planes = lambda r, c: [torch.randn(r, c, device=dev, generator=g).half() for _ in range(2)]   # noqa: E731
    x, out = planes(rows, 256), planes(rows, 256)
    eye = [(64 * torch.eye(256, device=dev)).half(), torch.zeros(256, 256, device=dev).half()]
    bias = torch.randn(256, device=dev, generator=g)
    nparam = (segs + max(MLP3_K1S) // 512) * 512
    mu, rstd = 0.1 * torch.randn(nparam, device=dev, generator=g), 1 + 0.1 * torch.rand(nparam, device=dev, generator=g)
    pts = []
    for K1 in MLP3_K1S:
        hid = torch.randn(rows, K1, device=dev, generator=g)
        w1 = planes(256, K1)
        # every row valid: frames of n_pad + m_pad rows with N = n_pad, M = m_pad
        desc = _lib.gemm_desc(epi=_lib.EPI_BIAS_PLANES, rows=rows, n_out=256, K1=K1, K2=256, b1_hi=w1[0], b1_lo=w1[1], b1_ld=K1,
                              a2_hi=x[0], a2_lo=x[1], a2_ld=256, b2_hi=eye[0], b2_lo=eye[1], b2_ld=256, b2_mode=2,
                              a_raw=hid, a_raw_ld=K1, mu=mu, rstd=rstd, B=MLP3_FRAMES, N=MLP3_NPAD, M=MLP3_MPAD,
                              n_pad=MLP3_NPAD, m_pad=MLP3_MPAD, bias=bias, out_hi=out[0], out_lo=out[1], out_ld=256)

        def launch():
            rc = lib.opb_debug_gemm(desc, None)
            if rc != 0:
                raise RuntimeError(f"opb_debug_gemm (mlp.3) rc={rc}")

        pts.append((K1,) + time_launches(launch, window))
        del hid, w1
    Ks = np.array([p[0] for p in pts], float)
    ts = np.array([p[1] for p in pts], float)
    slope, icept = np.polyfit(Ks, ts, 1)
    tflops = 3 * 2.0 * rows * 256 / (slope * 1e-3) / 1e12
    print(f"(b) mlp.3-shaped GEMM, rows={rows} n_out=256 K2=256")
    for K1, ms, n in pts:
        print(f"    K1={K1:5d}  {ms:8.3f} ms/launch  ({n} launches)")
    print(f"    main loop  {tflops:6.1f} TFLOP/s executed (K1 part)   intercept {icept:8.3f} ms per launch   "
          f"fit residual max {np.abs(ts - (slope * Ks + icept)).max():.4f} ms")
    return {"slope_tflops_executed": tflops, "intercept_ms": icept, "points": [{"K1": K1, "ms": ms} for K1, ms, _ in pts]}


def step_profile(runs=5):
    from onepose_b200 import GATsSuperGlue, synthetic
    dev = torch.device("cuda")
    hp = dict(synthetic.DEFAULT_HPARAMS)
    model = GATsSuperGlue(hp).eval()
    model.load_state_dict({k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in synthetic.make_state_dict(0).items()})
    model = model.to(dev)
    B, N, M = 32, 1024, 7000
    db, leaves = synthetic.make_object(0, M, 8)
    q = torch.from_numpy(np.stack([synthetic.make_frame(f, db, N)[0] for f in range(B)], 0)).to(dev)
    model.set_object(torch.from_numpy(db).to(dev), torch.from_numpy(leaves).to(dev), reserve=(B, N))
    for _ in range(4):
        model.match_frames(q)
    torch.cuda.synchronize()
    model.set_profiling(True)
    acc = {p: [0.0, 0.0, 0] for p, _ in PROFILE_PREFIXES}
    total = 0.0
    for _ in range(runs):
        model.match_frames(q)
        total += model.get_profile()["total_ms"]
        for p, _ in PROFILE_PREFIXES:
            e = model.get_profile_entry(p)
            acc[p][0] += e["ms"]; acc[p][1] += e["flops"]; acc[p][2] = e["launches"]
    model.set_profiling(False)
    total /= runs
    print(f"(c) match_frames B={B} N2D={N} N3D={M}, profiling on (an event after every launch), "
          f"mean of {runs} steps: {total:.3f} ms/step")
    print(f"    {'entry':22s} {'launches':>8s} {'ms/step':>8s} {'share':>6s} {'TFLOP/s alg.':>12s}  what")
    out = {"step_ms": total, "entries": {}}
    for p, what in PROFILE_PREFIXES:
        ms, fl, n = acc[p][0] / runs, acc[p][1] / runs, acc[p][2]
        if n == 0:
            continue
        tf = fl / (ms * 1e-3) / 1e12 if fl > 0 and ms > 0 else 0.0
        print(f"    {p:22s} {n:8d} {ms:8.3f} {100 * ms / total:5.1f}% {tf:12.1f}  {what}")
        out["entries"][p.strip()] = {"launches": n, "ms": ms, "share": ms / total, "tflops_algorithmic": tf}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None, help="path of the library build to load (default: the in-tree build)")
    ap.add_argument("--window", type=float, default=0.5, help="seconds of launches per K")
    ap.add_argument("--no-mlp3", action="store_true", help="skip the fit of the mlp.3-shaped GEMM")
    ap.add_argument("--no-step", action="store_true", help="skip the per-launch profile of the benchmarked call")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gemm_feed.py needs a CUDA device")
    from onepose_b200 import _lib
    if args.lib:
        _lib.LIB_PATH = os.path.abspath(args.lib)
    lib = _lib.load()
    print("card:", card(), "| library:", _lib.LIB_PATH)
    gemm_slope(lib, args.window)
    if not args.no_mlp3:
        mlp3_slope(lib, args.window)
    if not args.no_step:
        step_profile()


if __name__ == "__main__":
    main()
