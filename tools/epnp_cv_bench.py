"""EPnP-RANSAC with OpenCV's loop on one GPU: CUDA-event time per call of pnp.ransac_pnp_batch(method="epnp",
confidence=0.99) against the fixed-count path (method="epnp", all 10000 samples) and, if cv2 imports, the reference's host
loop (cv2.solvePnPRansac(EPNP) per frame, host clock; B <= 8), at B in {1, 8, 32} frames, n in {100, 500} pairs and 25 / 50 / 80 %
outliers (synthetic.make_pnp_scene, 1 px noise).  Alternated in one process, median and spread over repeats; also the
iterations the frames' loops ran.  ``--waves 256,1024`` adds the confidence mode at those fixed wave sizes (samples per frame
and wave).  Prints one JSON line with the card name and power limit of the run, and ptxas' register / stack use of the
new kernels if ``--ptxas`` is given (compiles csrc/pnp_ransac.cu into a temporary directory).

    python tools/epnp_cv_bench.py [--repeats 3] [--iters 5] [--waves 256,1024,4096] [--ptxas] [--out FILE]"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from onepose_b200 import _lib, pnp, synthetic  # noqa: E402
from tools.pose_bench import card, stats, timed  # noqa: E402


def frames(B, n, frac):
    sc = [synthetic.make_pnp_scene(9100 + 97 * b + n, n, outlier_frac=frac, noise_px=1.0) for b in range(B)]
    K = torch.from_numpy(np.stack([s[0] for s in sc])).cuda()
    p2 = torch.from_numpy(np.concatenate([s[1] for s in sc])).cuda()
    p3 = torch.from_numpy(np.concatenate([s[2] for s in sc]) * 1000).cuda()
    off = torch.arange(0, B * n + 1, n, dtype=torch.int32).cuda()
    return K, p2, p3, off, sc


def ptxas():
    """Registers, stack and spills of the EPnP-RANSAC kernels, from nvcc -Xptxas -v."""
    src = os.path.join(ROOT, "onepose_b200", "csrc", "pnp_ransac.cu")
    with tempfile.TemporaryDirectory() as d:
        r = subprocess.run(["/usr/local/cuda/bin/nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-c", src, "-o",
                            os.path.join(d, "p.o"), "-Xptxas", "-v"], capture_output=True, text=True)
    out, name = {}, None
    for line in r.stderr.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            name = next((k for k in ("epnp_cv_scan", "epnp_cv_wave", "epnp_cv_select_refit", "epnp_hypotheses", "epnp_select_refit")
                         if k in m.group(1)), None)
            continue
        if name is None:
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            out.setdefault(name, {}).update(stack=int(m.group(1)), spill_stores=int(m.group(2)), spill_loads=int(m.group(3)))
        m = re.search(r"Used (\d+) registers", line)
        if m:
            out.setdefault(name, {})["registers"] = int(m.group(1))
            name = None
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--waves", default="")
    ap.add_argument("--ptxas", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    waves = [int(w) for w in args.waves.split(",") if w]
    try:
        import cv2
    except ImportError:
        cv2 = None
    lib = _lib.load()
    result = {"card": card(), "hypotheses": pnp.EPNP_HYPOTHESES, "confidence": 0.99, "cv2": cv2.__version__ if cv2 else None, "rows": []}
    if args.ptxas:
        result["ptxas"] = ptxas()
    for n in (100, 500):
        for frac in (0.25, 0.5, 0.8):
            for B in (1, 8, 32):
                K, p2, p3, off, sc = frames(B, n, frac)
                its = torch.empty(B, dtype=torch.int32, device="cuda")
                variants = {"fixed": lambda: pnp.ransac_pnp_batch(K, p2, p3, off, method="epnp"),
                            "cv": lambda: pnp.ransac_pnp_batch(K, p2, p3, off, method="epnp", confidence=0.99, iterations_out=its)}
                for w in waves:
                    variants[f"cv_w{w}"] = (lambda w=w: (lib.opb_debug_set_cv_wave(w), variants["cv"](), lib.opb_debug_set_cv_wave(0)))
                for f in variants.values():
                    f()
                torch.cuda.synchronize()
                t = {k: [] for k in variants}
                for _ in range(args.repeats):
                    for k, f in variants.items():
                        t[k].append(timed(f, args.iters))
                variants["cv"]()
                it = its.cpu().numpy()
                row = {"B": B, "n": n, "outliers": frac, **{k: stats(v) for k, v in t.items()},
                       "iterations": {"min": int(it.min()), "median": float(np.median(it)), "max": int(it.max())}}
                if cv2 is not None and B <= 8:                 # 32 frames of the 80 % case take minutes on the host
                    hs = []
                    for _ in range(max(1, args.repeats // 2)):
                        t0 = time.perf_counter()
                        for s in sc:
                            cv2.solvePnPRansac(s[2] * 1000, s[1], s[0], np.zeros((8, 1)), reprojectionError=5, iterationsCount=10000,
                                               confidence=0.99, flags=cv2.SOLVEPNP_EPNP)
                        hs.append((time.perf_counter() - t0) * 1e3)
                    row["cv2_host"] = stats(hs)
                print(json.dumps(row), flush=True)
                result["rows"].append(row)
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
