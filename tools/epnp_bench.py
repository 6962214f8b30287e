"""EPnP-RANSAC on one GPU: CUDA-event time of pnp.poses_from_matches(method="epnp", 10000 hypotheses) against the P3P path
(method="p3p", its default 4096 hypotheses) and, if cv2 imports, the reference's host loop (cv2.solvePnPRansac(EPNP) per
frame, host clock), at B in {1, 8, 32} frames of n in {100, 500} pairs (synthetic.make_pnp_scene: 40 % outliers, 0.5 px noise).
Alternated in one process, median and spread over repeats; also the frames within 1cm@1degree of the ground truth.  Prints
one JSON line with the card name and power limit of the run.

    python tools/epnp_bench.py [--repeats 5] [--iters 10] [--out FILE]"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from onepose_b200 import pnp, synthetic  # noqa: E402
from tools.pose_bench import card, stats, timed  # noqa: E402


def frames(B, n):
    """matches0 [B,n] into a concatenated keypoints3d [B*n,3]: frame b's pair i is 3D row b*n + i."""
    Ks, uv, P, gt = zip(*(synthetic.make_pnp_scene(9000 + 97 * b + n, n) for b in range(B)))
    m0 = torch.arange(B * n, dtype=torch.int64).reshape(B, n)
    kp2 = torch.from_numpy(np.stack(uv).astype(np.float32))
    kp3 = torch.from_numpy(np.concatenate(P).astype(np.float32))
    return {"K": torch.from_numpy(np.stack(Ks)).cuda(), "kp2": kp2.cuda(), "kp3": kp3.cuda(), "m0": m0.cuda(),
            "gt": torch.from_numpy(np.stack(gt)).cuda(), "np": (np.stack(Ks), np.stack(uv).astype(np.float32), np.concatenate(P).astype(np.float32))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    try:
        import cv2
    except ImportError:
        cv2 = None
    result = {"card": card(), "hypotheses": {"epnp": pnp.EPNP_HYPOTHESES, "p3p": pnp.DEFAULT_HYPOTHESES}, "rows": []}
    for n in (100, 500):
        for B in (1, 8, 32):
            f = frames(B, n)

            def run(method):
                return pnp.poses_from_matches(f["K"], f["kp2"], f["kp3"], f["m0"], method=method)

            acc = {}
            for method in ("epnp", "p3p"):
                res = run(method)
                rot, trans = pnp.pose_errors(res["pose"], f["gt"])
                acc[method] = pnp.cm_degree(rot, trans)["1cm@1degree"]
            t = {"epnp": [], "p3p": []}
            for _ in range(args.repeats):
                for method in ("epnp", "p3p"):
                    t[method].append(timed(lambda: run(method), args.iters))
            row = {"B": B, "n": n, "epnp": stats(t["epnp"]), "p3p": stats(t["p3p"]), "cmd1": acc}
            if cv2 is not None:
                Ks, uv, P = f["np"]
                hs = []
                for _ in range(max(1, args.repeats // 2)):
                    t0 = time.perf_counter()
                    for b in range(B):
                        cv2.solvePnPRansac(P[b * n:(b + 1) * n].astype(np.float64) * 1000, uv[b].astype(np.float64), Ks[b],
                                           np.zeros((8, 1)), reprojectionError=5, iterationsCount=10000, flags=cv2.SOLVEPNP_EPNP)
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
