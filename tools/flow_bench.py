"""Times the tracker's flow step on the device: ``flow.lk_batch`` and ``flow.flow_track`` for B = 1 / 8 / 32 tracks of 512 x 512
crops and 100 / 1000 points, with CUDA events, and the reference's host path from the same device tensors (to the host, cv2
LK and solvePnPRansac per track, the pose back) where cv2 is installed.  Prints the card's name, power limit and SM clock
read in the same run, and one JSON line per configuration.

    python tools/flow_bench.py [--reps 20]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from onepose_b200 import flow, synthetic  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi unavailable: {e}"


def scene(B, n, S=512):
    rs = np.random.RandomState(B * 7 + n)
    tex = np.round(synthetic.make_image(1, S, S)[0] * 255).astype(np.uint8)
    shift = rs.uniform(-3, 3, (B, 2))
    nxt = np.stack([np.roll(tex, (int(round(dy)), int(round(dx))), (0, 1)) for dx, dy in shift])
    pts = rs.uniform(40, S - 40, (B, n, 2)).astype(np.float32)
    pts3d = np.concatenate([(pts - S / 2) / S * 0.2, np.zeros((B, n, 1), np.float32)], 2).astype(np.float32)
    return np.stack([tex] * B), nxt, pts, pts3d


def events(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    print("card:", card())
    try:
        import cv2
    except ImportError:
        cv2 = None
    dev = "cuda"
    K = torch.tensor([[600.0, 0, 256], [0, 600.0, 256], [0, 0, 1]], dtype=torch.float64, device=dev)
    for B in (1, 8, 32):
        for n in (100, 1000):
            prev, nxt, pts, pts3d = scene(B, n)
            P, N = torch.from_numpy(prev).to(dev), torch.from_numpy(nxt).to(dev)
            p2 = torch.from_numpy(pts).to(dev)
            off = torch.arange(0, (B + 1) * n, n, dtype=torch.int32, device=dev)
            kf = {"image": P, "pts2d": p2, "pts3d": torch.from_numpy(pts3d).to(dev), "counts": torch.full((B,), n, dtype=torch.int32, device=dev)}
            pose_ref = torch.eye(4, dtype=torch.float64, device=dev).expand(B, 4, 4).contiguous()
            t_lk = events(lambda: flow.lk_batch(P, N, p2.reshape(-1, 2), off), args.reps)
            t_ft = events(lambda: flow.flow_track(kf, N, K, pose_ref), args.reps)
            row = {"B": B, "points": n, "crop": 512, "lk_batch_ms": round(t_lk, 4), "flow_track_ms": round(t_ft, 4)}
            if cv2 is not None:
                def host():
                    a, b, q, q3 = P.cpu().numpy(), N.cpu().numpy(), p2.cpu().numpy(), kf["pts3d"].cpu().numpy()
                    Kn = K.cpu().numpy()
                    out = []
                    for i in range(B):
                        t, st, _ = cv2.calcOpticalFlowPyrLK(a[i], b[i], q[i][:, None], None, winSize=(15, 15), maxLevel=2, criteria=(3, 10, 0.03))
                        v = st[:, 0] == 1
                        try:
                            _, rv, tv, _ = cv2.solvePnPRansac(q3[i][v].astype(np.float64), t[:, 0][v].astype(np.float64), Kn, np.zeros(8),
                                                              reprojectionError=5, iterationsCount=10000, flags=cv2.SOLVEPNP_EPNP)
                            out.append(np.concatenate([cv2.Rodrigues(rv)[0], tv], 1))
                        except cv2.error:
                            out.append(np.eye(4)[:3])
                    return torch.from_numpy(np.stack(out)).to(dev)
                host()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(max(args.reps // 4, 2)):
                    host()
                torch.cuda.synchronize()
                row["host_cv2_ms"] = round((time.perf_counter() - t0) * 1e3 / max(args.reps // 4, 2), 4)
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
