"""Times the tracker's flow-only step on the device: ``track.step`` against ``flow.flow_track`` alone (the cost the gate, the
keyframe choice and the pose choice add) for B = 1 / 8 / 32 tracks of 512 x 512 crops and 100 / 1000 keyframe points, with
CUDA events, and against the reference's host path for the same step where cv2 is installed: the crops, points and poses to
the host, cv2 LK and solvePnPRansac per track, the numpy gate and rule of tests/track_reference.py, the poses back.  All three
follow the same keyframe (this frame's crop and points) into the crop, and the timed steps cycle through the demo's frames
(one in five an update frame).  Prints the card's name, power limit and SM clock
read in the same run, and one JSON line per configuration.

    python tools/track_bench.py [--reps 20]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from flow_bench import card, events, scene  # noqa: E402

from onepose_b200 import flow, track  # noqa: E402
from tests import track_reference as TR  # noqa: E402


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
            _, nxt, pts, pts3d = scene(B, n)
            N = torch.from_numpy(nxt).to(dev)
            p2 = torch.from_numpy(pts).to(dev)
            p3 = torch.from_numpy(pts3d).to(dev)
            pose = torch.eye(4, dtype=torch.float64, device=dev).expand(B, 4, 4).contiguous()
            pose[:, 2, 3] = 600.0 * 0.2 / 512                  # the depth at which pts3d projects onto the key points
            res = {"offsets": torch.arange(0, (B + 1) * n, n, dtype=torch.int32, device=dev), "inlier_mask": torch.ones(B * n, dtype=torch.bool, device=dev),
                   "pts2d": p2.reshape(-1, 2).double(), "pts3d": p3.reshape(-1, 3).double(), "pose_homo": pose}
            state = track.init_state(B, n, 512, dev)
            track.step(state, res, N, K)               # the keyframe is now this frame's, as the demo's state after its first frame
            kf = state["kf"]
            t_ft = events(lambda: flow.flow_track(kf, N, K, pose), args.reps)
            t_st = events(lambda: track.step(state, res, N, K), args.reps)
            row = {"B": B, "points": n, "crop": 512, "flow_track_ms": round(t_ft, 4), "step_ms": round(t_st, 4), "added_ms": round(t_st - t_ft, 4)}
            if cv2 is not None:
                host_state = TR.init_state(B)
                Kn = K.cpu().numpy()

                def host():
                    a, b, q, q3, pp = kf["image"].cpu().numpy(), N.cpu().numpy(), kf["pts2d"].cpu().numpy(), kf["pts3d"].cpu().numpy(), pose.cpu().numpy()
                    TR.gate(host_state, pp)
                    flow_pose, kd = np.zeros((B, 4, 4)), np.zeros(B)
                    for i in range(B):
                        t, st, _ = cv2.calcOpticalFlowPyrLK(a[i], b[i], q[i][:, None], None, winSize=(15, 15), maxLevel=2, criteria=(3, 10, 0.03))
                        v = st[:, 0] == 1
                        flow_pose[i] = np.eye(4)
                        try:
                            _, rv, tv, _ = cv2.solvePnPRansac(q3[i][v].astype(np.float64), t[:, 0][v].astype(np.float64), Kn, np.zeros(8),
                                                              reprojectionError=5, iterationsCount=10000, flags=cv2.SOLVEPNP_EPNP)
                            flow_pose[i, :3] = np.concatenate([cv2.Rodrigues(rv)[0], tv], 1)
                        except cv2.error:
                            pass
                        x = q3[i][v] @ flow_pose[i, :3, :3].T + flow_pose[i, :3, 3]
                        x = x @ Kn.T
                        kd[i] = np.mean(np.linalg.norm(x[:, :2] / x[:, 2:] - t[:, 0][v], axis=1))
                    out, _ = TR.select(host_state, pp, flow_pose, kd)
                    return torch.from_numpy(out).to(dev)
                host()
                torch.cuda.synchronize()
                reps = max(args.reps // 4, 2)
                t0 = time.perf_counter()
                for _ in range(reps):
                    host()
                torch.cuda.synchronize()
                row["host_ms"] = round((time.perf_counter() - t0) * 1e3 / reps, 4)
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
