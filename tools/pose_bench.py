"""Matcher -> pose hand-off on one GPU: CUDA-event time of pnp.gather_matches and pnp.poses_from_matches against the torch
argsort glue of bench.py's pipeline leg (alternated in the same process, median and spread over repeats), on planted scenes
(synthetic.make_planted_scene: N = 1024 query points, 512 planted) at B in {1, 8, 32} frames and M in {2500, 7000} 3D points,
plus the frames within 1cm@1degree of the ground truth.  Prints one JSON line with the card name and power limit of the run.

    python tools/pose_bench.py [--repeats 7] [--iters 20] [--out FILE]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from onepose_b200 import GATsSuperGlue, pnp, synthetic  # noqa: E402


def card():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        name, power = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power}
    except Exception as e:            # noqa: BLE001
        return {"name": torch.cuda.get_device_name(0), "power_limit": None, "note": f"nvidia-smi: {e}"}


def glue(m0, kp2, kp3_f64):
    """bench.py leg_pipeline's hand-off: valid pairs first, grouped by frame, by a stable argsort."""
    B, N = m0.shape
    frame_id = torch.arange(B, device=m0.device)[:, None].expand(B, N)
    valid = m0 > -1
    order = torch.argsort((~valid).long().flatten() * B + frame_id.flatten(), stable=True)
    p2 = kp2.reshape(B * N, 2)[order]
    p3 = kp3_f64[m0.clamp(min=0).flatten()[order]]
    off = torch.cat([torch.zeros(1, dtype=torch.int64, device=m0.device), valid.sum(1).cumsum(0)]).to(torch.int32)
    return p2, p3, off


def timed(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def stats(xs):
    return {"median_ms": statistics.median(xs), "min_ms": min(xs), "max_ms": max(xs)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("pose_bench.py measures on the GPU and there is none")
    dev = torch.device("cuda", 0)
    N = 1024
    rows = []
    for M in (2500, 7000):
        for B in (1, 8, 32):
            s = synthetic.make_planted_scene(M % 97, list(range(600, 600 + B)), N, M)
            mm = GATsSuperGlue(dict(synthetic.DEFAULT_HPARAMS)).eval()
            mm.load_state_dict({k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in synthetic.make_state_dict(0).items()})
            mm = mm.to(dev)
            mm.set_object(torch.from_numpy(s["desc3d"]).to(dev), torch.from_numpy(s["desc2d_db"]).to(dev))
            out = mm.match_frames(torch.from_numpy(s["descriptors2d"]).to(dev), return_conf=False)
            m0, s0 = out["matches0"], out["matching_scores0"]
            kp2, kp3, K = (torch.from_numpy(s[k]).to(dev) for k in ("keypoints2d", "keypoints3d", "K"))
            kp3_f64 = kp3.double()

            def new_gather():
                return pnp.gather_matches(m0, kp2, kp3, s0)

            def new_poses():
                return pnp.poses_from_matches(K, kp2, kp3, m0, s0)

            def glue_gather():
                return glue(m0, kp2, kp3_f64)

            def glue_poses():
                p2, p3, off = glue(m0, kp2, kp3_f64)
                pose, _, n_in = pnp.ransac_pnp_batch(K, p2, p3 * 1000.0, off)
                pose[:, :, 3] /= 1000.0
                return pose, n_in

            legs = {"gather": new_gather, "gather_argsort_glue": glue_gather, "poses": new_poses, "poses_argsort_glue": glue_poses}
            for fn in legs.values():
                fn()
            torch.cuda.synchronize()
            t = {k: [] for k in legs}
            for _ in range(a.repeats):                 # the new path and the glue alternate inside every repeat
                for k, fn in legs.items():
                    t[k].append(timed(fn, a.iters))
            res = new_poses()
            rot, trans = pnp.pose_errors(res["pose"], torch.from_numpy(s["pose_gt"]).to(dev))
            ref = glue_poses()
            g = new_gather()
            gp2, gp3, goff = glue_gather()
            T = int(g["offsets"][-1])
            row = {"B": B, "N": N, "M": M, "pairs": T, "frames_within_1cm_1deg": int(((rot < 1) & (trans < 1)).sum()),
                   "max_rot_err_deg": float(rot.max()), "max_trans_err_cm": float(trans.max()),
                   "same_pairs_as_glue": bool(torch.equal(g["offsets"], goff) and torch.equal(g["pts2d"][:T], gp2[:T].double())
                                              and torch.equal(g["pts3d"][:T], gp3[:T])),
                   "same_poses_as_glue": bool(torch.equal(res["pose"], ref[0]) and torch.equal(res["n_inliers"], ref[1]))}
            row.update({k: stats(v) for k, v in t.items()})
            rows.append(row)
            print(json.dumps(row), file=sys.stderr)
            del mm
    result = {"card": card(), "repeats": a.repeats, "iters_per_repeat": a.iters,
              "note": "CUDA events around iters back-to-back calls, per call; argsort glue = bench.py leg_pipeline's hand-off "
                      "(+ x1000 scale and /1000 translation for the poses leg, as poses_from_matches does)",
              "rows": rows}
    line = json.dumps(result)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
