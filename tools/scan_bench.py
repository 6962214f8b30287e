"""An annotated scan's poses and crops, on one GPU, at F in {1, 8, 32} BGR frames of 1440 x 1920 and 512 x 512 crops:
  device      scan.annotate on frames already on the device: poses, boxes, colour crops, K_crop, M and box_crop (CUDA events over
              --iters calls);
  host        the reference's host loop per frame (tests/scan_reference.py): numpy poses with np.linalg.inv, the projections,
              two cv2.warpAffine calls and parse_video's M and box_crop;
  png         the PNG round trip the evaluation puts the crops through: cv2.imencode(".png") of each BGR crop and
              cv2.imdecode(IMREAD_GRAYSCALE).
Host legs are timed by the host clock.  The legs alternate inside every repeat; median, min and max over the repeats.  The
device crops are checked against the host loop's before timing.  Prints a table and one JSON line with the card's name, power
limit and clocks.

    python tools/scan_bench.py [--repeats 5] [--iters 20]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from onepose_b200 import scan  # noqa: E402
from tests import scan_reference as sr  # noqa: E402

H, W, S = 1440, 1920, 512


def card():
    q = "name,power.limit,clocks.max.sm,clocks.sm,clocks.mem"
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return dict(zip(q.split(","), [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]))
    except Exception as e:            # noqa: BLE001
        return {"name": torch.cuda.get_device_name(0), "note": f"nvidia-smi: {e}"}


def scene(F):
    """F ARposes rows of a camera circling a 0.3 m box at 0.6-0.9 m, every box inside the frame; text lines as in the file."""
    fx = fy = 1450.0
    K = np.array([[fx, 0, W / 2 - 0.5], [0, fy, H / 2 + 0.25], [0, 0, 1]])
    box_lines = ["# position, extent, quaternion\n", "0.01,0.02,-0.03,0.3,0.22,0.26,0.98,0.1,0.05,0.15\n"]
    from scipy.spatial.transform import Rotation
    T_ow = sr.parse_box(box_lines)
    lines = []
    for i in range(F):
        a = 2 * np.pi * i / max(F, 1)
        R_cv = Rotation.from_rotvec([0.2 * np.sin(a), a, 0.1]).as_matrix()
        z = 0.6 + 0.3 * (i % 4) / 3
        p = T_ow[:3, 3] - R_cv @ (z * np.linalg.solve(K, [W / 2 + 100 * np.sin(a), H / 2 + 80 * np.cos(a), 1.0]))
        q = Rotation.from_matrix(R_cv @ sr.FLIP).as_quat()
        lines.append(",".join(repr(float(v)) for v in [0.033 * i, *p, q[3], *q[:3]]) + "\n")
    return K, box_lines, lines


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--frames", type=int, nargs="+", default=[1, 8, 32])
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("scan_bench needs a GPU")
    import cv2
    dev = torch.device("cuda:0")
    info = {"card": card(), "torch_name": torch.cuda.get_device_name(0), "cv2": cv2.__version__, "H": H, "W": W, "S": S, "results": {}}
    for F in a.frames:
        K, box_lines, lines = scene(F)
        bbox3d, homo = sr.get_bbox3d(box_lines)
        T_ow = sr.parse_box(box_lines)
        rows = np.array([[float(e) for e in ln.split(",")] for ln in lines])
        frames = [sr.colour_frame(H, W, f) for f in range(F)]
        fr = torch.from_numpy(np.stack(frames)).to(dev)
        args = [torch.from_numpy(np.ascontiguousarray(v)).to(dev) for v in (K, rows, T_ow, bbox3d)]

        def host():
            saved, _ = sr.process_poses(K, box_lines, lines)
            return sr.parse_video(frames, saved, K, homo, S)

        ann = scan.annotate(fr, *args, crop_size=S)
        ref = host()
        img = ann["image"].cpu().numpy()
        assert all(r is not None and np.array_equal(img[f], r["image"]) for f, r in enumerate(ref)), "device crops differ from the host loop's"
        crops = [r["image"] for r in ref]

        def png():
            return [cv2.imdecode(cv2.imencode(".png", c)[1], cv2.IMREAD_GRAYSCALE) for c in crops]

        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        legs = {"device": [], "host": [], "png": []}
        for _ in range(3):
            scan.annotate(fr, *args, crop_size=S)
        torch.cuda.synchronize()
        for _ in range(a.repeats):
            e0.record()
            for _ in range(a.iters):
                scan.annotate(fr, *args, crop_size=S)
            e1.record()
            torch.cuda.synchronize()
            legs["device"].append(e0.elapsed_time(e1) / a.iters)
            for name, fn in (("host", host), ("png", png)):
                t = time.perf_counter()
                fn()
                legs[name].append((time.perf_counter() - t) * 1e3)
        info["results"][F] = {k: {"median_ms": statistics.median(v), "min_ms": min(v), "max_ms": max(v)} for k, v in legs.items()}
        r = info["results"][F]
        print(f"F={F:3d}  device {r['device']['median_ms']:9.3f} ms   host loop {r['host']['median_ms']:9.2f} ms   png {r['png']['median_ms']:9.2f} ms")
    print(json.dumps(info))


if __name__ == "__main__":
    main()
