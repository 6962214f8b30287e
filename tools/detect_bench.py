"""Detection after the matcher on one GPU, at B in {1, 8, 32} frames of 1440 x 1920 against 15 reference views with 50-1000
matches per view and 25-90 % outliers (a planted similarity per view).  CUDA-event time, with a synchronise, of
  boxes        detect.boxes_from_matches: per-view counts, the choice, estimateAffinePartial2D on the chosen view, the box;
  detect       detect.detect_from_matches: the same, then the 512 x 512 crop and K_crop;
  host         the reference's path from the same device tensors: per frame and view matches0 to the host (one
               synchronisation each), cv2.estimateAffinePartial2D(ransacReprojThreshold=6) on views with >= 6 matches, the numpy
               box and choice, the two cv2.warpAffine of crop_img_by_bbox and the float image back to the device (frames already
               in host memory, as the reference reads them from disk).
The legs alternate inside every repeat; median and spread over the repeats.  Boxes of the device and host legs are compared.
Prints one JSON line with the card's name, power limit and clocks.

    python tools/detect_bench.py [--repeats 7] [--iters 10] [--out FILE]"""
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
from onepose_b200 import detect  # noqa: E402
from tests import crop_reference as cr  # noqa: E402

H, W, S, V, CAP_REF, CAP_Q = 1440, 1920, 512, 15, 1200, 4096


def card():
    q = "name,power.limit,clocks.max.sm,clocks.sm,clocks.mem"
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return dict(zip(q.split(","), [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]))
    except Exception as e:            # noqa: BLE001
        return {"name": torch.cuda.get_device_name(0), "note": f"nvidia-smi: {e}"}


def timed(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def stats(xs):
    return {"median_ms": statistics.median(xs), "min_ms": min(xs), "max_ms": max(xs)}


def workload(rng, B):
    """Reference views of 480 x 640 with CAP_REF key points; per frame and view 50-1000 matches, 25-90 % of them outliers."""
    ref_kp = np.stack([rng.integers(0, 640, CAP_REF), rng.integers(0, 480, CAP_REF)], axis=-1).astype(np.float32)[None].repeat(V, 0)
    ref_kp = ref_kp + rng.integers(0, 3, (V, 1, 2)).astype(np.float32)
    q_kp = rng.uniform([0, 0], [W, H], (B, CAP_Q, 2)).astype(np.float32)
    m0 = np.full((B, V, CAP_REF), -1, np.int64)
    for b in range(B):
        used = 0
        for v in range(V):
            k = int(rng.integers(50, 1001))
            frac = rng.uniform(0.25, 0.9)
            a, s = rng.uniform(-0.5, 0.5), rng.uniform(0.8, 1.6)
            R = s * np.array([[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]])
            t = np.array([W / 2, H / 2]) - R @ np.array([320, 240])
            idx = np.sort(rng.choice(CAP_REF, k, replace=False))
            k = min(k, CAP_Q - used)
            idx = idx[:k]
            q = np.arange(used, used + k)
            used += k
            inl = rng.random(k) >= frac
            q_kp[b, q[inl]] = np.round(ref_kp[v, idx[inl]] @ R.T + t + rng.normal(0, 0.7, (int(inl.sum()), 2)))
            m0[b, v, idx] = q
    return ref_kp, q_kp, m0


def host_path(cv2, frames_host, K, ref_kp_d, q_kp_d, m0_d, dev):
    """The reference's match_worker / detect_by_matching / crop_img_by_bbox from device tensors, one frame at a time."""
    images, boxes = [], []
    ref_kp = ref_kp_d.cpu().numpy()
    for b in range(len(frames_host)):
        q_kp = q_kp_d[b].cpu().numpy()
        best = None
        for v in range(V):
            m = m0_d[b, v].cpu().numpy()                                        # .cpu() per view, as match_worker does
            valid = m > -1
            n = int(valid.sum())
            if n < 6:
                cand = (0, np.array([0, 0, H, W]))
            else:
                affine, _ = cv2.estimateAffinePartial2D(ref_kp[v][valid], q_kp[m[valid]], ransacReprojThreshold=6)
                c = (affine @ np.array([[0, 0, 1], [640, 0, 1], [0, 480, 1], [640, 480, 1]]).T).T.astype(np.int32)
                cand = (n, np.concatenate([c.min(0), c.max(0)]))
            if best is None or cand[0] > best[0]:
                best = cand
        box = best[1].astype(np.int32)
        boxes.append(box)
        x0, y0, x1, y1 = (int(v) for v in box)
        T1 = cr.box_transform(box, y1 - y0, x1 - x0)
        im1 = cv2.warpAffine(frames_host[b], T1, (x1 - x0, y1 - y0), flags=cv2.INTER_LINEAR)
        T2 = cr.box_transform([0, 0, x1 - x0, y1 - y0], S, S)
        images.append(cv2.warpAffine(im1, T2, (S, S), flags=cv2.INTER_LINEAR).astype(np.float32) / 255)
    img = torch.from_numpy(np.stack(images)[:, None]).to(dev)
    return np.stack(boxes), img


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("detect_bench needs a CUDA device")
    import cv2
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(0)
    frames_all = torch.from_numpy(cr.synthetic_frame(H, W, 2)).to(dev)
    frame_host = frames_all.cpu().numpy()
    K = torch.tensor([[1500.0, 0, 960], [0, 1500.0, 720], [0, 0, 1]], dtype=torch.float64, device=dev)
    res = {"card": card(), "cv2": cv2.__version__, "shape": {"frame": [H, W], "views": V, "crop": S}, "results": {}}
    for B in (1, 8, 32):
        ref_kp, q_kp, m0 = workload(rng, B)
        ref = {"keypoints": torch.from_numpy(ref_kp).to(dev), "counts": torch.full((V,), CAP_REF, dtype=torch.int32, device=dev),
               "sizes": torch.tensor([[480, 640]] * V, dtype=torch.int32, device=dev)}
        query = {"keypoints": torch.from_numpy(q_kp).to(dev), "counts": torch.full((B,), CAP_Q, dtype=torch.int32, device=dev)}
        m0_d = torch.from_numpy(m0).to(dev)
        frames = frames_all[None].expand(B, -1, -1)
        frames_host = [frame_host] * B
        legs = {
            "boxes": lambda: detect.boxes_from_matches(ref, query, m0_d, (H, W)),
            "detect": lambda: detect.detect_from_matches(frames, K, ref, query, m0_d, S),
            "host": lambda: host_path(cv2, frames_host, K, ref["keypoints"], query["keypoints"], m0_d, dev),
        }
        for fn in legs.values():                                                 # warm-up of every shape
            fn()
        t = {k: [] for k in legs}
        for _ in range(args.repeats):
            for k, fn in legs.items():
                t[k].append(timed(fn, args.iters if k != "host" else max(1, args.iters // 5)))
        dev_box = detect.boxes_from_matches(ref, query, m0_d, (H, W))["box"].cpu().numpy()
        host_box, _ = host_path(cv2, frames_host, K, ref["keypoints"], query["keypoints"], m0_d, dev)
        res["results"][f"B{B}"] = {k: stats(v) for k, v in t.items()}
        res["results"][f"B{B}"]["boxes_equal"] = int((dev_box == host_box).all(axis=1).sum())
        res["results"][f"B{B}"]["frames"] = B
        print(f"B={B}: " + ", ".join(f"{k} {statistics.median(v):.3f} ms" for k, v in t.items()) +
              f"; boxes equal on {res['results'][f'B{B}']['boxes_equal']}/{B} frames", file=sys.stderr)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
