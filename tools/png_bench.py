"""Time the device PNG encoder against cv2 on the same frames: 512 x 512 x 3 crops and 1440 x 1920 x 3 frames at F = 1 / 8 / 32.

    python tools/png_bench.py [--reps 15] [--out result.json]

Per case, the medians of --reps calls after a warm-up call:
  encode_ms            CUDA-event time of png.encode (the kernels, on the device frames)
  imwrite_ms           wall clock of png.imwrite: encode, one device-to-host copy of the used bytes and the file writes
  cv2_imencode_ms      host loop of cv2.imencode('.png') over the frames already on the host
  cv2_imwrite_ms       host loop of cv2.imwrite over the frames already on the host
  cv2_imwrite_copy_ms  the same loop after a device-to-host copy of the frames (what a device pipeline pays for cv2)
Frames are smooth (a scene of gradients and edges, as a camera sees) with mild noise.  The card's name, power limit and SM
clock are read in the same run.  Files go to a temporary directory."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import cv2
import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from onepose_b200 import png  # noqa: E402


def frames(F, H, W, seed):
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:H, 0:W]
    out = np.empty((F, H, W, 3), np.uint8)
    for f in range(F):
        base = 96 + 60 * np.sin(x / (37.0 + f)) * np.cos(y / 53.0) + 40 * ((x // 97 + y // 71 + f) % 2)
        for c in range(3):
            out[f, :, :, c] = np.clip(base + 20 * c + rng.normal(0, 2.0, (H, W)), 0, 255).astype(np.uint8)
    return out


def median_ms(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t) * 1e3)
    return float(np.median(ts))


def event_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("png_bench needs a GPU")
    res = {"card": card(), "cases": []}
    with tempfile.TemporaryDirectory() as tmp:
        for H, W in [(512, 512), (1440, 1920)]:
            for F in (1, 8, 32):
                host = frames(F, H, W, F)
                dev = torch.from_numpy(host).cuda()
                buf, sizes = png.encode(dev)
                n = sizes.cpu().numpy()
                for f in range(F):
                    assert buf[f, :n[f]].cpu().numpy().tobytes() == cv2.imencode(".png", host[f])[1].tobytes()
                paths = [os.path.join(tmp, f"{f}.png") for f in range(F)]
                cpaths = [os.path.join(tmp, f"cv2_{f}.png") for f in range(F)]
                r = dict(H=H, W=W, F=F, mean_file_bytes=float(n.mean()))
                r["encode_ms"] = event_ms(lambda: png.encode(dev), args.reps)
                r["imwrite_ms"] = median_ms(lambda: png.imwrite(paths, dev), args.reps)
                reps_host = max(3, args.reps // (4 if H > 600 else 1))
                r["cv2_imencode_ms"] = median_ms(lambda: [cv2.imencode(".png", host[f]) for f in range(F)], reps_host)
                r["cv2_imwrite_ms"] = median_ms(lambda: [cv2.imwrite(cpaths[f], host[f]) for f in range(F)], reps_host)

                def copy_then_cv2():
                    h = dev.cpu().numpy()
                    for f in range(F):
                        cv2.imwrite(cpaths[f], h[f])
                r["cv2_imwrite_copy_ms"] = median_ms(copy_then_cv2, reps_host)
                for f in range(F):
                    assert open(paths[f], "rb").read() == open(cpaths[f], "rb").read()
                res["cases"].append(r)
                print(json.dumps(r), flush=True)
    res["card_after"] = card()
    print(json.dumps({"card": res["card"], "card_after": res["card_after"]}))
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
