"""Colour camera frames to the reference's grey frames, on one GPU, at F in {1, 8, 32} BGR frames of 1440 x 1920:
  kernel        frames.grey_frames on frames already on the device (CUDA events over --iters calls);
  kernel_fp32   the same with the fp32 [F,1,H,W] `/ 255` output as well;
  upload_bgr    the BGR frames from pinned host memory to the device, then grey_frames: what a live loop pays from the camera
                buffer to the device grey frame;
  cvtcolor      the host path it replaces: cv2.cvtColor(COLOR_BGR2GRAY) per frame (NOT the reference's pixels), then the grey
                frames' upload from pinned memory;
  model         the host path that does give the reference's pixels: tests/grey_reference.py's integer formula in numpy per
                frame, then the upload;
  png           the round trip that reproduces the reference's bytes through OpenCV itself: cv2.imencode(".png") at compression
                level 1 and cv2.imdecode(IMREAD_GRAYSCALE) per frame, then the upload.
Host legs are timed by the host clock around work that ends in a device synchronise (2 calls per repeat, 1 for png).  The frames
are waves and hashed noise, shifted per frame: only png's time depends on the content.  The legs alternate inside every repeat;
median, min and max over the repeats.  Every leg's grey frames are checked against the kernel's (cvtcolor's only counted).
Prints a table and one JSON line with the card's name, power limit and clocks.

    python tools/frames_bench.py [--repeats 5] [--iters 20]"""
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
from onepose_b200 import frames  # noqa: E402
from tests import crop_reference as cr  # noqa: E402
from tests import grey_reference as G  # noqa: E402

H, W = 1440, 1920


def card():
    q = "name,power.limit,clocks.max.sm,clocks.sm,clocks.mem"
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return dict(zip(q.split(","), [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]))
    except Exception as e:            # noqa: BLE001
        return {"name": torch.cuda.get_device_name(0), "note": f"nvidia-smi: {e}"}


def events(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def wall(fn, iters):
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(iters):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3 / iters


def stats(xs):
    return {"median_ms": statistics.median(xs), "min_ms": min(xs), "max_ms": max(xs)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--frames", type=int, nargs="+", default=[1, 8, 32])
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("frames_bench needs a GPU")
    import cv2
    dev = torch.device("cuda:0")
    info = {"card": card(), "torch_name": torch.cuda.get_device_name(0), "cv2": cv2.__version__, "H": H, "W": W, "results": {}}
    base = np.stack([cr.synthetic_frame(H, W, c) for c in range(3)], -1)            # waves and noise: a PNG compresses it as a camera frame
    for F in a.frames:
        bgr_host = torch.from_numpy(np.stack([np.roll(base, 7 * f, axis=1) for f in range(F)])).pin_memory()
        bgr_np = bgr_host.numpy()
        bgr_dev = bgr_host.to(dev)
        grey_pinned = torch.empty(F, H, W, dtype=torch.uint8).pin_memory()
        grey_dev = torch.empty(F, H, W, dtype=torch.uint8, device=dev)
        image_dev = torch.empty(F, 1, H, W, dtype=torch.float32, device=dev)
        staging = torch.empty_like(bgr_dev)

        def kernel():
            frames.grey_frames(bgr_dev, out={"grey": grey_dev})

        def kernel_fp32():
            frames.grey_frames(bgr_dev, out={"grey": grey_dev, "image": image_dev}, normalised=True)

        def upload_bgr():
            staging.copy_(bgr_host, non_blocking=True)
            frames.grey_frames(staging, out={"grey": grey_dev})

        def host_leg(convert):
            def run():
                g = grey_pinned.numpy()
                for f in range(F):
                    g[f] = convert(bgr_np[f])
                grey_dev.copy_(grey_pinned)
            return run

        def png(x):
            ok, buf = cv2.imencode(".png", x, [cv2.IMWRITE_PNG_COMPRESSION, 1])
            return cv2.imdecode(buf, cv2.IMREAD_GRAYSCALE)

        legs = {"kernel": (kernel, events), "kernel_fp32": (kernel_fp32, events), "upload_bgr": (upload_bgr, events),
                "cvtcolor": (host_leg(lambda x: cv2.cvtColor(x, cv2.COLOR_BGR2GRAY)), wall), "model": (host_leg(G.grey_from_bgr), wall),
                "png": (host_leg(png), wall)}
        want = frames.grey_frames(bgr_dev).cpu()
        check = {}
        for name, (fn, _) in legs.items():              # warm-up, and each leg's grey frames against the kernel's
            fn()
            torch.cuda.synchronize()
            check[name] = int((grey_dev.cpu() != want).sum())
        assert all(check[k] == 0 for k in check if k != "cvtcolor"), check
        times = {k: [] for k in legs}
        for _ in range(a.repeats):
            for name, (fn, clock) in legs.items():
                iters = a.iters if clock is events else 1 if name == "png" else 2
                times[name].append(clock(fn, iters))
        res = {k: stats(v) for k, v in times.items()}
        res["cvtcolor_pixels_differing"] = check["cvtcolor"]
        res["bytes_bgr"] = F * H * W * 3
        res["kernel_GBps"] = (F * H * W * 4) / (res["kernel"]["median_ms"] * 1e-3) / 1e9
        info["results"][F] = res
    print(f"{info['card']}  (1440 x 1920 BGR frames; median [min-max] ms per call over {a.repeats} repeats)")
    names = ["kernel", "kernel_fp32", "upload_bgr", "cvtcolor", "model", "png"]
    print("F   " + "".join(f"{n:>24}" for n in names))
    for F, r in info["results"].items():
        print(f"{F:<4}" + "".join(f"{r[n]['median_ms']:>9.3f} [{r[n]['min_ms']:.3f}-{r[n]['max_ms']:.3f}]".rjust(24) for n in names))
        print(f"    kernel: {r['kernel_GBps']:.0f} GB/s (BGR read + grey write); cvtColor's grey differs on {r['cvtcolor_pixels_differing']} of "
              f"{F * H * W} pixels")
    print(json.dumps(info))


if __name__ == "__main__":
    main()
