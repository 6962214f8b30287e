"""Time the device PNG reader against the host loop on the same files: cv2-written 512 x 512 x 3 crops at F = 1 / 8 / 32 / 128 and
1440 x 1920 x 3 frames at F = 1 / 8 / 32, with the default call (SUB rows) and with IMWRITE_PNG_COMPRESSION 9 (adaptive filters,
Paeth rows among them).

    python tools/png_read_bench.py [--reps 9] [--out result.json]

Per case, medians of --reps calls after a warm-up call:
  decode_ms       CUDA-event time of png.decode (grey, normalised) from device-resident bytes
  inflate_ms      of which the chunk walk and inflate kernels, and
  unfilter_ms     the unfilter and convert kernels (torch.profiler kernel times, in a separate pass)
  imread_ms       wall clock of png.imread(paths, IMREAD_GRAYSCALE, normalised=True): file reads, one copy, decode, status read
  host_ms         the host loop: cv2.imread(IMREAD_GRAYSCALE), upload and / 255 per file, then a device synchronise
The card's name, power limit and SM clock are read in the same run.  Files go to a temporary directory."""
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
    """Smooth scenes of gradients and edges with mild noise, as a camera sees."""
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
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        torch.cuda.synchronize()
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


def kernel_ms(fn, reps):
    """Median per call of the reader's kernels' device time: (chunks + inflate, rows + chain + convert)."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    inflate = unfilter = 0.0
    for e in prof.key_averages():
        t = e.device_time_total / 1e3 / reps if hasattr(e, "device_time_total") else e.cuda_time_total / 1e3 / reps
        if "png_chunks_kernel" in e.key or "png_inflate_kernel" in e.key:
            inflate += t
        elif any(k in e.key for k in ("png_rows_kernel", "png_chain_kernel", "png_convert_kernel")):
            unfilter += t
    return inflate, unfilter


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("png_read_bench needs a GPU")
    res = {"card": card(), "cases": []}
    cases = [(512, 512, F) for F in (1, 8, 32, 128)] + [(1440, 1920, F) for F in (1, 8, 32)]
    with tempfile.TemporaryDirectory() as tmp:
        for H, W, F in cases:
            fr = frames(F, H, W, seed=H + F)
            for call, params in (("default", []), ("compression9", [cv2.IMWRITE_PNG_COMPRESSION, 9])):
                paths = [os.path.join(tmp, f"{H}_{F}_{call}_{i}.png") for i in range(F)]
                blobs = []
                for p, f in zip(paths, fr):
                    cv2.imwrite(p, f, params)
                    with open(p, "rb") as fh:
                        blobs.append(fh.read())
                offsets = np.zeros(F + 1, np.int64)
                offsets[1:] = np.cumsum([len(b) for b in blobs])
                data = torch.from_numpy(np.frombuffer(b"".join(blobs), np.uint8).copy()).cuda()
                offs = torch.from_numpy(offsets).cuda()
                dec = lambda: png.decode(data, offs, H, W, cv2.IMREAD_GRAYSCALE, normalised=True)  # noqa: E731
                grey, image, status = dec()
                want = np.stack([cv2.imread(p, cv2.IMREAD_GRAYSCALE) for p in paths])
                assert (status.cpu() == 0).all() and np.array_equal(grey.cpu().numpy(), want), (H, F, call)

                def host():
                    for p in paths:
                        g = torch.from_numpy(cv2.imread(p, cv2.IMREAD_GRAYSCALE)).cuda()
                        g.float() / 255
                r = {"H": H, "W": W, "F": F, "call": call, "mb": round(offsets[-1] / 1e6, 2),
                     "decode_ms": event_ms(dec, args.reps)}
                r["inflate_ms"], r["unfilter_ms"] = kernel_ms(dec, args.reps)
                r["imread_ms"] = median_ms(lambda: png.imread(paths, cv2.IMREAD_GRAYSCALE, normalised=True), args.reps)
                r["host_ms"] = median_ms(host, args.reps)
                r = {k: round(v, 3) if isinstance(v, float) else v for k, v in r.items()}
                res["cases"].append(r)
                print(json.dumps(r), flush=True)
    res["card_after"] = card()
    print(json.dumps({"card": res["card"], "card_after": res["card_after"]}))
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
