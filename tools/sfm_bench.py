"""An object's SfM post-processing on one GPU, on synthetic models of P in {20 000, 60 000} points before filtering, F = 300
images of 2048 key points, D = 256 and max_num_kp3d = 2500, and a dense model: 20 000 points, half of them in clusters under a
millimetre, every point long enough to pass (the greedy merge's worst case among these):
  device      sfm.postprocess from the model's arrays and the padded device features (CUDA events around the call, which ends
              with its results on the device; median, min and max over --repeats), and each kernel's time from one profiled
              call (torch.profiler, CUDA activities);
  host        the numpy model of the same steps (tests/sfm_reference.py), host clock, one run.
The device result is checked against the model's before timing.  Prints a table and one JSON line with the card's name,
power limit and clocks.

    python tools/sfm_bench.py [--repeats 7]"""
import argparse
import json
import os
import re
import statistics
import subprocess
import sys
import time
from collections import defaultdict

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from onepose_b200 import sfm  # noqa: E402
from tests import sfm_reference as sr  # noqa: E402

F, CAP, D, MAX_KP3D = 300, 2048, 256, 2500


def card():
    q = "name,power.limit,clocks.max.sm,clocks.sm,clocks.mem"
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return dict(zip(q.split(","), [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]))
    except Exception as e:            # noqa: BLE001
        return {"name": torch.cuda.get_device_name(0), "note": f"nvidia-smi: {e}"}


def model(P, seed=0, dense=False):
    """P points in and around a 0.3 m box (a quarter outside), track lengths 2..60, 5 % of them in clusters under a millimetre;
    dense: half of them clustered and every length the same, so that all points in the box pass.  Each point observed in 1-3 of
    the F images, the rest of each image's CAP key points without a 3D point."""
    rng = np.random.default_rng(seed)
    corners = np.array([[0, 1, 0], [1, 1, 0], [1, 1, 1], [0, 1, 1], [0, 0, 0], [1, 0, 0], [1, 0, 1], [0, 0, 1]], np.float64) * 0.3
    xyz = rng.uniform(-0.03, 0.33, (P, 3))
    c = rng.choice(P, P // 2 if dense else P // 20, replace=False)
    xyz[c] = xyz[rng.choice(c, len(c))] + rng.normal(scale=3e-4, size=(len(c), 3))
    ids = rng.choice(np.arange(4 * P, dtype=np.int64), P, replace=False)
    lens = np.full(P, 10, np.int64) if dense else rng.integers(2, 61, P).astype(np.int64)
    pid = np.full((F, CAP), -1, np.int64)
    fill = np.zeros(F, np.int64)
    for i in rng.permutation(P):
        for f in rng.choice(F, 1 + int(rng.integers(0, 3)), replace=False):
            if fill[f] < CAP:
                pid[f, fill[f]] = ids[i]
                fill[f] += 1
    for f in range(F):
        pid[f] = pid[f, rng.permutation(CAP)]
    seen = np.isin(ids, pid)
    return ids[seen], xyz[seen], lens[seen], [(f"{f}.png", pid[f]) for f in range(F)], corners


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=7)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sfm_bench needs a GPU")
    info = card()
    rows = []
    for P, dense in ((20000, False), (60000, False), (20000, True)):
        ids, xyz, lens, images, corners = model(P, dense=dense)
        sc, de = sr.features(1, F, D, CAP)
        feats = {"scores": torch.from_numpy(sc).cuda(), "descriptors": torch.from_numpy(de).cuda()}
        t0 = time.perf_counter()
        m = sr.postprocess(ids, xyz, lens, [p for _, p in images], sc, de, corners, MAX_KP3D)
        host_s = time.perf_counter() - t0
        out = sfm.postprocess((ids, xyz, lens), images, feats, corners, MAX_KP3D)
        assert np.array_equal(out["descriptors3d"].cpu().numpy(), m["descriptors3d"]) and np.array_equal(out["idxs"], m["idxs"])
        for _ in range(2):
            sfm.postprocess((ids, xyz, lens), images, feats, corners, MAX_KP3D)
        times = []
        for _ in range(a.repeats):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            sfm.postprocess((ids, xyz, lens), images, feats, corners, MAX_KP3D)
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1))
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            sfm.postprocess((ids, xyz, lens), images, feats, corners, MAX_KP3D)
            torch.cuda.synchronize()
        phases = defaultdict(float)
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA:
                name = ev.name
                k = re.search(r"(\w+_kernel|\w+_f64)\b", name)
                key = ("cub radix sort" if "Radix" in name else "memcpy / memset" if "Memcpy" in name or "Memset" in name else
                       k.group(1) if k else name[:40])
                phases[key] += ev.device_time_total / 1000.0 if hasattr(ev, "device_time_total") else ev.cuda_time_total / 1000.0
        rows.append({"P": P, "dense": dense, "kept": int(len(m["kept_ids"])), "groups": int(len(m["idxs"])), "observations": int(m["idxs"].sum()),
                     "device_ms_median": statistics.median(times), "device_ms_min": min(times), "device_ms_max": max(times),
                     "host_model_s": host_s, "kernel_ms": {k: round(v, 4) for k, v in sorted(phases.items(), key=lambda kv: -kv[1])}})
        r = rows[-1]
        print(f"P={P:6d}{' dense' if dense else '      '} kept={r['kept']:5d} groups={r['groups']:5d} obs={r['observations']:6d}  device {r['device_ms_median']:8.2f} ms "
              f"(min {r['device_ms_min']:.2f}, max {r['device_ms_max']:.2f})  numpy model {host_s:7.2f} s")
        for k, v in r["kernel_ms"].items():
            print(f"    {k:40s} {v:9.3f} ms")
    print(json.dumps({"card": info, "F": F, "cap": CAP, "D": D, "max_num_kp3d": MAX_KP3D, "rows": rows}))


if __name__ == "__main__":
    main()
