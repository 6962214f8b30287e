"""Time the 2D annotation files of an object: sfm.assign_matrices / save_anno_2d on the device against the reference rule's
host model (tests/anno2d_reference.py: the same dict walk and json.dump as save_2d_anno) on the same host.

    python tools/anno2d_bench.py [--F 300] [--n 2048] [--D 256] [--host-images 3]

Prints one JSON line: the card and its power limit, device pairs and text time (CUDA events), the device-to-host copy and
file writes, and the host model's time per image scaled to F images."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from onepose_b200 import sfm  # noqa: E402
from tests import anno2d_reference as ar  # noqa: E402
from tests.test_anno2d_gpu import dense_case  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--F", type=int, default=300)
    ap.add_argument("--n", type=int, default=2048)
    ap.add_argument("--D", type=int, default=256)
    ap.add_argument("--host-images", type=int, default=3)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    dev = torch.device("cuda:0")
    images, result, (kp, de, sc) = dense_case(1, a.F, a.n, 12 * a.n, D=a.D)
    feats = {"keypoints": torch.from_numpy(kp).to(dev), "descriptors": torch.from_numpy(de).to(dev), "scores": torch.from_numpy(sc).to(dev)}
    ev = lambda: torch.cuda.Event(enable_timing=True)  # noqa: E731
    sfm.assign_matrices(result, images, feats)          # warm-up
    e0, e1 = ev(), ev()
    e0.record()
    sfm.assign_matrices(result, images, feats)
    e1.record()
    torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as tmp:
        paths = [os.path.join(tmp, n) for n, _ in images]
        sfm.save_anno_2d(os.path.join(tmp, "anno"), paths, result, images, feats)   # warm-up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        index = sfm.save_anno_2d(os.path.join(tmp, "anno"), paths, result, images, feats)
        torch.cuda.synchronize()
        t_save = time.perf_counter() - t0
        size = sum(os.path.getsize(x["anno_file"]) for x in index)
    gmap = ar.group_map(result["group_ids"], result["group_offsets"])
    t0 = time.perf_counter()
    with tempfile.TemporaryDirectory() as tmp:
        for f in range(a.host_images):
            n = len(images[f][1])
            with open(os.path.join(tmp, f"{f}.json"), "w") as fh:
                fh.write(ar.anno_text(kp[f, :n], de[f, :, :n], sc[f, :n], ar.assign_pairs(images[f][1], gmap)))
    t_host = (time.perf_counter() - t0) / a.host_images * a.F
    print(json.dumps({"card": card, "F": a.F, "n": a.n, "D": a.D, "text_bytes": size, "assign_matrices_ms": e0.elapsed_time(e1),
                      "save_anno_2d_s": t_save, "host_model_s_scaled": t_host}))


if __name__ == "__main__":
    main()
