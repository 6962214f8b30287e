"""Extractor time per batch at 8 x 512 x 512 for this tree and another checkout of the project (e.g. the commit before the
range guard), alternated in separate processes, and whether their outputs are bit-identical.

    python tools/sp_range_guard_time.py --other /path/to/other/checkout [--rounds 4] [--iters 50]

Each measurement: forward_padded on the benchmarked images and weights, 10 warm-up calls, then `iters` calls between two CUDA
events.  Prints the card's name and power limit with the numbers."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CHILD = r"""
import sys, json
sys.path.insert(0, sys.argv[1])
import numpy as np, torch
from onepose_b200 import SuperPoint, synthetic
sp = SuperPoint(synthetic.SUPERPOINT_CONF).eval()
sp.load_state_dict({k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in synthetic.make_superpoint_state_dict(0, 4.0).items()})
sp = sp.cuda()
img = torch.from_numpy(np.stack([synthetic.make_image(100 + i, 512, 512) for i in range(8)], 0)).cuda()
for _ in range(10):
    out = sp.forward_padded(img)
torch.cuda.synchronize()
a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
iters = int(sys.argv[3])
a.record()
for _ in range(iters):
    out = sp.forward_padded(img)
b.record()
torch.cuda.synchronize()
n = out["counts"].tolist()
np.savez(sys.argv[2], counts=np.array(n), **{f"{k}_{i}": (out[k][i, :c] if k != "descriptors" else out[k][i, :, :c]).cpu().numpy()
                                             for k in ("keypoints", "scores", "descriptors") for i, c in enumerate(n)})
print(json.dumps({"ms": a.elapsed_time(b) / iters}))
"""


def run(tree, path, iters):
    r = subprocess.run([sys.executable, "-c", CHILD, tree, path, str(iters)], capture_output=True, text=True, check=True)
    return json.loads(r.stdout.strip().splitlines()[-1])["ms"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--other", required=True, help="root of the other checkout (built)")
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--iters", type=int, default=50)
    a = ap.parse_args()
    import numpy as np
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    times = {"this": [], "other": []}
    with tempfile.TemporaryDirectory() as tmp:
        for r in range(a.rounds):
            for name, tree in (("other", os.path.abspath(a.other)), ("this", ROOT)) if r % 2 == 0 else (("this", ROOT), ("other", os.path.abspath(a.other))):
                times[name].append(run(tree, os.path.join(tmp, f"{name}.npz"), a.iters))
        x, y = np.load(os.path.join(tmp, "this.npz")), np.load(os.path.join(tmp, "other.npz"))
        identical = sorted(x.files) == sorted(y.files) and all(np.array_equal(x[k], y[k]) for k in x.files)
    print(json.dumps({"card": card, "ms_per_batch": {k: [round(t, 4) for t in v] for k, v in times.items()},
                      "median": {k: float(np.median(v)) for k, v in times.items()}, "bit_identical": identical}))


if __name__ == "__main__":
    main()
