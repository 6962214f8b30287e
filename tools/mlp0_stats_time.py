"""Time of the mlp.0 GEMM (EPI_F32_STATS: the InstanceNorm partials come out of its epilogue) and of in_stats_final at the
bench shape (32 frames of N = 1024 queries against M = 7000 points, 8 leaves), from the library's own profile events.

    python tools/mlp0_stats_time.py [--root TREE] [--reps 30]

--root: the source tree whose built library is imported (default: this one), so that two builds can be compared in one
session, alternating.  Prints one JSON line: the median per forward of both entries over --reps profiled forwards, the GPU
and its power limit."""
import argparse
import json
import os
import subprocess
import sys

ap = argparse.ArgumentParser()
ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
ap.add_argument("--reps", type=int, default=30)
args = ap.parse_args()
sys.path.insert(0, os.path.abspath(args.root))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from onepose_b200 import GATsSuperGlue, synthetic  # noqa: E402

B, N, M, L = 32, 1024, 7000, 8
dev = torch.device("cuda", 0)
model = GATsSuperGlue(dict(synthetic.DEFAULT_HPARAMS)).eval()
model.load_state_dict({k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in synthetic.make_state_dict(0).items()})
model = model.to(dev)
db, leaves = synthetic.make_object(0, M, L)
model.set_object(torch.from_numpy(db).to(dev), torch.from_numpy(leaves).to(dev), reserve=(B, N))
q = torch.from_numpy(np.stack([synthetic.make_frame(f, db, N)[0] for f in range(B)])).to(dev)
for _ in range(3):
    model.match_frames(q, return_conf=False)
model.set_profiling(True)
mlp0, stats = [], []
for _ in range(args.reps):
    model.match_frames(q, return_conf=False)
    e = model.get_profile_entry("gemm epi1 ")
    mlp0.append(e["ms"])
    stats.append(model.get_profile_entry("in_stats_final")["ms"])
model.set_profiling(False)
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print(json.dumps({"root": args.root, "mlp0_gemm_ms": float(np.median(mlp0)), "in_stats_final_ms": float(np.median(stats)),
                  "mlp0_launches": e["launches"], "reps": args.reps, "gpu": gpu}))
