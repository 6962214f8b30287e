"""Several objects per matcher call: one match_objects call against K serial per-object match_frames calls.

    python tools/multi_object_bench.py [--reps 30] [--warmup 5]

The serial route is what a host tracking K objects does without mixed calls: one matcher handle per object (its object set
once), one match_frames call per object per time step.  The mixed route registers the K objects on one handle and matches
all frames in one match_objects call.  The two alternate within each repetition on one stream; each step is timed with CUDA
events and the median is reported.  Configurations: K in {2, 4, 8, 16}, 1 frame per object (tracking) or 4, N = 1024 query
points, M drawn from U[800, 2500] (config 5's range) or M = 7000, return_conf=False.  The matches of both routes are checked to
be equal.  Prints the card name and power limit read in the same run, then one JSON line per configuration.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from onepose_b200 import GATsSuperGlue, synthetic  # noqa: E402


def card():
    """Name and power limit of the device this process runs on, selected by PCI bus id (nvidia-smi does not follow
    CUDA_VISIBLE_DEVICES numbering)."""
    try:
        p = torch.cuda.get_device_properties(torch.cuda.current_device())
        bus = f"{p.pci_domain_id:08X}:{p.pci_bus_id:02X}:{p.pci_device_id:02X}.0"
        q = subprocess.run(["nvidia-smi", "-i", bus, "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        line = q.stdout.strip()
        if q.returncode != 0 or not line:
            raise RuntimeError(q.stderr.strip() or f"no nvidia-smi entry for {bus}")
        return f"{line} (PCI {bus})"
    except Exception as e:      # the tool still measures; the line says why the card is unknown
        return f"{torch.cuda.get_device_name()} (power limit unavailable: {e})"


def module(sd):
    m = GATsSuperGlue(dict(synthetic.DEFAULT_HPARAMS)).eval()
    m.load_state_dict({k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in sd.items()})
    return m.cuda()


def run(K, fpo, m_mode, reps, warmup, sd, N=1024):
    rs = np.random.RandomState(K * 100 + fpo + (7 if m_mode == "7000" else 0))
    Ms = [7000] * K if m_mode == "7000" else [int(x) for x in rs.randint(800, 2501, size=K)]
    objs = [synthetic.make_object(500 + k, M, 8) for k, M in enumerate(Ms)]
    qs = [torch.from_numpy(np.stack([synthetic.make_frame(2000 + k * 10 + f, objs[k][0], N)[0] for f in range(fpo)])).cuda() for k in range(K)]
    serial = []
    for db, lv in objs:
        s = module(sd)
        s.set_object(torch.from_numpy(db).cuda(), torch.from_numpy(lv).cuda())
        serial.append(s)
    mixed = module(sd)
    ids = [mixed.add_object(torch.from_numpy(db).cuda(), torch.from_numpy(lv).cuda()) for db, lv in objs]
    q_all = torch.cat(qs)
    id_list = [ids[k] for k in range(K) for _ in range(fpo)]

    def step_serial():
        return [serial[k].match_frames(qs[k], return_conf=False) for k in range(K)]

    def step_mixed():
        return mixed.match_objects(q_all, id_list, return_conf=False)

    for _ in range(warmup):
        step_serial()
        step_mixed()
    torch.cuda.synchronize()
    ts, tm = [], []
    e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    for _ in range(reps):
        e[0].record()
        outs_s = step_serial()
        e[1].record()
        out_m = step_mixed()
        e[2].record()
        torch.cuda.synchronize()
        ts.append(e[0].elapsed_time(e[1]))
        tm.append(e[1].elapsed_time(e[2]))
    equal = all(torch.equal(outs_s[k]["matches0"], out_m["matches0"][k * fpo:(k + 1) * fpo]) and
                torch.equal(outs_s[k]["matches1"], out_m["matches1"][k * fpo:(k + 1) * fpo, :Ms[k]]) for k in range(K))
    for m in serial + [mixed]:
        m.check_range()
    frames = K * fpo
    ms_s, ms_m = float(np.median(ts)), float(np.median(tm))
    return {"K": K, "frames_per_object": fpo, "M": m_mode, "N": N, "serial_ms_per_step": round(ms_s, 4), "mixed_ms_per_step": round(ms_m, 4),
            "serial_frames_per_s": round(frames / ms_s * 1e3, 1), "mixed_frames_per_s": round(frames / ms_m * 1e3, 1),
            "speedup": round(ms_s / ms_m, 3), "serial_spread_ms": [round(float(np.percentile(ts, 10)), 4), round(float(np.percentile(ts, 90)), 4)],
            "mixed_spread_ms": [round(float(np.percentile(tm, 10)), 4), round(float(np.percentile(tm, 90)), 4)], "matches_equal": bool(equal)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--K", type=int, nargs="*", default=[2, 4, 8, 16])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("multi_object_bench needs a GPU")
    print(f"card: {card()}", flush=True)
    sd = synthetic.make_state_dict(0)
    ok = True
    for m_mode in ("U[800,2500]", "7000"):
        for fpo in (1, 4):
            for K in args.K:
                r = run(K, fpo, m_mode, args.reps, args.warmup, sd)
                ok = ok and r["matches_equal"]
                print(json.dumps(r), flush=True)
    if not ok:
        raise SystemExit("the two routes gave different matches")


if __name__ == "__main__":
    main()
