"""Interleaved A/B of the library's debug switches at the bench configuration (B=32, 1024 x 7000): the settings alternate
step by step so that clock / thermal drift under the power cap cancels.  Prints mean step time per setting and the in-stream
time of selected kernels.     python tools/ab_test.py [pairs]"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from onepose_b200 import GATsSuperGlue, _lib, synthetic  # noqa: E402

lib = _lib.load()
dev = torch.device("cuda", 0)
hp = dict(synthetic.DEFAULT_HPARAMS)
sd = synthetic.make_state_dict(0)
model = GATsSuperGlue(hp).eval()
model.load_state_dict({k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in sd.items()})
model = model.to(dev)
B, N, M = 32, 1024, 7000
db, leaves = synthetic.make_object(0, M, 8)
q = [torch.from_numpy(np.stack([synthetic.make_frame(1000 * s + f, db, N)[0] for f in range(B)], 0)).to(dev) for s in range(4)]
model.set_object(torch.from_numpy(db).to(dev), torch.from_numpy(leaves).to(dev), reserve=(B, N))
conf = torch.empty(B, N, M, device=dev)
m0 = torch.empty(B, N, dtype=torch.int64, device=dev)
m1 = torch.empty(B, M, dtype=torch.int64, device=dev)
s0 = torch.empty(B, N, device=dev)
s1 = torch.empty(B, M, device=dev)
st = torch.cuda.current_stream(dev).cuda_stream


def step(i):
    _lib.check(lib.opb_forward(model._handle, q[i % 4].data_ptr(), None, B, N, m0.data_ptr(), m1.data_ptr(), s0.data_ptr(), s1.data_ptr(),
                               conf.data_ptr(), st), model._handle)


SWITCHES = {
    "pdl": lambda v: lib.opb_debug_set_pdl(v),
    "kv_2pass": lambda v: lib.opb_debug_set_kv_passes(model._handle, 2 if v else 3),
}
pairs = int(sys.argv[1]) if len(sys.argv) > 1 else 12
for w in range(30):          # reach the power-capped steady state first
    step(w)
torch.cuda.synchronize()
for name, setter in SWITCHES.items():
    t = {0: [], 1: []}
    for it in range(2 * pairs):
        v = it & 1
        setter(v)
        step(it)             # one untimed step under the new setting (prologue / first-use effects)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); step(it + 1); e1.record()
        torch.cuda.synchronize()
        t[v].append(e0.elapsed_time(e1))
    setter(1)
    a, b = np.array(t[0]), np.array(t[1])
    print(f"{name:12s} off {a.mean():6.3f} +- {a.std():.3f} ms   on {b.mean():6.3f} +- {b.std():.3f} ms   on/off {b.mean() / a.mean():.4f}", flush=True)
    # per-kernel view
    prof = {}
    for v in (0, 1):
        setter(v)
        step(0)
        model.set_profiling(True)
        acc = {}
        for r in range(3):
            step(r)
            for k in ("gemm epi1 ", "gemm epi10 n256 k768", "gemm epi9 ", "gemm epi2 ", "gats_aggregate", "kv_state_h"):
                acc[k] = acc.get(k, 0.0) + model.get_profile_entry(k)["ms"] / 3
            acc["total"] = acc.get("total", 0.0) + model.get_profile()["total_ms"] / 3
        model.set_profiling(False)
        prof[v] = acc
    setter(1)
    print("             " + "  ".join(f"{k.strip()[:22]}: {prof[0][k]:.3f}->{prof[1][k]:.3f}" for k in prof[0]), flush=True)
