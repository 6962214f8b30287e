"""The matcher's stage walk (tests/test_matcher_stages_gpu.py: every step of every layer and of the tail against its fp64
reference, the input and hand-off checks, conf entry by entry) at the benchmarked shape and past it, where the code runs in
regimes the small cases never reach:
  * the state kernel's row groups of several 256-row slabs with a shorter tail group (3 at 32 x N 1024 x M 7000 on a 132-SM
    H100; the cap of 8 at 64 x N 2048), which kv_state_reduce combines;
  * the persistent GEMM running 15-70 tiles per CTA, and the score GEMM's 28-59 column tiles meeting in the packed arg-maxes,
    with a partial last tile stored through the 3-D conf tensor map, or plain stores when the conf row is not 16-byte aligned;
  * later chunks on a workspace a larger chunk has just used, the second 16-frame sub-batch of the host-input query pass, and
    conf columns past a chunk's m_pad (conf_fill_tail).
The references run in fp64 on the GPU through ATen.  Each case prints its error / bar table, its wall time and its peak device
memory; the cases free their memory before the next starts."""
import gc
import time

import numpy as np
import pytest
import torch

from onepose_b200 import synthetic
from oracle import gats_spg_oracle as oracle
from tests.test_matcher_stages_gpu import Stages, _attention_live, _module

pytestmark = pytest.mark.gpu

RAGGED = [0, 1, 255, 256, 257, 1024]

CASES = {
    # name: dict(weights, frames, N, objects [(seed, M)], order (frame -> object), nlen, chunk frames, hoist, stop chunk,
    #            query-pass sub-batch, call)
    "bench": dict(frames=32, N=1024, objects=[(0, 7000)]),
    "bench_host": dict(frames=32, N=1024, objects=[(0, 7000)], call="host", piece=1),
    "bench_attention_live_ragged": dict(frames=32, N=1024, objects=[(0, 7000)], weights="attention_live",
                                        nlen=[RAGGED[b % 6] if b < 12 else 1024 - 23 * (b - 12) for b in range(32)]),
    "chunk64": dict(frames=64, N=2048, objects=[(0, 7000)], chunk_frames=64, hoist=False),
    "last_chunk": dict(frames=33, N=1024, objects=[(0, 7000)], chunk=1),
    "shrinking_objects": dict(frames=4, N=512, objects=[(0, 7000), (1, 300)], order=[0, 0, 1, 1], chunk_frames=2, chunk=1,
                              call="objects"),
    "cap_n": dict(frames=2, N=4096, objects=[(2, 1030)]),
    "dense": dict(frames=1, N=2000, objects=[(3, 15000)]),
}


def _free():
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


@pytest.mark.parametrize("name", list(CASES))
def test_stages_at_scale(name):
    c = dict(dict(weights="fixture", order=None, nlen=None, chunk_frames=None, hoist=True, chunk=0, piece=0, call="frames"), **CASES[name])
    _free()
    torch.cuda.reset_peak_memory_stats()
    free0 = torch.cuda.mem_get_info()[0]
    t0 = time.perf_counter()
    hp = dict(synthetic.DEFAULT_HPARAMS)
    sd = synthetic.make_state_dict(0)
    if c["weights"] == "attention_live":
        sd = _attention_live(sd)
    B, N = c["frames"], c["N"]
    host = [synthetic.make_object(seed, M, 8) for seed, M in c["objects"]]
    order = c["order"] or [0] * B
    queries = np.stack([synthetic.make_frame(100 + b, host[order[b]][0], N)[0] for b in range(B)])
    nlen = c["nlen"]
    if nlen is not None:
        for b, n in enumerate(nlen):
            queries[b, :, n:] = 7.0       # garbage past each length: the device must leave zero pad rows
    m = _module(sd, hp, c["hoist"])
    st = None
    try:   # the handle, its workspace and the fp64 references are freed whatever happens
        if c["chunk_frames"]:
            m.set_chunk_frames(c["chunk_frames"])
        dev = lambda a: torch.from_numpy(a).cuda()
        q = dev(queries)
        lengths = None if nlen is None else torch.tensor(nlen, dtype=torch.int32).cuda()
        solo = None
        if c["call"] == "objects":
            ids = [m.add_object(dev(db), dev(lv)) for db, lv in host]
            M_out = max(M for _, M in c["objects"])
            out = {"matches1": torch.empty(B, M_out, dtype=torch.int64, device="cuda")}
            call = lambda: m.match_objects(q, [ids[k] for k in order], lengths=lengths, out=out)
            solo = lambda b: m.match_objects(q[b:b + 1], [ids[order[b]]], lengths=None if lengths is None else lengths[b:b + 1])
        else:
            m.set_object(dev(host[0][0]), dev(host[0][1]), reserve=(B, N))
            if c["call"] == "host":
                M = host[0][0].shape[1]
                pin = dict(pin_memory=True)
                q_pin = torch.from_numpy(queries).pin_memory()
                hout = {"matches0": torch.empty(B, N, dtype=torch.int64, **pin), "matches1": torch.empty(B, M, dtype=torch.int64, **pin),
                        "matching_scores0": torch.empty(B, N, **pin), "matching_scores1": torch.empty(B, M, **pin),
                        "conf_matrix": torch.empty(B, N, M, **pin)}

                def call():
                    r = m.match_frames_host(q_pin, out=hout, lengths=None if nlen is None else torch.tensor(nlen, dtype=torch.int32))
                    return dict(r, conf_matrix=r["conf_matrix"].view(B, N, M))
            else:
                call = lambda: m.match_frames(q, lengths=lengths)
        st = Stages(m, call, oracle.params_from_numpy(sd, torch.float64), hp, queries, [host[k] for k in order], nlen,
                    chunk=c["chunk"], chunk_frames=c["chunk_frames"], piece=c["piece"], piece_frames=16 if c["call"] == "host" else None,
                    solo=solo)
        st.run(c["hoist"])
        torch.cuda.synchronize()
        used = free0 - torch.cuda.mem_get_info()[0]
        peak = torch.cuda.max_memory_allocated()
        seconds = time.perf_counter() - t0
        print(f"\n{name}: {seconds:.1f} s, peak {peak / 2**30:.2f} GiB in torch tensors, {used / 2**30:.2f} GiB of device memory held "
              f"at the end (library workspace included)")
        st.report(name)
    finally:   # a failure's traceback keeps this frame: drop every name that holds the handle or device memory
        st = m = q = lengths = call = solo = out = hout = q_pin = None
        _free()
