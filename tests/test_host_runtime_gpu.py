"""Host runtime shared by the matcher and extractor handles (csrc/host_util.cuh): launch accounting and the profiling timeline,
the error codes of weight loading and of create, the create-error message both handle kinds report, and the return
of every device buffer when a handle is destroyed.  Launch counts and FLOPs are pinned to the values the handles have always
reported: a change to the host code must not move them."""
import ctypes as C
import gc

import numpy as np
import pytest
import torch

from onepose_b200 import GATsSuperGlue, SuperPoint, _lib, synthetic

pytestmark = pytest.mark.gpu

OPB_E_INVALID, OPB_E_STATE = -1, -3

# matcher: one object (M = 300, 8 leaves), 6 frames of N = 200 in chunks of 4 + 2, hoisting on
MATCHER_LAUNCHES = [160, 150]                  # the first call also runs the object prologue
MATCHER_EPI1_FLOPS = [11796480000.0, 11639193600.0]
# extractor: forward_padded of 2 images of 64 x 80
EXTRACTOR_LAUNCHES = 20            # DESIGN §5.5
EXTRACTOR_NAMES = ["sp_conv1a", "conv1b", "sp_pool2x2", "conv2a", "conv2b", "sp_pool2x2", "conv3a", "conv3b", "sp_pool2x2", "conv4a",
                   "conv4b", "convPa|convDa", "convPb", "convDb", "sp_scores", "sp_nms", "sp_count", "sp_compact", "sp_emit", "sp_sample"]
CONVS = {   # name: (stage, C_out as packed, taps, C_in)
    "conv1b": (0, 64, 9, 64), "conv2a": (1, 64, 9, 64), "conv2b": (1, 64, 9, 64), "conv3a": (2, 128, 9, 64),
    "conv3b": (2, 128, 9, 128), "conv4a": (3, 128, 9, 128), "conv4b": (3, 128, 9, 128), "convPa|convDa": (3, 512, 9, 128),
    "convPb": (3, 128, 1, 256), "convDb": (3, 256, 1, 256),
}


def _matcher(seed=0):
    m = GATsSuperGlue(dict(synthetic.DEFAULT_HPARAMS)).eval()
    m.load_state_dict({k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in synthetic.make_state_dict(seed).items()})
    return m.cuda()


def _extractor():
    m = SuperPoint(synthetic.SUPERPOINT_CONF).eval()
    m.load_state_dict({k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in synthetic.make_superpoint_state_dict(0, 4.0).items()})
    return m.cuda()


def _set_object(m, seed, M, L=8):
    db, leaves = synthetic.make_object(seed, M, L)
    m.set_object(torch.from_numpy(db).cuda(), torch.from_numpy(leaves).cuda())
    return db


def _queries(db, B, N):
    return torch.from_numpy(np.stack([synthetic.make_frame(f, db, N)[0] for f in range(B)], 0)).cuda()


# ----------------------------------------------------------------------------- launch accounting and profiles
def test_matcher_launch_accounting():
    m = _matcher()
    m.set_chunk_frames(4)
    q = _queries(_set_object(m, 1, 300), 6, 200)
    m.set_profiling(True)
    counts = []
    for i in range(2):
        m.match_frames(q)
        torch.cuda.synchronize()
        counts.append(m.launch_count())
        assert m.get_profile_entry("")["launches"] == counts[-1]
        prof, gemm = m.get_profile(), m.get_profile_entry("gemm")
        assert prof["gemm_launches"] == gemm["launches"] > 0
        assert prof["gemm_flops"] == gemm["flops"]
        assert prof["total_ms"] >= gemm["ms"] > 0
        assert m.get_profile_entry("gemm epi1 ")["flops"] == MATCHER_EPI1_FLOPS[i]
    assert counts == MATCHER_LAUNCHES
    m.set_profiling(False)
    m.match_frames(q)
    torch.cuda.synchronize()
    assert m.launch_count() == counts[1]             # profiling does not change what is launched


def test_extractor_launch_accounting():
    sp = _extractor()
    B, H, W = 2, 64, 80
    img = torch.from_numpy(np.stack([synthetic.make_image(i, H, W) for i in (1, 2)], 0)).cuda()     # [B, 1, H, W]
    sp.forward_padded(img, cap=256)                 # creates the handle
    sp.set_profiling(True)
    sp.forward_padded(img, cap=256)
    torch.cuda.synchronize()
    assert sp.launch_count() == EXTRACTOR_LAUNCHES
    prof = sp.get_profile()
    names = [p[0] for p in prof]
    assert names == EXTRACTOR_NAMES
    assert all(ms >= 0 for _, ms, _ in prof)
    for name, _, flops in prof:
        if name in CONVS:
            s, cout, taps, cin = CONVS[name]
            assert flops == 2.0 * B * (H >> s) * (W >> s) * cout * taps * cin, name
        else:
            assert flops == 0.0, name
    assert sorted(n for n in names if n in CONVS) == sorted(CONVS)


# ----------------------------------------------------------------------------- error paths
def _handles():
    lib = _lib.load()
    hp = synthetic.DEFAULT_HPARAMS
    cfg = _lib.OpbConfig(256, 4, float(hp["scale_factor"]), float(hp["match_threshold"]), int(bool(hp["include_self"])),
                         int(bool(hp["additional"])), int(bool(hp["with_linear_transform"])), 0)
    m = C.c_void_p()
    assert lib.opb_create(C.byref(cfg), C.byref(m)) == 0
    c = synthetic.SUPERPOINT_CONF
    scfg = _lib.OpbSpConfig(256, int(c["nms_radius"]), 0.005, int(c["max_keypoints"]), 4, 1, 0)
    s = C.c_void_p()
    assert lib.opb_sp_create(C.byref(scfg), C.byref(s)) == 0
    return lib, m, s


def _load(lib, fn, h, sd, skip=None, resize=None):
    for k, v in sd.items():
        if k == skip:
            continue
        a = np.ascontiguousarray(v, np.float32).ravel()
        if k == resize:
            a = a[:-1].copy()
        assert fn(h, k.encode(), a.ctypes.data, a.size) == 0


def test_weight_errors():
    sd, ssd = synthetic.make_state_dict(0), synthetic.make_superpoint_state_dict(0, 4.0)
    for case in ("missing", "size"):
        lib, m, s = _handles()
        try:
            key, skey = "gnn.layers.4.attn.merge.bias", "conv3b.weight"
            arg = {"skip": key} if case == "missing" else {"resize": key}
            sarg = {"skip": skey} if case == "missing" else {"resize": skey}
            _load(lib, lib.opb_load_weight, m, sd, **arg)
            _load(lib, lib.opb_sp_load_weight, s, ssd, **sarg)
            want = OPB_E_STATE if case == "missing" else OPB_E_INVALID
            assert lib.opb_finalize_weights(m) == want
            assert key.encode() in lib.opb_last_error(m)
            assert lib.opb_sp_finalize_weights(s) == want
            assert skey.encode() in lib.opb_sp_last_error(s)
        finally:
            lib.opb_destroy(m)
            lib.opb_sp_destroy(s)


def test_each_failed_create_leaves_its_message_for_both_handle_kinds():
    """Calls without a handle share one message per thread: opb_last_error(NULL) and opb_sp_last_error(NULL) both give the
    message of the last failed create, whichever kind it was."""
    lib = _lib.load()
    h = C.c_void_p()

    def refused(create, cfg, text):
        assert create(C.byref(cfg), C.byref(h)) == OPB_E_INVALID
        assert text in lib.opb_last_error(None) and text in lib.opb_sp_last_error(None)

    refused(lib.opb_create, _lib.OpbConfig(256, 4, 0.0, 0.2, 1, 1, 0, 0), b"scale_factor")
    refused(lib.opb_sp_create, _lib.OpbSpConfig(128, 4, 0.005, -1, 4, 1, 0), b"descriptor_dim")
    refused(lib.opb_create, _lib.OpbConfig(128, 4, 1.0, 0.2, 1, 1, 0, 0), b"descriptor_dim")
    refused(lib.opb_sp_create, _lib.OpbSpConfig(256, 4, 0.005, 0, 4, 1, 0), b"max_keypoints")


# ----------------------------------------------------------------------------- memory is returned
def _free_bytes():
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return torch.cuda.mem_get_info()[0]


def _fill_handles(M, frames, N, H, W):
    """A matcher with weights, two registered objects (one removed again), a workspace reserved for `frames` frames of N + M
    rows and a host-buffer call; an extractor that has run a batch of 4 images H x W.  No torch tensor outlives the call."""
    m = _matcher()
    db, leaves = synthetic.make_object(1, M)
    m.set_object(torch.from_numpy(db).cuda(), torch.from_numpy(leaves).cuda(), reserve=(frames, N))
    ids = [m.add_object(*(torch.from_numpy(a).cuda() for a in synthetic.make_object(s, Ms))) for s, Ms in ((2, M // 2), (3, M))]
    m.remove_object(ids[0])
    m.match_frames_host(_queries(db, 2, N).cpu().pin_memory())
    sp = _extractor()
    sp.forward_padded(torch.from_numpy(np.stack([synthetic.make_image(i, H, W) for i in range(4)], 0)).cuda(), cap=1024)
    torch.cuda.synchronize()
    return m, sp


def test_destroy_returns_device_memory():
    # run every kernel once first, so that memory taken by lazy module loading is not counted as held by the handles
    m, sp = _fill_handles(300, 2, 200, 64, 80)
    del m, sp
    for r in range(3):
        before = _free_bytes()
        m, sp = _fill_handles(7000, 32, 1024, 480, 640)
        alive = _free_bytes()
        held = before - alive
        assert held > 1.5e9, f"round {r}: the handles hold only {held / 1e9:.2f} GB"
        del m, sp
        after = _free_bytes()
        print(f"round {r}: handles held {held / 1e9:.3f} GB, destroy returned {(after - alive) / 1e9:.3f} GB")
        assert after - alive >= 0.97 * held, f"round {r}: {held / 1e9:.3f} GB held, {(after - alive) / 1e9:.3f} GB returned"


def test_create_rejects_negative_device():
    lib = _lib.load()
    hp = synthetic.DEFAULT_HPARAMS
    cfg = _lib.OpbConfig(256, 4, float(hp["scale_factor"]), float(hp["match_threshold"]), 1, 1, 0, -1)
    h = C.c_void_p()
    assert lib.opb_create(C.byref(cfg), C.byref(h)) == OPB_E_INVALID
    scfg = _lib.OpbSpConfig(256, 4, 0.005, -1, 4, 1, -1)
    assert lib.opb_sp_create(C.byref(scfg), C.byref(h)) == OPB_E_INVALID
