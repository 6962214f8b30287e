"""Drop-in ``GATsSuperGlue`` for the reference's 2D-3D matching forward.

Mirrors reference ``src/models/GATsSPG_architectures/GATs_SuperGlue.py:143-241``:
same constructor (``hparams`` mapping), same parameter names / shapes (so a
reference ``state_dict`` -- or the ``matcher.*`` slice of a Lightning checkpoint
-- loads verbatim, dead ``kenc_*`` / ``bin_score`` included), same
``forward(data) -> (pred, conf_matrix)`` contract, including the bare-dict early
return for empty inputs (:195-203) and ``pred`` = batch element 0 (:232-237).

The arithmetic runs in hand-written sm_90a CUDA kernels behind the C ABI of
``include/onepose_b200.h``; PyTorch only owns device memory and the stream.
There is no CPU path: tensors must live on a CUDA device.
"""
from __future__ import annotations

import ctypes as C
from copy import deepcopy

import torch
import torch.nn as nn

from . import _lib

GNN_LAYERS = ["GATs", "self", "cross"] * 4          # GATs_SuperGlue.py:162
_CURRENT = -1                                       # key of the current object (set_object) in _objects; add_object's ids are >= 0


class _GATsParams(nn.Module):
    """Parameter holder of GraphAttentionLayer (reference GATs.py:25-28)."""

    def __init__(self, dim):
        super().__init__()
        self.W = nn.Parameter(torch.empty(dim, dim))
        nn.init.xavier_normal_(self.W.data, gain=1.414)
        self.a = nn.Parameter(torch.empty(2 * dim, 1))
        nn.init.xavier_normal_(self.a.data, gain=1.414)


class _AttnParams(nn.Module):
    """MultiHeadedAttention parameters (GATs_SuperGlue.py:85-91): proj.* start as copies of merge."""

    def __init__(self, dim):
        super().__init__()
        self.merge = nn.Conv1d(dim, dim, kernel_size=1)
        self.proj = nn.ModuleList([deepcopy(self.merge) for _ in range(3)])


def _mlp_params(channels):
    """MLP (GATs_SuperGlue.py:116-128): convs sit at Sequential indices 0, 3, 6, ... ."""
    mods = {}
    for i in range(1, len(channels)):
        mods[str(3 * (i - 1))] = nn.Conv1d(channels[i - 1], channels[i], kernel_size=1, bias=True)
    return nn.ModuleDict(mods)


class _PropagationParams(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.attn = _AttnParams(dim)
        self.mlp = _mlp_params([2 * dim, 2 * dim, dim])
        nn.init.constant_(self.mlp["3"].bias, 0.0)              # GATs_SuperGlue.py:109


class _KencParams(nn.Module):
    """Dead at inference (never called in the reference forward) but part of the checkpoint."""

    def __init__(self, inp_dim, feature_dim, layers):
        super().__init__()
        chans = [inp_dim] + list(layers) + [feature_dim]
        self.encoder = _mlp_params(chans)
        nn.init.constant_(self.encoder[str(3 * (len(chans) - 2))].bias, 0.0)


class _GnnParams(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.layers = nn.ModuleList(
            [_GATsParams(dim) if i % 3 == 0 else _PropagationParams(dim) for i in range(len(GNN_LAYERS))])


def _out_view(out, name, shape, dtype, dev):
    """A result tensor of `shape`: a view of the caller's flat buffer out[name] if given, else a fresh allocation."""
    n = 1
    for d in shape:
        n *= int(d)
    if out is not None and name in out:
        t = out[name]
        if t.dtype != dtype or t.device != dev or t.numel() < n or not t.is_contiguous():
            raise ValueError(f"out['{name}'] must be a contiguous {dtype} buffer on {dev} with at least {n} elements")
        return t.view(-1)[:n].view(shape)
    return torch.empty(shape, dtype=dtype, device=dev)


class GATsSuperGlue(nn.Module):
    def __init__(self, hparams):
        super().__init__()
        self.hparams = hparams
        self.match_type = hparams["match_type"]
        d = hparams["descriptor_dim"]
        self.kenc_2d = _KencParams(3, d, hparams["keypoints_encoder"])
        self.kenc_3d = _KencParams(4, d, hparams["keypoints_encoder"])
        self.gnn = _GnnParams(d)
        self.final_proj = nn.Conv1d(d, d, kernel_size=1, bias=True)
        self.register_parameter("bin_score", nn.Parameter(torch.tensor(1.0)))
        self._lib = _lib.load()        # raises if the CUDA library is not built
        self._handle = None
        self._handle_device = None
        self._weights_key = None
        self._obj_key = None           # (data_ptr, _version, shape) of the caller tensors the current object was packed from
        self._obj_ref = None           # strong reference to those tensors: their storage cannot be recycled under the key
        self._obj_copy = None          # private copy of the packed object (exact comparison on a key miss)
        self._chunk_frames = 0
        self._hoist = True
        self._objects = {}             # M of each registered object by id (add_object), and of the current one under _CURRENT
        self.last_batched = None       # batched outputs of the last forward (all B frames)

    # ------------------------------------------------------------------ handle / weights
    def __del__(self):
        try:
            if self._handle is not None:
                self._lib.opb_destroy(self._handle)
        except Exception:
            pass

    def _ensure_handle(self, device: torch.device):
        if self._handle is not None and self._handle_device == device:
            return
        if self._handle is not None:
            self._lib.opb_destroy(self._handle)
            self._handle = None
        hp = self.hparams
        cfg = _lib.OpbConfig(int(hp["descriptor_dim"]), 4, float(hp["scale_factor"]), float(hp["match_threshold"]),
                             int(bool(hp["include_self"])), int(bool(hp["additional"])),
                             int(bool(hp["with_linear_transform"])), device.index or 0)
        h = C.c_void_p()
        _lib.check(self._lib.opb_create(C.byref(cfg), C.byref(h)))
        self._handle, self._handle_device = h, device
        self._weights_key = self._obj_key = self._obj_ref = self._obj_copy = None
        self._objects = {}             # objects live on the handle
        if self._chunk_frames:
            _lib.check(self._lib.opb_set_chunk_frames(self._handle, self._chunk_frames), self._handle)
        if not self._hoist:
            _lib.check(self._lib.opb_set_hoist(self._handle, 0), self._handle)

    def _sync_weights(self):
        key = tuple((n, p.data_ptr(), p._version) for n, p in self.named_parameters())
        if key == self._weights_key:
            return
        for name, p in self.named_parameters():
            w = p.detach().to("cpu", torch.float32).contiguous()
            _lib.check(self._lib.opb_load_weight(self._handle, name.encode(), w.data_ptr(), w.numel()), self._handle)
        _lib.check(self._lib.opb_finalize_weights(self._handle), self._handle)
        self._weights_key = key
        self._obj_key = self._obj_ref = self._obj_copy = None
        self._objects.pop(_CURRENT, None)      # a weight reload keeps the registered objects, not the current one

    def set_hoist(self, enable: bool):
        """Evaluate the frame-invariant GNN layers once per call (default) or per frame like the reference."""
        self._hoist = bool(enable)
        if self._handle is not None:
            _lib.check(self._lib.opb_set_hoist(self._handle, int(self._hoist)), self._handle)

    def set_chunk_frames(self, frames: int):
        """Frames pushed through the GNN together (workspace-size knob of the C ABI)."""
        if self._handle is not None:
            _lib.check(self._lib.opb_set_chunk_frames(self._handle, int(frames)), self._handle)
        self._chunk_frames = int(frames)

    # ------------------------------------------------------------------ fast API
    def set_object(self, descriptors3d_db: torch.Tensor, descriptors2d_db: torch.Tensor, reserve=None):
        """Upload per-object constants once (what inference.py:113-130 builds per sequence).
        descriptors3d_db [256, M], descriptors2d_db [256, M*L], CUDA fp32.  reserve = (frames, N): size the
        workspace now instead of on the first call."""
        d3, d2, M, L, st = self._prepare_object(descriptors3d_db, descriptors2d_db)
        _lib.check(self._lib.opb_set_object(self._handle, d3.data_ptr(), d2.data_ptr(), M, L, st), self._handle)
        self._objects[_CURRENT] = M
        self._obj_key = self._obj_ref = self._obj_copy = None
        if reserve is not None:
            _lib.check(self._lib.opb_reserve_workspace(self._handle, int(reserve[0]), int(reserve[1])), self._handle)

    def _prepare_object(self, descriptors3d_db: torch.Tensor, descriptors2d_db: torch.Tensor):
        """(d3, d2, M, L, stream) of an object to load: fp32 contiguous CUDA tensors, with the handle on their device and its
        weights current."""
        d3 = descriptors3d_db.float().contiguous()
        d2 = descriptors2d_db.float().contiguous()
        if not d3.is_cuda:
            raise RuntimeError("onepose_b200 has no CPU path: tensors must be on a CUDA device")
        self._ensure_handle(d3.device)
        self._sync_weights()
        M = d3.shape[1]
        if M == 0 or d2.shape[1] % M:
            raise ValueError(f"descriptors2d_db has {d2.shape[1]} columns, not a multiple of M={M}")
        return d3, d2, M, d2.shape[1] // M, torch.cuda.current_stream(d3.device).cuda_stream

    def _require_object(self):
        if self._handle is None or _CURRENT not in self._objects:
            raise RuntimeError("no object set: call set_object(descriptors3d_db, descriptors2d_db) first (or use forward(data))")

    def _check_device(self, q: torch.Tensor):
        """The handle's work runs on its own device, so the queries (and every buffer of the call) must live there."""
        if q.device != self._handle_device:
            raise ValueError(f"descriptors2d_query is on {q.device}, the matcher's objects and workspace are on {self._handle_device}")

    def match_frames(self, descriptors2d_query: torch.Tensor, return_conf: bool = True, lengths: torch.Tensor | None = None,
                     out: dict | None = None):
        """B frames of the current object.  descriptors2d_query [B, 256, N] CUDA fp32; lengths (optional) CUDA int32 [B] =
        valid query points per frame (ragged batch: SuperPoint yields a different count per frame).
        Returns dict of batched tensors (matches0 [B,N] int64, ..., conf_matrix [B,N,M] or None).  Asynchronous: no host
        synchronisation; a range violation (see check_range) turns the call's matches into -1.
        out (optional): flat CUDA buffers {"matches0", "matches1": int64, "matching_scores0", "matching_scores1", "conf_matrix":
        fp32} at least as large as the results; the returned tensors are views of them (a serving loop allocates once)."""
        self._require_object()
        self._check_device(descriptors2d_query)
        q = descriptors2d_query.float().contiguous()
        B, _, N = q.shape
        return self._match(q, B, N, self._objects[_CURRENT], return_conf, lengths, out,
                           lambda lens, *res: self._lib.opb_forward(self._handle, q.data_ptr(), lens, B, N, *res))

    def _match(self, q, B, N, M, return_conf, lengths, out, call):
        """match_frames / match_objects for B frames of N queries, M-wide rows: the result tensors (views of `out` or fresh),
        `lengths` on the device, then call(lengths, matches0, matches1, scores0, scores1, conf, stream), all pointers."""
        dev = q.device

        def buf(name, shape, dtype):
            return _out_view(out, name, shape, dtype, dev)

        m0 = buf("matches0", (B, N), torch.int64)
        m1 = buf("matches1", (B, M), torch.int64)
        s0 = buf("matching_scores0", (B, N), torch.float32)
        s1 = buf("matching_scores1", (B, M), torch.float32)
        conf = buf("conf_matrix", (B, N, M), torch.float32) if return_conf else None
        if lengths is not None:
            lengths = lengths.to(device=dev, dtype=torch.int32).contiguous()
            if lengths.numel() != B:
                raise ValueError("lengths must have one entry per frame")
        st = torch.cuda.current_stream(dev).cuda_stream
        _lib.check(call(lengths.data_ptr() if lengths is not None else None, m0.data_ptr(), m1.data_ptr(), s0.data_ptr(), s1.data_ptr(),
                        conf.data_ptr() if conf is not None else None, st), self._handle)
        return {"matches0": m0, "matches1": m1, "matching_scores0": s0, "matching_scores1": s1, "conf_matrix": conf}

    # ------------------------------------------------------------------ several objects per call
    def add_object(self, descriptors3d_db: torch.Tensor, descriptors2d_db: torch.Tensor) -> int:
        """Register an object (descriptors3d_db [256, M], descriptors2d_db [256, M*L], CUDA fp32) next to the current one and
        return its id for match_objects.  Its frame-invariant GNN layers run on its first use; reloading the weights keeps it."""
        d3, d2, M, L, st = self._prepare_object(descriptors3d_db, descriptors2d_db)
        oid = C.c_int32()
        _lib.check(self._lib.opb_add_object(self._handle, d3.data_ptr(), d2.data_ptr(), M, L, st, C.byref(oid)), self._handle)
        self._objects[oid.value] = M
        return oid.value

    def remove_object(self, object_id: int):
        """Forget a registered object (waits for the calls in flight that may use it)."""
        if self._handle is None:
            raise ValueError(f"unknown object id {object_id}")
        _lib.check(self._lib.opb_remove_object(self._handle, int(object_id)), self._handle)
        self._objects.pop(int(object_id), None)

    def match_objects(self, descriptors2d_query: torch.Tensor, object_ids, return_conf: bool = True, lengths: torch.Tensor | None = None,
                      out: dict | None = None):
        """B frames of registered objects in one call: frame b matches against object object_ids[b] (a host sequence of ids, or a
        CPU tensor; objects of one call share L).  descriptors2d_query [B, 256, N] CUDA fp32, lengths and out as in match_frames.
        Returns the batched dict of match_frames with the M-wide outputs (matches1, matching_scores1, conf_matrix) padded to the
        largest M of the call -- or, when out["matches1"] is a 2-D [B', M_out] buffer, to its width M_out (fixed-width rows across
        calls; M_out must cover the call's largest M).  Columns past frame b's own M are -1 / 0 / 0.  Other out buffers are flat
        storage as in match_frames.  Asynchronous: no host synchronisation."""
        if self._handle is None:
            raise RuntimeError("no object registered: call add_object first")
        self._check_device(descriptors2d_query)
        self._sync_weights()
        ids = [int(i) for i in (object_ids.tolist() if isinstance(object_ids, torch.Tensor) else object_ids)]
        q = descriptors2d_query.float().contiguous()
        B, _, N = q.shape
        if len(ids) != B:
            raise ValueError(f"object_ids has {len(ids)} entries for {B} frames")
        for i in ids:
            if i == _CURRENT or i not in self._objects:
                raise ValueError(f"unknown object id {i}")
        M = max(self._objects[i] for i in ids)
        if out is not None and "matches1" in out and out["matches1"].dim() == 2:
            if out["matches1"].shape[1] < M:
                raise ValueError(f"out['matches1'] is {out['matches1'].shape[1]} wide, below the call's largest M = {M}")
            M = int(out["matches1"].shape[1])
        ids_host = (C.c_int32 * B)(*ids)

        def call(lens, *res):
            _lib.check(self._lib.opb_poll_range(self._handle), self._handle)
            return self._lib.opb_forward_objects(self._handle, ids_host, q.data_ptr(), lens, B, N, M, *res)
        return self._match(q, B, N, M, return_conf, lengths, out, call)

    def match_frames_host(self, q_host: torch.Tensor, out: dict | None = None, lengths: torch.Tensor | None = None,
                          materialize_conf: bool = True):
        """End-to-end call on HOST buffers (bench.py e2e leg): pinned fp32 [B,256,N] in; matches /
        scores copied back to pinned host tensors.  conf_matrix is computed on the device and stays
        there (the reference caller discards it: inference.py:146); materialize_conf=False skips it.  A host buffer
        out["conf_matrix"] (fp32, B * N * M elements) receives a copy of it."""
        self._require_object()
        B, _, N = q_host.shape
        M = self._objects[_CURRENT]
        if out is None:
            pin = dict(pin_memory=True)
            out = {"matches0": torch.empty(B, N, dtype=torch.int64, **pin), "matches1": torch.empty(B, M, dtype=torch.int64, **pin),
                   "matching_scores0": torch.empty(B, N, dtype=torch.float32, **pin),
                   "matching_scores1": torch.empty(B, M, dtype=torch.float32, **pin)}
        if lengths is not None:
            lengths = lengths.to(device="cpu", dtype=torch.int32).contiguous()
        conf = out.get("conf_matrix")
        if conf is not None and (conf.is_cuda or conf.dtype != torch.float32 or conf.numel() < B * N * M or not conf.is_contiguous()):
            raise ValueError(f"out['conf_matrix'] must be a contiguous fp32 host buffer with at least {B * N * M} elements")
        st = torch.cuda.current_stream(self._handle_device).cuda_stream
        _lib.check(self._lib.opb_forward_host(self._handle, q_host.data_ptr(), lengths.data_ptr() if lengths is not None else None, B, N,
                                              out["matches0"].data_ptr(), out["matches1"].data_ptr(), out["matching_scores0"].data_ptr(),
                                              out["matching_scores1"].data_ptr(), conf.data_ptr() if conf is not None else None,
                                              int(bool(materialize_conf)), st), self._handle)
        return out

    def check_range(self):
        """Wait for the last call and raise OpbError(OPB_E_RANGE) if it left the fp16-split operand range (its matches were
        reported as -1).  forward() / match_frames() never block for this: they deliver the error of an EARLIER call."""
        if self._handle is not None:
            _lib.check(self._lib.opb_check_range(self._handle, None), self._handle)

    def set_profiling(self, enable: bool):
        _lib.check(self._lib.opb_set_profiling(self._handle, int(enable)), self._handle)

    def get_profile(self):
        g, f, t = C.c_double(), C.c_double(), C.c_double()
        n = C.c_int32()
        _lib.check(self._lib.opb_get_profile(self._handle, C.byref(g), C.byref(f), C.byref(n), C.byref(t)), self._handle)
        return {"gemm_ms": g.value, "gemm_flops": f.value, "gemm_launches": n.value, "total_ms": t.value}

    def get_profile_entry(self, prefix: str):
        g, f = C.c_double(), C.c_double()
        n = C.c_int32()
        _lib.check(self._lib.opb_get_profile_entry(self._handle, prefix.encode(), C.byref(g), C.byref(f), C.byref(n)), self._handle)
        return {"ms": g.value, "flops": f.value, "launches": n.value}

    def launch_count(self) -> int:
        return int(self._lib.opb_last_launch_count(self._handle)) if self._handle is not None else 0

    # ------------------------------------------------------------------ test hooks (opb_debug_set_stop / opb_debug_read)
    DEBUG_BUFFERS = {"x": 0, "kvt": 1, "kmean": 2, "bd": 3, "qp": 4, "g": 5, "hid": 6, "mu": 7, "rstd": 8, "pn": 9,
                     "inv_rowsum": 10, "inv_colsum": 11, "rowbest": 12, "colbest": 13, "gats_pre": 14}

    def debug_stop_after(self, layer: int, step: int = 0, chunk: int = 0, piece: int = 0):
        """Stop the next call after step `step` of GNN layer `layer` (12 = tail, 16 / 17 = the object prologue's layers 0 / 1;
        see opb_debug_set_stop) in chunk `chunk`, and in sub-batch `piece` of the hoisted query pass (layer 1; see
        opb_debug_set_stop_pass); -1 runs everything."""
        _lib.check(self._lib.opb_debug_set_stop_pass(self._handle, int(chunk), int(piece)), self._handle)
        _lib.check(self._lib.opb_debug_set_stop(self._handle, int(layer), int(step)), self._handle)

    def debug_invalidate_prologues(self):
        """The next call runs every object's prologue again (opb_debug_invalidate_prologues)."""
        _lib.check(self._lib.opb_debug_invalidate_prologues(self._handle), self._handle)

    def debug_layout(self) -> dict:
        """Layout of the pass the last call stopped in: B, N, M, n_pad, m_pad, R, S."""
        v = (C.c_int32 * 7)()
        _lib.check(self._lib.opb_debug_stopped_layout(self._handle, v), self._handle)
        return dict(zip(("B", "N", "M", "n_pad", "m_pad", "R", "S"), list(v)))

    def debug_read(self, name: str) -> torch.Tensor:
        """A buffer of the stopped pass (opb_debug_read), shaped: [rows, C] / [S, ...] / [B, ...] (int64 for the arg-maxes)."""
        L = self.debug_layout()
        rows, S, B = L["B"] * L["R"], L["S"], L["B"]
        shapes = {"x": (rows, 256), "kvt": (rows, 512), "kmean": (S, 256), "bd": (S, 256, 256), "qp": (rows, 256), "g": (S, 512, 256),
                  "hid": (rows, 512), "mu": (S, 512), "rstd": (S, 512), "pn": (rows, 256), "inv_rowsum": (B, L["n_pad"]),
                  "inv_colsum": (B, L["m_pad"]), "rowbest": (B, L["N"]), "colbest": (B, L["M"]), "gats_pre": (B * L["m_pad"], 256)}
        shape = shapes[name]
        n_want = 1
        for d in shape:
            n_want *= d
        dtype = torch.int64 if name in ("rowbest", "colbest") else torch.float32
        out = torch.empty(max(n_want, 1), dtype=dtype, device=self._handle_device)
        n = C.c_int64()
        st = torch.cuda.current_stream(self._handle_device).cuda_stream
        _lib.check(self._lib.opb_debug_read(self._handle, self.DEBUG_BUFFERS[name], out.data_ptr(), out.numel(), C.byref(n), st),
                   self._handle)
        return out[:n.value].view(shape)

    # ------------------------------------------------------------------ reference contract
    @staticmethod
    def _tensor_key(t: torch.Tensor):
        return (t.data_ptr(), t._version, tuple(t.shape), tuple(t.stride()))

    def _use_object(self, d3: torch.Tensor, d2: torch.Tensor, base3: torch.Tensor, base2: torch.Tensor):
        """Make (d3 [256,M], d2 [256,M*L]) the current object.  The reference caller re-sends the per-object tensors with every
        frame (inference.py:80-94); they are packed once:
          * same tensors as last time (data_ptr, _version, shape; a strong reference keeps their storage from being recycled)
            -> nothing to do, no device work, no synchronisation;
          * different tensors -> exact comparison with a private copy of the packed object (one device reduction + one
            4-byte read-back); only a real change re-packs (opb_set_object)."""
        key = (self._tensor_key(d3), self._tensor_key(d2))
        if key == self._obj_key:
            return
        same = (self._obj_copy is not None and self._obj_copy[0].shape == d3.shape and self._obj_copy[1].shape == d2.shape
                and self._obj_copy[0].device == d3.device
                and bool(torch.equal(self._obj_copy[0], d3)) and bool(torch.equal(self._obj_copy[1], d2)))
        if not same:
            self.set_object(d3, d2)
            self._obj_copy = (d3.clone(), d2.clone())
        self._obj_key = key
        self._obj_ref = (base3, base2)

    @torch.no_grad()
    def forward(self, data):
        """Same keys / shapes as the reference (GATs_SuperGlue.py:180-190).  No host synchronisation on the common path
        (same object tensors as the previous call); a range violation of an earlier call is raised here."""
        kpts2d, kpts3d = data["keypoints2d"].float(), data["keypoints3d"].float()
        desc2d_query = data["descriptors2d_query"].float()
        desc3d_db, desc2d_db = data["descriptors3d_db"].float(), data["descriptors2d_db"].float()

        if kpts2d.shape[1] == 0 or kpts3d.shape[1] == 0:                  # :195-203 -- bare dict, int32
            shape0, shape1 = kpts2d.shape[:-1], kpts3d.shape[:-1]
            return {
                "matches0": kpts2d.new_full(shape0, -1, dtype=torch.int)[0],
                "matches1": kpts3d.new_full(shape1, -1, dtype=torch.int)[0],
                "matching_scores0": kpts2d.new_zeros(shape0)[0],
                "matching_scores1": kpts3d.new_zeros(shape1)[0],
                "skip_train": True,
            }
        if self.match_type != "softmax":
            raise NotImplementedError                                     # :238-239
        if not desc2d_query.is_cuda:
            raise RuntimeError("onepose_b200 has no CPU path: move the module and its inputs to a CUDA device")

        B = desc2d_query.shape[0]
        self._ensure_handle(desc2d_query.device)
        self._sync_weights()
        _lib.check(self._lib.opb_poll_range(self._handle), self._handle)  # deferred report of an earlier call (never blocks)
        # runs of frames that share an object (the reference accepts per-element 3D descriptors; its callers use B = 1)
        if B == 1 or (desc3d_db.stride(0) == 0 and desc2d_db.stride(0) == 0):
            groups = [list(range(B))]
        else:
            same = ((desc3d_db[1:] == desc3d_db[:-1]).flatten(1).all(1) & (desc2d_db[1:] == desc2d_db[:-1]).flatten(1).all(1)).cpu()
            groups = [[0]]
            for b in range(1, B):
                if bool(same[b - 1]):
                    groups[-1].append(b)
                else:
                    groups.append([b])
        outs = []
        for g in groups:
            self._use_object(desc3d_db[g[0]], desc2d_db[g[0]], desc3d_db, desc2d_db)
            outs.append(self.match_frames(desc2d_query[g[0]:g[-1] + 1]))
        out = outs[0] if len(outs) == 1 else {k: torch.cat([o[k] for o in outs], 0) for k in outs[0]}
        self.last_batched = out
        pred = {
            "matches0": out["matches0"][0],                               # :232-237: element 0 only
            "matches1": out["matches1"][0],
            "matching_scores0": out["matching_scores0"][0],
            "matching_scores1": out["matching_scores1"][0],
        }
        return pred, out["conf_matrix"]


class LitModelGATsSPG(nn.Module):
    """Stand-in for the reference's Lightning wrapper (src/models/GATsSPG_lightning_model.py:15-37):
    ``forward(x) = self.matcher(x)`` and a ``load_from_checkpoint`` that reads a Lightning ``.ckpt``
    (``state_dict`` with ``matcher.*`` / ``extractor.*`` keys + ``hyper_parameters``) without
    pytorch_lightning.  Training / validation steps are out of scope (SURVEY 8)."""

    def __init__(self, *args, **kwargs):
        super().__init__()
        self.hparams = dict(kwargs)
        self.matcher = GATsSuperGlue(hparams=self.hparams)

    def forward(self, x):
        return self.matcher(x)

    def freeze(self):
        for p in self.parameters():
            p.requires_grad = False
        return self.eval()

    @classmethod
    def load_from_checkpoint(cls, checkpoint_path, map_location="cpu", **overrides):
        ckpt = torch.load(checkpoint_path, map_location=map_location, weights_only=False)
        hp = dict(ckpt.get("hyper_parameters", {}))
        hp.update(overrides)
        model = cls(**hp)
        sd = {k[len("matcher."):]: v for k, v in ckpt["state_dict"].items() if k.startswith("matcher.")}
        model.matcher.load_state_dict(sd, strict=True)
        return model
