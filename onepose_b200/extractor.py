"""``SuperPoint`` -- drop-in for the reference's key-point extractor on an H100.

Same constructor (``config`` mapping merged over ``default_config``), same parameter names (``conv1a.weight`` ...
``convDb.bias``, so ``load_state_dict`` / ``load_network`` of a reference checkpoint work unchanged) and same ``forward(inp)``
result -- ``{'keypoints': [n_b x 2 (x, y) fp32], 'scores': [n_b], 'descriptors': [256 x n_b]}`` per image -- as
``src/models/extractors/SuperPoint/superpoint.py:94-197`` of the reference; the computation is the hand-written sm_90a
path of ``csrc/superpoint.cu`` behind the C ABI ``opb_sp_*``.  There is no CPU path.

``forward_padded`` is the device-resident hand-off to the matcher (SURVEY 8f N1): fixed-capacity outputs
``descriptors [B, 256, cap]`` + ``counts [B]`` that ``GATsSuperGlue.match_frames(descriptors, lengths=counts)`` consumes
without the reference's numpy round trip (``inference.py:140-146``) and without a host synchronisation.
"""
from __future__ import annotations

import ctypes as C

import torch
from torch import nn

from . import _lib


class SuperPoint(nn.Module):
    default_config = {
        # superpoint.py:97-103
        "descriptor_dim": 256,
        "nms_radius": 4,
        "keypoint_threshold": 0.005,
        "max_keypoints": -1,
        "remove_borders": 4,
    }

    def __init__(self, config, align_corners: bool = True):
        """``align_corners``: the reference passes align_corners=True to grid_sample under its pinned torch 1.8
        (superpoint.py:86, a check of ``torch.__version__[2]``); the same source run on torch >= 1.10 falls back to False.
        The pinned environment's behaviour is the default."""
        super().__init__()
        self.config = {**self.default_config, **config}
        c1, c2, c3, c4, c5 = 64, 64, 128, 128, 256
        self.conv1a = nn.Conv2d(1, c1, kernel_size=3, stride=1, padding=1)
        self.conv1b = nn.Conv2d(c1, c1, kernel_size=3, stride=1, padding=1)
        self.conv2a = nn.Conv2d(c1, c2, kernel_size=3, stride=1, padding=1)
        self.conv2b = nn.Conv2d(c2, c2, kernel_size=3, stride=1, padding=1)
        self.conv3a = nn.Conv2d(c2, c3, kernel_size=3, stride=1, padding=1)
        self.conv3b = nn.Conv2d(c3, c3, kernel_size=3, stride=1, padding=1)
        self.conv4a = nn.Conv2d(c3, c4, kernel_size=3, stride=1, padding=1)
        self.conv4b = nn.Conv2d(c4, c4, kernel_size=3, stride=1, padding=1)
        self.convPa = nn.Conv2d(c4, c5, kernel_size=3, stride=1, padding=1)
        self.convPb = nn.Conv2d(c5, 65, kernel_size=1, stride=1, padding=0)
        self.convDa = nn.Conv2d(c4, c5, kernel_size=3, stride=1, padding=1)
        self.convDb = nn.Conv2d(c5, self.config["descriptor_dim"], kernel_size=1, stride=1, padding=0)
        mk = self.config["max_keypoints"]
        if mk == 0 or mk < -1:
            raise ValueError('"max_keypoints" must be positive or "-1"')       # superpoint.py:133-135
        self.align_corners = bool(align_corners)
        self._lib = _lib.load()        # raises if the CUDA library is not built
        self._handle = None
        self._handle_device = None
        self._weights_key = None

    def __del__(self):
        try:
            if self._handle is not None:
                self._lib.opb_sp_destroy(self._handle)
        except Exception:
            pass

    # ------------------------------------------------------------------ handle / weights
    def _ensure_handle(self, device: torch.device):
        if self._handle is not None and self._handle_device == device:
            return
        if self._handle is not None:
            self._lib.opb_sp_destroy(self._handle)
            self._handle = None
        c = self.config
        cfg = _lib.OpbSpConfig(int(c["descriptor_dim"]), int(c["nms_radius"]), float(c["keypoint_threshold"]), int(c["max_keypoints"]),
                               int(c["remove_borders"]), int(self.align_corners), device.index or 0)
        h = C.c_void_p()
        _lib.check(self._lib.opb_sp_create(C.byref(cfg), C.byref(h)))
        self._handle, self._handle_device, self._weights_key = h, device, None

    def _sync_weights(self):
        key = tuple((n, p.data_ptr(), p._version) for n, p in self.named_parameters())
        if key == self._weights_key:
            return
        for name, p in self.named_parameters():
            w = p.detach().to("cpu", torch.float32).contiguous()
            _lib.check(self._lib.opb_sp_load_weight(self._handle, name.encode(), w.data_ptr(), w.numel()), self._handle, "extractor")
        _lib.check(self._lib.opb_sp_finalize_weights(self._handle), self._handle, "extractor")
        self._weights_key = key

    def _prepare(self, inp: torch.Tensor):
        if not inp.is_cuda:
            raise RuntimeError("onepose_b200 has no CPU path: move the module and its input to a CUDA device")
        if inp.dim() != 4 or inp.shape[1] != 1:
            raise ValueError(f"expected a grey image batch [B, 1, H, W], got {tuple(inp.shape)}")
        img = inp.float().contiguous()
        self._ensure_handle(img.device)
        self._sync_weights()
        return img, torch.cuda.current_stream(img.device).cuda_stream

    # ------------------------------------------------------------------ device-resident API
    @torch.no_grad()
    def forward_padded(self, inp: torch.Tensor, cap: int | None = None, descriptors: bool = True):
        """Fixed-capacity outputs, no host synchronisation: keypoints [B, cap, 2], scores [B, cap], descriptors [B, 256, cap],
        counts int32 [B] (entries >= counts[b] are unspecified).  cap defaults to max_keypoints (which must then be >= 0).
        A call whose activations leave the operand range reports count 0 everywhere (see check_range); its error is raised by
        check_range() or by a later call."""
        img, st = self._prepare(inp)
        B, _, H, W = img.shape
        if cap is None:
            cap = int(self.config["max_keypoints"])
            if cap < 0:
                raise ValueError("forward_padded needs a capacity when max_keypoints is -1")
        dev = img.device
        kp = torch.empty(B, cap, 2, dtype=torch.float32, device=dev)
        sc = torch.empty(B, cap, dtype=torch.float32, device=dev)
        de = torch.empty(B, 256, cap, dtype=torch.float32, device=dev) if descriptors else None
        cnt = torch.empty(B, dtype=torch.int32, device=dev)
        _lib.check(self._lib.opb_sp_forward(self._handle, img.data_ptr(), B, H, W, kp.data_ptr(), sc.data_ptr(),
                                            de.data_ptr() if de is not None else None, cnt.data_ptr(), cap, st), self._handle, "extractor")
        return {"keypoints": kp, "scores": sc, "descriptors": de, "counts": cnt}

    # ------------------------------------------------------------------ reference contract
    @torch.no_grad()
    def forward(self, inp):
        """Compute keypoints, scores, descriptors for image (superpoint.py:140-197).  One host synchronisation -- the read of the
        per-image key-point counts -- where the reference has torch.nonzero."""
        img, st = self._prepare(inp)
        B, _, H, W = img.shape
        dev = img.device
        cnt = torch.empty(B, dtype=torch.int32, device=dev)
        _lib.check(self._lib.opb_sp_detect(self._handle, img.data_ptr(), B, H, W, cnt.data_ptr(), st), self._handle, "extractor")
        n = [int(v) for v in cnt.cpu()]
        self.check_range()                 # the read of the counts has synchronised: an out-of-range call raises here
        cap = max(max(n), 1)
        kp = torch.empty(B, cap, 2, dtype=torch.float32, device=dev)
        sc = torch.empty(B, cap, dtype=torch.float32, device=dev)
        de = torch.empty(B, 256, cap, dtype=torch.float32, device=dev)
        _lib.check(self._lib.opb_sp_describe(self._handle, kp.data_ptr(), sc.data_ptr(), de.data_ptr(), cnt.data_ptr(), cap, st),
                   self._handle, "extractor")
        return {
            "keypoints": [kp[b, :n[b]] for b in range(B)],
            "scores": [sc[b, :n[b]] for b in range(B)],
            "descriptors": [de[b, :, :n[b]].contiguous() for b in range(B)],
        }

    def check_range(self):
        """Wait for the last call and raise OpbError(OPB_E_RANGE) if an activation left the fp16-split operand range
        (|x| >= 1023) or became NaN; that call reported no key points.  Reporting clears the error."""
        if self._handle is not None:
            _lib.check(self._lib.opb_sp_check_range(self._handle, None), self._handle, "extractor")

    # ------------------------------------------------------------------ measurement / test hooks
    def launch_count(self) -> int:
        return int(self._lib.opb_sp_last_launch_count(self._handle)) if self._handle is not None else 0

    def set_profiling(self, enable: bool):
        _lib.check(self._lib.opb_sp_set_profiling(self._handle, int(enable)), self._handle, "extractor")

    def get_profile(self):
        """[(name, ms, algorithmic flops)] of the launches of the last call (profiling on)."""
        out = []
        name = C.create_string_buffer(64)
        ms, fl = C.c_double(), C.c_double()
        i = 0
        while self._lib.opb_sp_get_profile(self._handle, i, name, 64, C.byref(ms), C.byref(fl)) == 0:
            out.append((name.value.decode(), ms.value, fl.value))
            i += 1
        return out

    def debug_stop_after(self, layer: int):
        _lib.check(self._lib.opb_sp_debug_set_stop(self._handle, int(layer)), self._handle, "extractor")

    def debug_read(self, which: int, capacity: int):
        out = torch.empty(capacity, dtype=torch.float32, device=self._handle_device)
        n = C.c_int64()
        st = torch.cuda.current_stream(self._handle_device).cuda_stream
        _lib.check(self._lib.opb_sp_debug_read(self._handle, which, out.data_ptr(), capacity, C.byref(n), st), self._handle, "extractor")
        return out[:n.value]
