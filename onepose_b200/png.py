"""PNG files of camera frames and crops on the device, byte for byte as ``cv2.imencode('.png', frame)`` / ``cv2.imwrite`` write
them (OpenCV 4.13's default call).

``parse_scanned_data.py`` writes every annotated frame twice -- its 512 x 512 crop to ``color/{i}.png`` and the full frame to
``color_full/{i}.png`` (``:173``, ``:177``), and every test frame to ``color_full/`` (``:264-273``) -- and every later stage reads
those files back.  ``imwrite`` writes the same files from device frames with one encode call and one device-to-host copy:

    out = scan.annotate(...)
    png.imwrite([f"{root}/color/{i}.png" for i in ids], out["image"])        # the crops
    png.imwrite([f"{root}/color_full/{i}.png" for i in ids], frames_bgr)    # the frames

The encoder is ``csrc/png.cu`` behind ``opb_png_encode``; the byte model is ``tests/png_reference.py``."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib

MAX_FRAMES = 65535
MAX_FILTERED = 1 << 28          # H * (1 + W * C) per frame


def _check(frames: torch.Tensor, batched: bool):
    if not isinstance(frames, torch.Tensor):
        raise ValueError(f"frames must be a torch.Tensor, got {type(frames).__name__}")
    want = "[F, H, W], [F, H, W, 3] or [F, H, W, 4]" if batched else "[H, W], [H, W, 3] or [H, W, 4]"
    d = 3 if batched else 2
    if frames.dtype != torch.uint8 or frames.dim() not in (d, d + 1) or (frames.dim() == d + 1 and frames.shape[-1] not in (1, 3, 4)):
        raise ValueError(f"frames must be uint8 {want}, got {frames.dtype} {list(frames.shape)}")
    if not batched:
        frames = frames.unsqueeze(0)
    if frames.dim() == 3:
        frames = frames.unsqueeze(-1)
    F, H, W, Ch = (int(v) for v in frames.shape)
    if not (0 < F <= MAX_FRAMES and H > 0 and W > 0 and H * (1 + W * Ch) <= MAX_FILTERED):
        raise ValueError(f"frames must be 1..{MAX_FRAMES} images with H * (1 + W * C) <= {MAX_FILTERED}, got {list(frames.shape)}")
    row = frames.stride(1) if H > 1 else W * Ch
    frame = frames.stride(0) if F > 1 else H * row
    if ((Ch > 1 and frames.stride(3) != 1) or (W > 1 and frames.stride(2) != Ch) or row < W * Ch
            or not (frame == 0 or frame >= H * row)):
        raise ValueError(f"frames must have packed pixels, rows that do not overlap and frames that do not overlap (or a frame "
                         f"stride of 0), got strides {frames.stride()}")
    return frames, F, H, W, Ch, frame, row


def frame_bytes(H: int, W: int, Ch: int) -> int:
    """The slot one file of an H x W x Ch frame needs: zlib's deflateBound of its filtered bytes, 12 bytes per IDAT chunk and 45
    for the signature, IHDR and IEND."""
    out = C.c_int64()
    _lib.check(_lib.load().opb_png_frame_bytes(H, W, Ch, C.byref(out)))
    return out.value


def encode(frames: torch.Tensor):
    """PNG files of uint8 frames on the device: ``[F, H, W]`` grey, ``[F, H, W, 3]`` BGR or ``[F, H, W, 4]`` BGRA (cv2's channel
    order), packed pixels with rows and frames at any stride that does not overlap them.

    Returns ``(buf, sizes)``: buf uint8 ``[F, slot]`` on the frames' device, frame f's file in ``buf[f, :sizes[f]]``, and sizes
    int64 ``[F]`` on the device.  Each file is the bytes ``cv2.imencode('.png', frame)`` gives.  Runs on the current stream
    without a host synchronisation."""
    frames, F, H, W, Ch, frame_pitch, row_pitch = _check(frames, True)
    dev = _lib.cuda_device(frames)
    lib = _lib.load()
    ws = C.c_int64()
    _lib.check(lib.opb_png_workspace_bytes(F, H, W, Ch, C.byref(ws)))
    slot = frame_bytes(H, W, Ch)
    workspace = torch.empty(ws.value, dtype=torch.uint8, device=dev)
    buf = torch.empty((F, slot), dtype=torch.uint8, device=dev)
    sizes = torch.empty(F, dtype=torch.int64, device=dev)
    _lib.call(dev, "opb_png_encode", frames, frame_pitch, row_pitch, F, H, W, Ch, workspace, ws.value, buf, slot, sizes)
    return buf, sizes


def _host_files(frames: torch.Tensor):
    """encode, then the used bytes of every file in one copy to pinned host memory: (uint8 [F, max size], sizes)."""
    buf, sizes = encode(frames)
    n = sizes.cpu().numpy()
    if (n < 0).any():
        raise _lib.OpbError(f"frames {np.flatnonzero(n < 0).tolist()} did not fit their slots")
    host = torch.empty((buf.shape[0], int(n.max())), dtype=torch.uint8, pin_memory=True)
    host.copy_(buf[:, :host.shape[1]])
    return host.numpy(), n


def imencode(frame: torch.Tensor) -> np.ndarray:
    """``cv2.imencode('.png', frame)[1]`` of one uint8 frame on the device: ``[H, W]``, ``[H, W, 3]`` BGR or ``[H, W, 4]`` BGRA."""
    _check(frame, False)
    host, n = _host_files(frame.unsqueeze(0))
    return host[0, :n[0]].copy()


def imwrite(paths, frames: torch.Tensor) -> None:
    """``cv2.imwrite(paths[f], frames[f])`` for every frame of uint8 ``[F, H, W]``, ``[F, H, W, 3]`` BGR or ``[F, H, W, 4]`` BGRA
    device frames: one encode call, one device-to-host copy of the used bytes, then the file writes."""
    paths = list(paths)
    F = _check(frames, True)[1]
    if len(paths) != F:
        raise ValueError(f"{len(paths)} paths for {F} frames")
    host, n = _host_files(frames)
    for p, row, k in zip(paths, host, n):
        with open(p, "wb") as fh:
            fh.write(row[:k].tobytes())
