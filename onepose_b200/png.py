"""PNG files of camera frames and crops on the device, byte for byte as ``cv2.imencode('.png', frame)`` / ``cv2.imwrite`` write
them (OpenCV 4.13's default call), and read back as ``cv2.imread`` / ``cv2.imdecode`` read them.

``parse_scanned_data.py`` writes every annotated frame twice -- its 512 x 512 crop to ``color/{i}.png`` and the full frame to
``color_full/{i}.png`` (``:173``, ``:177``), and every test frame to ``color_full/`` (``:264-273``) -- and every later stage reads
those files back.  ``imwrite`` writes the same files from device frames with one encode call and one device-to-host copy:

    out = scan.annotate(...)
    png.imwrite([f"{root}/color/{i}.png" for i in ids], out["image"])        # the crops
    png.imwrite([f"{root}/color_full/{i}.png" for i in ids], frames_bgr)    # the frames

The encoder is ``csrc/png.cu`` behind ``opb_png_encode``; the byte model is ``tests/png_reference.py``.

Every stage of the reference reads those files with ``cv2.imread`` (NormalizedDataset, the SfM feature extraction, the
detector's views and queries).  ``imread`` gives the same pixels from one host-to-device copy and one decode call:

    grey, inp = png.imread([f"{root}/color/{i}.png" for i in ids], cv2.IMREAD_GRAYSCALE, normalised=True)

The reader is ``csrc/png_decode.cu`` behind ``opb_png_decode``; its model is ``tests/png_decode_reference.py``."""
from __future__ import annotations

import ctypes as C
import struct

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


IMREAD_GRAYSCALE, IMREAD_COLOR = 0, 1      # cv2's flag values
READ_MODES = {IMREAD_GRAYSCALE: 0, IMREAD_COLOR: 1}   # OPB_PNG_READ_GREY, OPB_PNG_READ_BGR
STATUS = {0: "ok", 1: "not a PNG or bad chunk structure", 2: "CRC mismatch", 3: "unsupported format", 4: "shape differs",
          5: "bad deflate stream", 6: "Adler-32 mismatch", 7: "too little image data", 8: "bad row filter"}
OK, UNSUPPORTED = 0, 3
_SIGNATURE = b"\x89PNG\r\n\x1a\n"


def _mode(flags) -> int:
    if not isinstance(flags, int) or isinstance(flags, bool) or flags not in READ_MODES:
        raise ValueError(f"flags must be cv2.IMREAD_GRAYSCALE ({IMREAD_GRAYSCALE}) or cv2.IMREAD_COLOR ({IMREAD_COLOR}), got {flags!r}")
    return READ_MODES[flags]


def read_ihdr(buf: bytes):
    """(H, W, colour type) of a PNG file's IHDR, or None when the bytes do not start with a signature and an IHDR.  Raises
    ValueError for a format the reader does not take: bit depth other than 8, colour type other than 0, 2 or 6, interlace."""
    if len(buf) < 33 or bytes(buf[:8]) != _SIGNATURE or bytes(buf[8:16]) != b"\x00\x00\x00\rIHDR":
        return None
    W, H, depth, ct, comp, filt, inter = struct.unpack(">IIBBBBB", bytes(buf[16:29]))
    if depth != 8 or ct not in (0, 2, 6) or comp or filt or inter:
        raise ValueError(f"unsupported PNG format: bit depth {depth}, colour type {ct}, interlace {inter} (8-bit grey, RGB or RGBA, "
                         f"not interlaced, is read)")
    return H, W, ct


def decode(data: torch.Tensor, offsets: torch.Tensor, H: int, W: int, flags: int, normalised: bool = False, out=None):
    """Decode F PNG files of one shape on the device as ``cv2.imdecode(file, flags)`` does.

    data: uint8 device tensor holding the files back to back; offsets: int64 ``[F + 1]`` on the same device, non-decreasing
    from 0, file f at ``data[offsets[f]:offsets[f + 1]]`` (offsets that decrease anywhere make every file's status 1).  flags: ``cv2.IMREAD_GRAYSCALE`` (uint8 ``[F, H, W]``) or ``cv2.IMREAD_COLOR`` (BGR uint8
    ``[F, H, W, 3]``).  ``normalised`` (grey only) adds NormalizedDataset's fp32 ``[F, 1, H, W]`` ``image / 255.``.  ``out``
    optionally takes the pixel tensor to write.

    Returns ``(pixels, status)`` or ``(pixels, image, status)``, status int32 ``[F]`` (``STATUS``; 0 is ok).  A file whose status
    is not 0 has its pixels left as they were.  Runs on the current stream without a host synchronisation."""
    mode = _mode(flags)
    if normalised and mode != 0:
        raise ValueError("normalised=True takes cv2.IMREAD_GRAYSCALE")
    if not isinstance(data, torch.Tensor) or data.dtype != torch.uint8 or data.dim() != 1 or not data.is_contiguous():
        raise ValueError("data must be a contiguous 1-D uint8 tensor")
    if (not isinstance(offsets, torch.Tensor) or offsets.dtype != torch.int64 or offsets.dim() != 1 or not offsets.is_contiguous()
            or offsets.device != data.device):
        raise ValueError("offsets must be a contiguous 1-D int64 tensor on data's device")
    dev = _lib.cuda_device(data)
    F = offsets.numel() - 1
    if not (0 < F <= MAX_FRAMES and H > 0 and W > 0 and H * (1 + 4 * W) <= MAX_FILTERED):
        raise ValueError(f"decode takes 1..{MAX_FRAMES} files with H * (1 + 4 W) <= {MAX_FILTERED}, got F={F}, H={H}, W={W}")
    shape = (F, H, W) if mode == 0 else (F, H, W, 3)
    if out is None:
        out = torch.empty(shape, dtype=torch.uint8, device=dev)
    elif (not isinstance(out, torch.Tensor) or out.dtype != torch.uint8 or tuple(out.shape) != shape or out.device != data.device
          or not out.is_contiguous()):
        raise ValueError(f"out must be a contiguous uint8 tensor of shape {list(shape)} on data's device")
    image = torch.empty((F, 1, H, W), dtype=torch.float32, device=dev) if normalised else None
    status = torch.empty(F, dtype=torch.int32, device=dev)
    ws = C.c_int64()
    lib = _lib.load()
    _lib.check(lib.opb_png_decode_workspace_bytes(F, H, W, data.numel(), C.byref(ws)))
    workspace = torch.empty(ws.value, dtype=torch.uint8, device=dev)
    px = 1 if mode == 0 else 3
    _lib.call(dev, "opb_png_decode", data, offsets, F, H, W, mode, workspace, ws.value, out, H * W * px, W * px, image, status)
    return (out, image, status) if normalised else (out, status)


def imdecode(buf, flags: int, device=None):
    """``cv2.imdecode(buf, flags)`` of one PNG file's bytes (numpy uint8 or bytes) on the device: a numpy ``[H, W]`` grey or
    ``[H, W, 3]`` BGR array, or None where cv2 returns None.  A format the reader does not take raises ValueError."""
    _mode(flags)
    raw = np.frombuffer(bytes(buf), dtype=np.uint8)
    head = read_ihdr(raw)
    if head is None:
        return None
    H, W, _ = head
    if not (H > 0 and W > 0 and H * (1 + 4 * W) <= MAX_FILTERED):
        return None
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    data = torch.from_numpy(raw.copy()).to(dev)
    offsets = torch.tensor([0, raw.size], dtype=torch.int64, device=dev)
    pixels, status = decode(data, offsets, H, W, flags)
    s = int(status.item())
    if s == UNSUPPORTED:
        raise ValueError(f"unsupported PNG: {STATUS[s]} (a colour file read grey with gAMA, sRGB or iCCP)")
    return pixels[0].cpu().numpy() if s == OK else None


def imread(paths, flags: int, normalised: bool = False, device=None):
    """``cv2.imread(path, flags)`` of every file in ``paths`` -- PNG files of one width and height -- on the device: one pinned
    host buffer, one host-to-device copy, one decode call and one status read.

    Returns the pixels (uint8 ``[F, H, W]`` grey or ``[F, H, W, 3]`` BGR), and with ``normalised`` (grey only) also
    NormalizedDataset's fp32 ``[F, 1, H, W]`` ``image / 255.``.  Raises ValueError for a file that is not a PNG of the first
    file's width and height, or of a format the reader does not take, and OpbError naming every file the decoder refused."""
    _mode(flags)
    paths = [str(p) for p in paths]
    if not paths:
        raise ValueError("imread takes at least one path")
    blobs = []
    for p in paths:
        with open(p, "rb") as fh:
            blobs.append(fh.read())
    shape = None
    for p, b in zip(paths, blobs):
        head = read_ihdr(b)
        if head is None:
            raise ValueError(f"{p} is not a PNG file")
        shape = shape or head[:2]
        if head[:2] != shape:
            raise ValueError(f"{p} is {head[1]} x {head[0]}, the first file {shape[1]} x {shape[0]}")
    H, W = shape
    offsets = np.zeros(len(blobs) + 1, dtype=np.int64)
    offsets[1:] = np.cumsum([len(b) for b in blobs])
    host = torch.empty(int(offsets[-1]) + 8 * (len(blobs) + 2), dtype=torch.uint8, pin_memory=True)
    hv = host.numpy()
    for b, o in zip(blobs, offsets):
        hv[o:o + len(b)] = np.frombuffer(b, dtype=np.uint8)
    n = int(offsets[-1])
    n8 = (n + 7) & ~7                        # the offsets follow the files, 8-byte aligned
    hv[n8:n8 + 8 * len(offsets)] = offsets.view(np.uint8)
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    dev_buf = host.to(dev, non_blocking=True)
    data, offs = dev_buf[:n], dev_buf[n8:n8 + 8 * len(offsets)].view(torch.int64)
    res = decode(data, offs, H, W, flags, normalised)
    status = res[-1].cpu().numpy()
    bad = np.flatnonzero(status != OK)
    if bad.size:
        raise _lib.OpbError("PNG files not decoded: " + "; ".join(f"{paths[i]}: {STATUS.get(int(status[i]), status[i])}" for i in bad))
    return res[:-1] if normalised else res[0]
