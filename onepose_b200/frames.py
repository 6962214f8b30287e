"""Colour camera frames to the reference's grey frames on the GPU.

The reference reads every frame as ``cv2.imread(path, cv2.IMREAD_GRAYSCALE)`` of the colour PNGs ``parse_scanned_data.py``
writes (``NormalizedDataset``, ``src/datasets/normalized_dataset.py:25-34``), and every frame consumer here -- ``crop``,
``detect``, ``flow`` -- takes those grey uint8 ``[F, H, W]`` frames.  A live caller holds colour frames instead: BGR from
``cv2.VideoCapture``, RGB or RGBA from a camera API.  ``grey_frames`` turns them into the reference's grey pixels on the device
(``csrc/frames.cu`` behind ``opb_grey_frames``), so the frame goes to the GPU as the camera delivers it:

    grey = frames.grey_frames(bgr_u8)                                   # [F,H,W,3] uint8 CUDA -> [F,H,W] uint8
    bbox, inp, K_crop = crop.previous_pose_detect(grey, K, res_prev["pose"], bbox3d)

``cv2.cvtColor(COLOR_BGR2GRAY)`` is no substitute: it differs from the PNG reader's grey by one level on half of the colours,
and SuperPoint, the crop and the flow then see other bytes than the reference's.
"""
from __future__ import annotations

import torch

from . import _lib

ORDERS = {"bgr": 0, "rgb": 1, "bgra": 2, "rgba": 3}      # OPB_ORDER_* (include/onepose_b200.h)
MAX_FRAMES = 65535
MAX_SIDE = 32767


def _pitches(t: torch.Tensor, row_bytes: int):
    """(frame, row) pitches in bytes of a [F, H, ...] uint8 tensor; the stride of a dimension of size 1 does not address
    anything, so it is given the value of a packed layout."""
    F, H = int(t.shape[0]), int(t.shape[1])
    row = t.stride(1) if H > 1 else row_bytes
    return (t.stride(0) if F > 1 else H * row), row


def _check_frames(frames: torch.Tensor, order: str):
    if not isinstance(frames, torch.Tensor):
        raise ValueError(f"frames must be a torch.Tensor, got {type(frames).__name__}")
    if order not in ORDERS:
        raise ValueError(f"order must be one of {sorted(ORDERS)}, got {order!r}")
    C = len(order)
    if frames.dtype != torch.uint8 or frames.dim() not in (3, 4) or frames.shape[-1] != C:
        raise ValueError(f"frames must be uint8 [F, H, W, {C}] or [H, W, {C}] for order {order!r}, got {frames.dtype} {list(frames.shape)}")
    if frames.dim() == 3:
        frames = frames.unsqueeze(0)
    F, H, W = (int(v) for v in frames.shape[:3])
    if not (0 < F <= MAX_FRAMES and 0 < H <= MAX_SIDE and 0 < W <= MAX_SIDE):
        raise ValueError(f"frames must be 1..{MAX_FRAMES} images of 1..{MAX_SIDE} pixels a side, got {list(frames.shape)}")
    frame_pitch, row_pitch = _pitches(frames, W * C)
    if (frames.stride(3) != 1 or (W > 1 and frames.stride(2) != C) or row_pitch < W * C
            or not (frame_pitch == 0 or frame_pitch >= H * row_pitch)):
        raise ValueError(f"frames must have packed pixels (strides [.., .., {C}, 1]), rows that do not overlap and frames that do not "
                         f"overlap (or a frame stride of 0), got strides {frames.stride()}")
    return frames, F, H, W, frame_pitch, row_pitch


def _out(out, name, shape, dtype, dev):
    t = out.get(name) if out is not None else None
    if t is None:
        return torch.empty(shape, dtype=dtype, device=dev)
    if not isinstance(t, torch.Tensor) or t.dtype != dtype or tuple(t.shape) != shape or t.device != dev:
        raise ValueError(f"out['{name}'] must be a {dtype} tensor of shape {list(shape)} on {dev}")
    return t


def grey_frames(frames: torch.Tensor, order: str = "bgr", out: dict | None = None, normalised: bool = False):
    """The reference's grey frames -- ``cv2.imread(path, cv2.IMREAD_GRAYSCALE)`` (OpenCV 4.13) of a colour PNG of the same pixels,
    bit for bit -- of colour frames on the device.

    frames: uint8 ``[F, H, W, C]`` CUDA tensor, or ``[H, W, C]`` for one frame (then F = 1); C = 3 for ``order`` "bgr" / "rgb",
    4 for "bgra" / "rgba" (alpha is ignored).  Pixels packed (channel stride 1, pixel stride C); rows and frames at any stride
    that does not overlap them, or a frame stride of 0 (one frame for all F).  F <= 65535, sides <= 32767.

    Returns grey uint8 ``[F, H, W]``, the frames ``crop``, ``detect`` and ``flow`` take; with ``normalised=True`` the pair
    (grey, image) where image is fp32 ``[F, 1, H, W]`` equal bit for bit to the reference's ``image / 255.`` (the extractor's
    input): a float32 division, as ``grey.float() / 255`` on the CPU -- not torch's ``/ 255`` of a CUDA tensor, a multiply by
    the reciprocal that is one ulp off on 126 of the 256 levels.  ``out`` takes caller-owned result tensors {"grey": uint8
    [F, H, W] with packed pixels and rows and frames that do not overlap, "image": contiguous fp32 [F, 1, H, W]} on the frames'
    device, which are then the results; they must not overlap the frames.  One launch on the current stream, no allocation when ``out`` holds
    every result, no host synchronisation.  Argument mistakes raise ValueError before anything runs."""
    frames, F, H, W, frame_pitch, row_pitch = _check_frames(frames, order)
    dev = frames.device
    grey = _out(out, "grey", (F, H, W), torch.uint8, dev)
    g_frame, g_row = _pitches(grey, W)
    if grey.stride(2) != 1 and W > 1 or g_row < W or g_frame < H * g_row:
        raise ValueError(f"out['grey'] must have packed pixels and rows and frames that do not overlap, got strides {grey.stride()}")
    image = None
    if normalised:
        image = _out(out, "image", (F, 1, H, W), torch.float32, dev)
        if not image.is_contiguous():
            raise ValueError("out['image'] must be contiguous")
    _lib.cuda_device(frames)
    _lib.call(dev, "opb_grey_frames", frames, frame_pitch, row_pitch, F, H, W, ORDERS[order], grey, g_frame, g_row, image)
    return (grey, image) if normalised else grey
