"""Pose-guided crop on the GPU: from the pose of the previous frame to the extractor's input for the next.

The reference's live loop (``inference_demo.py:193-247``) crops every frame after the first around the object's 3D box
projected by the previous pose: ``previous_pose_detect`` (``local_feature_2D_detector.py:232-259``), host numpy and
``cv2.warpAffine`` between a pose that ``pnp.poses_from_matches`` leaves on the device and an extractor that reads from it.
``boxes_from_poses``, ``crop_frames`` and ``previous_pose_detect`` do it for B frames on the device, with no host
synchronisation (``csrc/crop.cu`` behind ``opb_boxes_from_poses`` / ``opb_crop_resize``); the live step becomes

    bbox, inp, K_crop = crop.previous_pose_detect(frames_u8, K, res_prev["pose"], bbox3d)
    det = extractor.forward_padded(inp)
    out = matcher.match_frames(det["descriptors"], return_conf=False, lengths=det["counts"])
    res = pnp.poses_from_matches(K_crop, det["keypoints"], keypoints3d, out["matches0"], out["matching_scores0"], scale=1000)

The cropped pixels are ``cv2.warpAffine``'s bit for bit, and the 2x3 transforms ``cv2.getAffineTransform``'s (OpenCV 4.13).
``reproj``, ``get_K_crop_resize`` and ``get_image_crop_resize`` mirror the reference's functions of those names
(``src/utils/vis_utils.py:209-236``, ``src/utils/data_utils.py:233-272``): numpy in, numpy out, computed on the device.
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib

MAX_SIDE = 32767        # the box sides and |coordinates| opb_crop_resize accepts (include/onepose_b200.h)
MAX_COORD = 1 << 20
MAX_FRAMES = 65535


def _per_frame(t: torch.Tensor, B: int, shape: tuple, name: str, dev) -> torch.Tensor:
    """``t`` of ``shape`` (shared by the frames) or ``[B, *shape]`` -> contiguous f64 ``[B, *shape]`` on ``dev``."""
    if not t.dtype.is_floating_point:
        raise ValueError(f"{name} must be a floating-point tensor, got {t.dtype}")
    if tuple(t.shape) == shape:
        t = t.expand(B, *shape)
    elif tuple(t.shape) != (B, *shape):
        raise ValueError(f"{name} must be {list(shape)} or {[B, *shape]}, got {list(t.shape)}")
    return t.to(device=dev, dtype=torch.float64).contiguous()


def _project(K, pose, pts, want_proj: bool):
    dev = _lib.cuda_device(pose)
    if pose.dim() != 3 or tuple(pose.shape[1:]) not in ((3, 4), (4, 4)) or not pose.dtype.is_floating_point:
        raise ValueError(f"pose must be a floating-point [B, 3, 4] or [B, 4, 4], got {pose.dtype} {list(pose.shape)}")
    B = int(pose.shape[0])
    if not 0 < B <= MAX_FRAMES:
        raise ValueError(f"1 to {MAX_FRAMES} frames per call, got {B}")
    if pts.dim() not in (2, 3) or pts.shape[-1] != 3 or pts.shape[-2] == 0:
        raise ValueError(f"bbox3d must be [n, 3] or [B, n, 3], got {list(pts.shape)}")
    n = int(pts.shape[-2])
    K = _per_frame(K, B, (3, 3), "K", dev)
    pts = _per_frame(pts, B, (n, 3), "bbox3d", dev)
    pose = pose[:, :3].to(torch.float64).contiguous()
    box = torch.empty(B, 4, dtype=torch.int32, device=dev)
    proj = torch.empty(B, n, 2, dtype=torch.float64, device=dev) if want_proj else None
    _lib.call(dev, "opb_boxes_from_poses", K, pose, pts, B, n, proj, box)
    return box, proj


def boxes_from_poses(K: torch.Tensor, pose: torch.Tensor, bbox3d: torch.Tensor) -> torch.Tensor:
    """The boxes ``previous_pose_detect`` crops (local_feature_2D_detector.py:246-249) for B frames: ``reproj`` of the object's
    box corners, min / max, ``astype(np.int32)`` (truncation towards zero).  K [3,3] or [B,3,3], pose [B,3,4] or [B,4,4]
    (``poses_from_matches``' ``pose`` / ``pose_homo``), bbox3d [8,3] or [B,8,3] -- CUDA tensors, computed in fp64.  Returns int32
    [B,4] = [x0, y0, x1, y1] on the device; a non-finite projection or one outside int32 gives the empty box [0,0,0,0], which
    ``crop_frames`` answers with status 0.  No host synchronisation."""
    return _project(K, pose, bbox3d, False)[0]


def _frames_args(frames: torch.Tensor):
    dev = _lib.cuda_device(frames)
    if frames.dtype != torch.uint8 or frames.dim() != 3:
        raise ValueError(f"frames must be uint8 [B, H, W], got {frames.dtype} {list(frames.shape)}")
    B, H, W = (int(v) for v in frames.shape)
    if not 0 < B <= MAX_FRAMES or not 0 < H <= MAX_SIDE or not 0 < W <= MAX_SIDE:
        raise ValueError(f"frames must be 1..{MAX_FRAMES} images of 1..{MAX_SIDE} pixels a side, got {list(frames.shape)}")
    if frames.stride(2) != 1 or frames.stride(1) < W or frames.stride(0) < 0:
        raise ValueError(f"frames must have unit pixel stride and rows that do not overlap, got strides {frames.stride()}")
    return dev, B, H, W


def _colour_frames_args(frames: torch.Tensor):
    dev = _lib.cuda_device(frames)
    if frames.dtype != torch.uint8 or frames.dim() != 4 or frames.shape[-1] not in (3, 4):
        raise ValueError(f"frames must be uint8 [B, H, W, C] with C = 3 or 4, got {frames.dtype} {list(frames.shape)}")
    B, H, W, C = (int(v) for v in frames.shape)
    if not 0 < B <= MAX_FRAMES or not 0 < H <= MAX_SIDE or not 0 < W <= MAX_SIDE:
        raise ValueError(f"frames must be 1..{MAX_FRAMES} images of 1..{MAX_SIDE} pixels a side, got {list(frames.shape)}")
    row_pitch = frames.stride(1) if H > 1 else W * C          # the stride of a dimension of size 1 addresses nothing
    if frames.stride(3) != 1 or (W > 1 and frames.stride(2) != C) or row_pitch < W * C:
        raise ValueError(f"frames must have packed pixels (strides [.., .., {C}, 1]) and rows that do not overlap, got strides {frames.stride()}")
    return dev, B, H, W, C, row_pitch


def _boxes(boxes: torch.Tensor, B: int, dev) -> torch.Tensor:
    if boxes.dtype != torch.int32 or tuple(boxes.shape) != (B, 4):
        raise ValueError(f"boxes must be int32 [{B}, 4], got {boxes.dtype} {list(boxes.shape)}")
    return boxes.to(dev).contiguous()


def _indices(index, n: int, bound: int, name: str, dev) -> torch.Tensor:
    """An integer [n] sequence or tensor -> contiguous int32 [n] on ``dev``.  Other integer dtypes are clamped to [-1, bound]
    first, so that no entry wraps into the range the kernels accept (which lies inside [0, bound)); the kernels reject what
    is out of range.  No host synchronisation for a device tensor."""
    t = torch.as_tensor(index)
    if t.dtype.is_floating_point or t.dtype == torch.bool or t.is_complex() or tuple(t.shape) != (n,):
        raise ValueError(f"{name} must be an integer [{n}] sequence or tensor, got {t.dtype} {list(t.shape)}")
    t = t.to(dev)
    if t.dtype != torch.int32:
        t = t.clamp(-1, bound).to(torch.int32)
    return t.contiguous()


def crop_frames(frames: torch.Tensor, boxes: torch.Tensor, K: torch.Tensor, crop_size: int = 512, frame_index=None) -> dict:
    """``crop_img_by_bbox`` (local_feature_2D_detector.py:160-186) and the ``/ 255`` after it, for B frames: frames uint8 [B,H,W]
    CUDA (full grey camera frames; any row and frame stride, unit pixel stride), boxes int32 [B,4] = [x0, y0, x1, y1], K [3,3] or
    [B,3,3], crop_size S (S % 8 == 0).  Returns device tensors: image fp32 [B,1,S,S] (the extractor's input; the pixels are
    ``cv2.warpAffine``'s), K_crop f64 [B,3,3], trans f64 [B,2,2,3] (T1 and T2: ``T2 @ T1`` in homogeneous form maps a frame
    position into the crop) and status int32 [B]: 0, with a zero image and K_crop = K, for a box with x1 <= x0 or y1 <= y0, a
    side over 32767 or a coordinate beyond 2^20.  A zero image gives no key points, so the failure shows as 0 inliers in the
    pose of that frame.  No host synchronisation.

    With ``frame_index`` (integer [B], on the device for no host synchronisation), frames is [F,H,W] and crop b reads frame
    frame_index[b]: several boxes per frame, each crop equal to the one ``crop_frames(frames[frame_index], ...)`` makes without
    the copy.  boxes and K are then per crop; an index outside [0, F) gives status 0 as a rejected box does."""
    dev, B, H, W = _frames_args(frames)
    S = int(crop_size)
    if S <= 0 or S % 8 or S > MAX_SIDE:
        raise ValueError(f"crop_size must be a positive multiple of 8 up to {MAX_SIDE}, got {crop_size!r}")
    F = B
    if frame_index is not None:
        frame_index = torch.as_tensor(frame_index)
        B = int(frame_index.shape[0]) if frame_index.dim() == 1 else 0
        if not 0 < B <= MAX_FRAMES:
            raise ValueError(f"frame_index must be an integer [B] sequence or tensor with 1 <= B <= {MAX_FRAMES}")
        frame_index = _indices(frame_index, B, F, "frame_index", dev)
    boxes = _boxes(boxes, B, dev)
    K = _per_frame(K, B, (3, 3), "K", dev)
    out = {"image": torch.empty(B, 1, S, S, dtype=torch.float32, device=dev), "K_crop": torch.empty(B, 3, 3, dtype=torch.float64, device=dev),
           "trans": torch.empty(B, 2, 2, 3, dtype=torch.float64, device=dev), "status": torch.empty(B, dtype=torch.int32, device=dev)}
    if frame_index is None:
        _lib.call(dev, "opb_crop_resize", frames, frames.stride(0), frames.stride(1), B, H, W, boxes, K, S, out["image"], out["K_crop"],
                  out["trans"], out["status"])
    else:
        _lib.call(dev, "opb_crop_resize_indexed", frames, frames.stride(0), frames.stride(1), F, H, W, frame_index, B, boxes, K, S, out["image"],
                  out["K_crop"], out["trans"], out["status"])
    return out


def crop_frames_colour(frames: torch.Tensor, boxes: torch.Tensor, K: torch.Tensor, crop_size: int = 512, frame_index=None) -> dict:
    """``crop_frames``' two warps on colour frames, kept in uint8: the crops ``parse_scanned_data.py``'s ``parse_video`` writes
    (``:151-159``), ``cv2.warpAffine`` of the BGR frame and then of its first-stage crop.  frames uint8 [B,H,W,C] CUDA with C = 3
    or 4 (packed pixels; any row and frame stride), boxes int32 [B,4], K [3,3] or [B,3,3], crop_size S (S % 8 == 0).

    Returns device tensors: image uint8 [B,S,S,C], channel c equal bit for bit to ``cv2.warpAffine`` of the C-channel image
    (which warps each channel plane as the grey warp does), and K_crop, trans and status exactly as ``crop_frames`` returns
    them.  A rejected box gives a zero crop.  ``frame_index`` is ``crop_frames``': frames is then [F,H,W,C] and crop b reads frame
    frame_index[b].  No host synchronisation.

    The reference turns a crop grey only after it: ``cv2.imwrite`` of the colour crop, then ``IMREAD_GRAYSCALE``.  Making the
    frame grey first and cropping the grey frame gives other pixels, so ``frames.grey_frames(image)`` is the extractor's
    input for a scanned sequence, not ``crop_frames(grey_frames(frames))``."""
    dev, B, H, W, C, row_pitch = _colour_frames_args(frames)
    S = int(crop_size)
    if S <= 0 or S % 8 or S > MAX_SIDE:
        raise ValueError(f"crop_size must be a positive multiple of 8 up to {MAX_SIDE}, got {crop_size!r}")
    F = B
    if frame_index is not None:
        frame_index = torch.as_tensor(frame_index)
        B = int(frame_index.shape[0]) if frame_index.dim() == 1 else 0
        if not 0 < B <= MAX_FRAMES:
            raise ValueError(f"frame_index must be an integer [B] sequence or tensor with 1 <= B <= {MAX_FRAMES}")
        frame_index = _indices(frame_index, B, F, "frame_index", dev)
    boxes = _boxes(boxes, B, dev)
    K = _per_frame(K, B, (3, 3), "K", dev)
    out = {"image": torch.empty(B, S, S, C, dtype=torch.uint8, device=dev), "K_crop": torch.empty(B, 3, 3, dtype=torch.float64, device=dev),
           "trans": torch.empty(B, 2, 2, 3, dtype=torch.float64, device=dev), "status": torch.empty(B, dtype=torch.int32, device=dev)}
    _lib.call(dev, "opb_crop_resize_colour", frames, frames.stride(0), row_pitch, F, H, W, C, frame_index, B, boxes, K, S, out["image"],
              out["K_crop"], out["trans"], out["status"])
    return out


def previous_pose_detect(frames: torch.Tensor, K: torch.Tensor, pre_pose: torch.Tensor, bbox3d: torch.Tensor, crop_size: int = 512,
                         frame_index=None):
    """The reference method of this name (local_feature_2D_detector.py:232-259) for B frames on the device: frames uint8 [B,H,W]
    in place of the image path, K, pre_pose and bbox3d as in ``boxes_from_poses``.  Returns its triple (bbox int32 [B,4],
    image_crop fp32 [B,1,S,S], K_crop f64 [B,3,3]).  No host synchronisation.

    With ``frame_index`` (as in ``crop_frames``), frames is [F,H,W] and B = len(frame_index) objects are cropped from them: K,
    pre_pose and bbox3d are per object (or shared), and object b's box is cut from frame frame_index[b]."""
    _frames_args(frames)
    bbox = boxes_from_poses(K, pre_pose, bbox3d)
    out = crop_frames(frames, bbox, K, crop_size, frame_index)
    return bbox, out["image"], out["K_crop"]


# ---- the reference's numpy functions, computed on the device ----

def _np_box(box) -> np.ndarray:
    b = np.asarray(box, dtype=np.float64).reshape(-1)
    if b.shape != (4,) or not np.all(np.isfinite(b)) or not np.all(b == np.rint(b)):
        raise ValueError(f"box must be four integers [x0, y0, x1, y1], got {box!r}")
    w, h = b[2] - b[0], b[3] - b[1]
    if not (0 < w <= MAX_SIDE and 0 < h <= MAX_SIDE and np.all(np.abs(b) <= MAX_COORD)):
        raise ValueError(f"box {b.astype(np.int64).tolist()} is empty or beyond what cv2.warpAffine addresses")
    return b.astype(np.int32)


def _np_shape(resize_shape):
    h, w = (int(v) for v in resize_shape)
    if not (0 < h <= MAX_SIDE and 0 < w <= MAX_SIDE):
        raise ValueError(f"resize_shape must be [h, w] within 1..{MAX_SIDE}, got {resize_shape!r}")
    return h, w


def _warp_crop_np(image, box, K, resize_shape, device):
    dev = torch.device(device if device is not None else "cuda")
    if dev.type != "cuda":
        raise RuntimeError("onepose_b200 has no CPU path: tensors must be on a CUDA device")
    box = _np_box(box)
    h, w = _np_shape(resize_shape)
    frames = out = Kd = Kc = None
    fargs = (None, 0, 0, 1, 0, 0)
    if image is not None:
        image = np.asarray(image)
        if image.dtype != np.uint8 or image.ndim != 2:
            raise ValueError(f"image must be uint8 [H, W], got {image.dtype} {list(image.shape)}")
        frames = torch.from_numpy(np.ascontiguousarray(image))[None].to(dev)
        _, _, H, W = _frames_args(frames)
        out = torch.empty(1, h, w, dtype=torch.uint8, device=dev)
        fargs = (frames, frames.stride(0), frames.stride(1), 1, H, W)
    if K is not None:
        K = np.asarray(K, dtype=np.float64)
        if K.shape != (3, 3):
            raise ValueError(f"K_orig must be [3, 3], got {list(K.shape)}")
        Kd = torch.from_numpy(np.ascontiguousarray(K)).to(dev)
        Kc = torch.empty(3, 3, dtype=torch.float64, device=dev)
    trans = torch.empty(2, 3, dtype=torch.float64, device=dev)
    boxd = torch.from_numpy(box).to(dev)
    _lib.call(dev, "opb_warp_crop_u8", *fargs, boxd, Kd, h, w, out, trans, Kc)
    return (out[0].cpu().numpy() if out is not None else None, trans.cpu().numpy(), Kc.cpu().numpy() if K is not None else None)


def get_image_crop_resize(image, box, resize_shape, device=None):
    """Drop-in for the reference function (data_utils.py:233-247): image uint8 [H,W], box [x0, y0, x1, y1] (integers),
    resize_shape [h, w] -> (image_crop uint8 [h,w], trans_crop_homo f64 [3,3]), both bit-equal to the reference's with OpenCV
    4.13.  An empty box raises ValueError (the reference raises inside cv2)."""
    img, trans, _ = _warp_crop_np(image, box, None, resize_shape, device)
    return img, np.concatenate([trans, np.array([[0, 0, 1]])], axis=0)


def get_K_crop_resize(box, K_orig, resize_shape, device=None):
    """Drop-in for the reference function (data_utils.py:250-272) for K_orig [3,3] -> (K_crop [3,3], K_crop_homo [3,4]) f64."""
    _, _, K_crop = _warp_crop_np(None, box, K_orig, resize_shape, device)
    return K_crop, np.concatenate([K_crop, np.zeros((3, 1))], axis=1)


def reproj(K, pose, pts_3d, device=None):
    """Drop-in for the reference ``reproj`` (vis_utils.py:209-236): K [3,3], pose [3,4] or [4,4], pts_3d [n,3] -> [n,2] f64."""
    dev = torch.device(device if device is not None else "cuda")
    K, pose = np.asarray(K, dtype=np.float64), np.asarray(pose, dtype=np.float64)
    pts = np.asarray(pts_3d, dtype=np.float64).reshape(-1, 3)
    if K.shape != (3, 3) or pose.shape not in ((3, 4), (4, 4)):
        raise ValueError(f"K must be [3, 3] and pose [3, 4] or [4, 4], got {list(K.shape)} and {list(pose.shape)}")
    _, proj = _project(torch.from_numpy(K).to(dev), torch.from_numpy(pose)[None].to(dev), torch.from_numpy(pts).to(dev), True)
    return proj[0].cpu().numpy()
