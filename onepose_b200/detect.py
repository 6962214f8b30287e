"""Object detection by 2D-2D matching on the GPU: the reference's first-frame (and lost-track) detector.

The reference's ``LocalFeatureObjectDetector.detect`` (``src/local_feature_2D_detector/local_feature_2D_detector.py:76-147,
196-230``) runs SuperPoint on the full frame, matches it against ``n_ref_view`` reference views with the caller's 2D-2D
matcher, pulls each view's ``matches0`` to the host, runs ``cv2.estimateAffinePartial2D(ref, query, ransacReprojThreshold=6)``
per view, keeps the box of the view with the most matches and crops it.  Here everything after the matcher stays on the
device (``csrc/detect.cu`` behind ``opb_boxes_from_matches`` / ``opb_estimate_affine_partial``, then ``crop.crop_frames``):

    bbox, inp, K_crop = detect.detect_from_matches(frames_u8, K, ref, query, matches0)

``estimate_affine_partial_2d`` is a numpy drop-in for ``cv2.estimateAffinePartial2D`` (RANSAC) computed on the device;
``LocalFeatureObjectDetector`` is the reference class with reference images in place of the SfM workspace.  The matcher stays
the caller's module, as in the reference.
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib, crop

MAX_VIEWS = 256         # opb_boxes_from_matches' bounds (include/onepose_b200.h)
MAX_REF_POINTS = 8192
MIN_MATCHES = 6         # match_worker: fewer matches give the [0, 0, H, W] box


def _check_params(threshold, max_iters, confidence, refine_iters):
    if not np.isfinite(threshold):
        raise ValueError(f"ransacReprojThreshold must be finite, got {threshold!r}")
    if not 0 < confidence < 1:
        raise ValueError(f"confidence must lie in (0, 1) (OpenCV asserts it), got {confidence!r}")
    if int(max_iters) < 0 or int(refine_iters) < 0:
        raise ValueError(f"maxIters and refineIters must be >= 0, got {max_iters!r}, {refine_iters!r}")


def affine_partial_batch(from_pts: torch.Tensor, to_pts: torch.Tensor, offsets: torch.Tensor, threshold: float = 3.0,
                         max_iters: int = 2000, confidence: float = 0.99, refine_iters: int = 10) -> dict:
    """``cv2.estimateAffinePartial2D(from, to, method=RANSAC, ...)`` for B independent problems in one launch.  from_pts / to_pts
    CUDA [sum n, 2] (used as fp32, as cv2 does), offsets int32 [B + 1] on the same device (problem b is rows offsets[b] ..
    offsets[b+1] - 1).  Returns device tensors: affine f64 [B, 2, 3] (zeros where cv2 returns None), inliers uint8 [sum n]
    (cv2's mask), iterations int32 [B] (the RANSAC loop's) and status int32 [B] (1: a model, 0: None).  No host
    synchronisation."""
    dev = _lib.cuda_device(from_pts)
    _check_params(threshold, max_iters, confidence, refine_iters)
    if from_pts.dim() != 2 or from_pts.shape[1] != 2 or tuple(to_pts.shape) != tuple(from_pts.shape):
        raise ValueError(f"from_pts and to_pts must both be [n, 2], got {list(from_pts.shape)} and {list(to_pts.shape)}")
    if offsets.dtype != torch.int32 or offsets.dim() != 1 or offsets.numel() < 2 or offsets.device != dev or to_pts.device != dev:
        raise ValueError(f"offsets must be int32 [B + 1] on {dev}, with to_pts there too")
    B = offsets.numel() - 1
    f = from_pts.to(torch.float32).contiguous()
    t = to_pts.to(torch.float32).contiguous()
    o = offsets.contiguous()
    out = {"affine": torch.empty(B, 2, 3, dtype=torch.float64, device=dev), "inliers": torch.empty(f.shape[0], dtype=torch.uint8, device=dev),
           "iterations": torch.empty(B, dtype=torch.int32, device=dev), "status": torch.empty(B, dtype=torch.int32, device=dev)}
    _lib.call(dev, "opb_estimate_affine_partial", f, t, o, B, float(threshold), int(max_iters), float(confidence), int(refine_iters), out["affine"],
              out["inliers"] if f.shape[0] else None, out["iterations"], out["status"])
    return out


def estimate_affine_partial_2d(from_pts, to_pts, *, ransacReprojThreshold=3, maxIters=2000, confidence=0.99, refineIters=10, device=None):
    """Drop-in for ``cv2.estimateAffinePartial2D(from_pts, to_pts, ransacReprojThreshold=..., ...)`` (method RANSAC): numpy
    [n, 2] (or [n, 1, 2]) in, ``(affine f64 [2, 3] or None, inliers uint8 [n, 1])`` out, computed on the device.  The samples,
    the mask and the unrefined model are OpenCV 4.13's bit for bit; the refined model agrees to rounding (DESIGN 5.8)."""
    dev = torch.device(device if device is not None else "cuda")
    f = np.asarray(from_pts, dtype=np.float64).reshape(-1, 2).astype(np.float32)
    t = np.asarray(to_pts, dtype=np.float64).reshape(-1, 2).astype(np.float32)
    if f.shape != t.shape:
        raise ValueError(f"from_pts and to_pts must hold the same number of points, got {len(f)} and {len(t)}")
    n = len(f)
    out = affine_partial_batch(torch.from_numpy(f).to(dev), torch.from_numpy(t).to(dev),
                               torch.tensor([0, n], dtype=torch.int32, device=dev), float(ransacReprojThreshold), int(maxIters),
                               float(confidence), int(refineIters))
    mask = out["inliers"].cpu().numpy().reshape(n, 1)
    return (out["affine"][0].cpu().numpy() if int(out["status"][0]) == 1 else None), mask


def _ref_args(ref: dict, dev):
    kp, cnt, size = ref["keypoints"], ref["counts"], ref["sizes"]
    if kp.dim() != 3 or kp.shape[2] != 2 or not 0 < kp.shape[0] <= MAX_VIEWS or not 0 < kp.shape[1] <= MAX_REF_POINTS:
        raise ValueError(f"ref['keypoints'] must be [V, cap, 2] with 1 <= V <= {MAX_VIEWS}, 1 <= cap <= {MAX_REF_POINTS}, got {list(kp.shape)}")
    V = int(kp.shape[0])
    if tuple(cnt.shape) != (V,) or tuple(size.shape) != (V, 2) or cnt.dtype.is_floating_point or size.dtype.is_floating_point:
        raise ValueError(f"ref['counts'] must be integer [{V}] and ref['sizes'] integer [{V}, 2] (H, W)")
    return (kp.to(dev, torch.float32).contiguous(), cnt.to(dev, torch.int32).contiguous(), size.to(dev, torch.int32).contiguous())


def boxes_from_matches(ref: dict, query: dict, matches0: torch.Tensor, query_size) -> dict:
    """``match_worker`` + ``detect_by_matching`` for B frames against V reference views, on the device.
    ref: {"keypoints": [V, cap_ref, 2], "counts": [V], "sizes": [V, 2] (H, W)}; query: {"keypoints": [B, cap_q, 2], "counts":
    [B]} (``SuperPoint.forward_padded``'s layout); matches0 int32 / int64 [B, V, cap_ref] (the matcher's matches0 of frame b
    against view v; an entry counts iff 0 <= m < counts[b]); query_size (H, W) of the frames.  Returns device tensors: box int32
    [B, 4] (the input of ``crop.crop_frames``), view int32 [B], n_matches int32 [B], affine f64 [B, 2, 3] and status int32 [B]:
    1 for the box of the affine, 2 where no view has 6 matches and the box is the reference's [0, 0, H, W], 0 for the empty box
    where the reference fails (the chosen view has no affine) or a corner leaves int32.  No host synchronisation."""
    dev = _lib.cuda_device(matches0)
    rk, rc, rs = _ref_args(ref, dev)
    V, cap_ref = int(rk.shape[0]), int(rk.shape[1])
    qk, qc = query["keypoints"], query["counts"]
    if qk.dim() != 3 or qk.shape[2] != 2 or qk.shape[1] == 0 or qc.dim() != 1 or qc.shape[0] != qk.shape[0] or qc.dtype.is_floating_point:
        raise ValueError(f"query must hold keypoints [B, cap, 2] and integer counts [B], got {list(qk.shape)} and {list(qc.shape)}")
    B = int(qk.shape[0])
    if matches0.dtype not in (torch.int32, torch.int64) or tuple(matches0.shape) != (B, V, cap_ref):
        raise ValueError(f"matches0 must be int32 or int64 [{B}, {V}, {cap_ref}], got {matches0.dtype} {list(matches0.shape)}")
    H, W = (int(v) for v in query_size)
    if H <= 0 or W <= 0:
        raise ValueError(f"query_size must be positive (H, W), got {query_size!r}")
    qk = qk.to(dev, torch.float32).contiguous()
    qc = qc.to(dev, torch.int32).contiguous()
    m = matches0.contiguous()
    out = {"box": torch.empty(B, 4, dtype=torch.int32, device=dev), "view": torch.empty(B, dtype=torch.int32, device=dev),
           "n_matches": torch.empty(B, dtype=torch.int32, device=dev), "affine": torch.empty(B, 2, 3, dtype=torch.float64, device=dev),
           "status": torch.empty(B, dtype=torch.int32, device=dev)}
    _lib.call(dev, "opb_boxes_from_matches", rk, rc, rs, V, cap_ref, qk, qc, int(qk.shape[1]), m, int(m.dtype == torch.int64), B, H, W, out["box"],
              out["view"], out["n_matches"], out["affine"], out["status"])
    return out


def detect_from_matches(frames_u8: torch.Tensor, K: torch.Tensor, ref: dict, query: dict, matches0: torch.Tensor, crop_size: int = 512):
    """``detect_by_matching`` and ``crop_img_by_bbox`` (local_feature_2D_detector.py:135-147, 160-186, 222-228) for B frames:
    frames uint8 [B, H, W] CUDA, K [3, 3] or [B, 3, 3], ref / query / matches0 as in ``boxes_from_matches``.  Returns the
    reference's triple (bbox int32 [B, 4], image_crop fp32 [B, 1, S, S], K_crop f64 [B, 3, 3]) on the device.  A frame whose
    box is empty gets a zero image, hence no key points and 0 inliers downstream.  No host synchronisation."""
    _, _, H, W = crop._frames_args(frames_u8)
    bbox = boxes_from_matches(ref, query, matches0, (H, W))["box"]
    out = crop.crop_frames(frames_u8, bbox, K, crop_size)
    return bbox, out["image"], out["K_crop"]


def _pad(rows, cap, dev):
    out = torch.zeros(len(rows), cap, 2, dtype=torch.float32, device=dev)
    for i, r in enumerate(rows):
        out[i, :len(r)] = r
    return out


class LocalFeatureObjectDetector:
    """The reference class (local_feature_2D_detector.py:43-259) with the reference views given as images: ``ref_images`` is a
    list of grey uint8 [H, W] images (numpy or torch) in the reference's sampling order, ``images[idx]`` for ``idx in range(1,
    len(images), len(images) // n_ref_view)`` of its COLMAP model (INTEGRATION shows how to load them).  ``extractor`` is a
    ``SuperPoint``; ``matcher`` any torch module taking the reference's match dict and returning ``matches0`` [1, n0].  The
    views are extracted once; their features stay on the device.  Writing crops and K to disk stays with the caller."""

    def __init__(self, extractor, matcher, ref_images, crop_size: int = 512, device=None):
        self.extractor, self.matcher, self.crop_size = extractor, matcher, int(crop_size)
        self.device = torch.device(device if device is not None else "cuda")
        if not 0 < len(ref_images) <= MAX_VIEWS:
            raise ValueError(f"1 to {MAX_VIEWS} reference views, got {len(ref_images)}")
        self.views = []
        for img in ref_images:
            img = torch.as_tensor(np.asarray(img) if not torch.is_tensor(img) else img)
            if img.dtype != torch.uint8 or img.dim() != 2:
                raise ValueError(f"reference views must be grey uint8 [H, W], got {img.dtype} {list(img.shape)}")
            det = extractor.forward(img.to(self.device)[None, None].float() / 255)       # pack_extract_data: image / 255.0
            self.views.append({"keypoints": det["keypoints"][0], "scores": det["scores"][0], "descriptors": det["descriptors"][0],
                               "size": tuple(int(v) for v in img.shape)})
        cap = max(max(len(v["keypoints"]) for v in self.views), 1)
        if cap > MAX_REF_POINTS:
            raise ValueError(f"a reference view has {cap} key points; at most {MAX_REF_POINTS} are supported")
        self.ref = {"keypoints": _pad([v["keypoints"] for v in self.views], cap, self.device),
                    "counts": torch.tensor([len(v["keypoints"]) for v in self.views], dtype=torch.int32, device=self.device),
                    "sizes": torch.tensor([v["size"] for v in self.views], dtype=torch.int32, device=self.device)}

    def _match_data(self, view, kp, sc, de, frame_hw):
        """pack_match_data's dict; image0 / image1 carry only their shape, (1, 1) + size[::-1] as the reference builds it."""
        one = torch.empty(1, device=self.device)
        return {"keypoints0": view["keypoints"][None], "scores0": view["scores"][None], "descriptors0": view["descriptors"][None],
                "keypoints1": kp[None], "scores1": sc[None], "descriptors1": de[None],
                "image0": one.expand(1, 1, view["size"][1], view["size"][0]), "image1": one.expand(1, 1, frame_hw[1], frame_hw[0])}

    @torch.no_grad()
    def detect(self, frames_u8: torch.Tensor, K: torch.Tensor):
        """``detect`` for B frames uint8 [B, H, W] on the device and K [3, 3] or [B, 3, 3]: one extractor call (one host
        synchronisation, for the key-point counts the matcher needs at exact size), one matcher call per (frame, view), then
        ``detect_from_matches``.  Returns (bbox int32 [B, 4], image_crop fp32 [B, 1, S, S], K_crop f64 [B, 3, 3])."""
        _, B, H, W = crop._frames_args(frames_u8)
        det = self.extractor.forward(frames_u8[:, None].float() / 255)
        cap_ref = int(self.ref["keypoints"].shape[1])
        matches0 = torch.full((B, len(self.views), cap_ref), -1, dtype=torch.int64, device=frames_u8.device)
        for b in range(B):
            kp, sc, de = det["keypoints"][b], det["scores"][b], det["descriptors"][b]
            for v, view in enumerate(self.views):
                m = self.matcher(self._match_data(view, kp, sc, de, (H, W)))["matches0"][0]
                matches0[b, v, :m.shape[0]] = m
        cap_q = max(max(len(k) for k in det["keypoints"]), 1)
        query = {"keypoints": _pad(det["keypoints"], cap_q, frames_u8.device),
                 "counts": torch.tensor([len(k) for k in det["keypoints"]], dtype=torch.int32).to(frames_u8.device)}
        return detect_from_matches(frames_u8, K, self.ref, query, matches0, self.crop_size)

    def previous_pose_detect(self, frames_u8, K, pre_pose, bbox3d):
        """The reference method for B frames: ``crop.previous_pose_detect``."""
        return crop.previous_pose_detect(frames_u8, K, pre_pose, bbox3d, self.crop_size)
