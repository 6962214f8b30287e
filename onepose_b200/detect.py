"""Object detection by 2D-2D matching on the GPU: the reference's first-frame (and lost-track) detector.

The reference's ``LocalFeatureObjectDetector.detect`` (``src/local_feature_2D_detector/local_feature_2D_detector.py:76-147,
196-230``) runs SuperPoint on the full frame, matches it against ``n_ref_view`` reference views with the caller's 2D-2D
matcher, pulls each view's ``matches0`` to the host, runs ``cv2.estimateAffinePartial2D(ref, query, ransacReprojThreshold=6)``
per view, keeps the box of the view with the most matches and crops it.  Here everything after the matcher stays on the
device (``csrc/detect.cu`` behind ``opb_boxes_from_matches`` / ``opb_estimate_affine_partial``, then ``crop.crop_frames``):

    bbox, inp, K_crop = detect.detect_from_matches(frames_u8, K, ref, query, matches0)

``estimate_affine_partial_2d`` is a numpy drop-in for ``cv2.estimateAffinePartial2D`` (RANSAC) computed on the device;
``LocalFeatureObjectDetector`` is the reference class with reference images in place of the SfM workspace.  The matcher stays
the caller's module, as in the reference.  For several objects in the same frames, ``boxes_from_matches_objects`` /
``detect_from_matches_objects`` (``opb_boxes_from_matches_objects``) take (frame, object) pairs against one table of every
object's views, and ``ObjectDetectors`` extracts the frames once for all of them.
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib, crop

MAX_VIEWS = 256         # opb_boxes_from_matches' bounds (include/onepose_b200.h)
MAX_REF_POINTS = 8192
MIN_MATCHES = 6         # match_worker: fewer matches give the [0, 0, H, W] box
MAX_TABLE_VIEWS = 2**31 - 1     # the views of all objects in one opb_boxes_from_matches_objects table
INT32_MAX = 2**31 - 1           # maxIters and refineIters reach the library as int32; larger values are refused, not wrapped


def _check_params(threshold, max_iters, confidence, refine_iters):
    if not np.isfinite(threshold):
        raise ValueError(f"ransacReprojThreshold must be finite, got {threshold!r}")
    if not 0 < confidence < 1:
        raise ValueError(f"confidence must lie in (0, 1) (OpenCV asserts it), got {confidence!r}")
    if not 0 <= int(max_iters) <= INT32_MAX or not 0 <= int(refine_iters) <= INT32_MAX:
        raise ValueError(f"maxIters and refineIters must lie in [0, 2**31 - 1], got {max_iters!r}, {refine_iters!r}")


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
    the mask and the unrefined model are OpenCV 4.13's bit for bit; the refined model follows its LMSolver step for step and
    was measured within 1.7e-13 relative of cv2's (refineIters 1 to 1000, coordinates up to 1e6; DESIGN 5.8).  maxIters and
    refineIters above 2**31 - 1 are refused, where cv2 casts them to int."""
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


def _ref_args(ref: dict, dev, max_views: int = MAX_VIEWS):
    kp, cnt, size = ref["keypoints"], ref["counts"], ref["sizes"]
    if kp.dim() != 3 or kp.shape[2] != 2 or not 0 < kp.shape[0] <= max_views or not 0 < kp.shape[1] <= MAX_REF_POINTS:
        raise ValueError(f"ref['keypoints'] must be [V, cap, 2] with 1 <= V <= {max_views}, 1 <= cap <= {MAX_REF_POINTS}, got {list(kp.shape)}")
    V = int(kp.shape[0])
    if tuple(cnt.shape) != (V,) or tuple(size.shape) != (V, 2) or cnt.dtype.is_floating_point or size.dtype.is_floating_point:
        raise ValueError(f"ref['counts'] must be integer [{V}] and ref['sizes'] integer [{V}, 2] (H, W)")
    return (kp.to(dev, torch.float32).contiguous(), cnt.to(dev, torch.int32).contiguous(), size.to(dev, torch.int32).contiguous())


def _query_args(query: dict):
    qk, qc = query["keypoints"], query["counts"]
    if qk.dim() != 3 or qk.shape[2] != 2 or qk.shape[1] == 0 or qc.dim() != 1 or qc.shape[0] != qk.shape[0] or qc.dtype.is_floating_point:
        raise ValueError(f"query must hold keypoints [B, cap, 2] and integer counts [B], got {list(qk.shape)} and {list(qc.shape)}")
    return qk, qc


def _size_args(query_size):
    H, W = (int(v) for v in query_size)
    if H <= 0 or W <= 0:
        raise ValueError(f"query_size must be positive (H, W), got {query_size!r}")
    return H, W


def _outputs(B: int, dev) -> dict:
    return {"box": torch.empty(B, 4, dtype=torch.int32, device=dev), "view": torch.empty(B, dtype=torch.int32, device=dev),
            "n_matches": torch.empty(B, dtype=torch.int32, device=dev), "affine": torch.empty(B, 2, 3, dtype=torch.float64, device=dev),
            "status": torch.empty(B, dtype=torch.int32, device=dev)}


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
    qk, qc = _query_args(query)
    B = int(qk.shape[0])
    if matches0.dtype not in (torch.int32, torch.int64) or tuple(matches0.shape) != (B, V, cap_ref):
        raise ValueError(f"matches0 must be int32 or int64 [{B}, {V}, {cap_ref}], got {matches0.dtype} {list(matches0.shape)}")
    H, W = _size_args(query_size)
    qk = qk.to(dev, torch.float32).contiguous()
    qc = qc.to(dev, torch.int32).contiguous()
    m = matches0.contiguous()
    out = _outputs(B, dev)
    _lib.call(dev, "opb_boxes_from_matches", rk, rc, rs, V, cap_ref, qk, qc, int(qk.shape[1]), m, int(m.dtype == torch.int64), B, H, W, out["box"],
              out["view"], out["n_matches"], out["affine"], out["status"])
    return out


def boxes_from_matches_objects(refs: dict, view_first, view_count, query: dict, query_index, matches0: torch.Tensor, query_size) -> dict:
    """``boxes_from_matches`` for B (frame, object) pairs in one launch, each against its own object's reference views.
    refs: the views of every object in one table, {"keypoints": [n_views, cap_ref, 2], "counts": [n_views], "sizes": [n_views,
    2]}; view_first / view_count integer [B]: pair b's object is views view_first[b] .. + view_count[b] - 1 (1 <= count <= 256);
    query: the frames' key points as in ``boxes_from_matches``, one row per frame; query_index integer [B]: the row of pair b's
    frame, so that a frame shared by several pairs is extracted once; matches0 int32 / int64 [B, V_max, cap_ref]: row [b, v]
    is the matcher's matches0 of pair b's frame against its object's view v (rows past view_count[b] are never read).  The
    index tensors may live on the host or the device; on the device there is no host synchronisation.  Returns what
    ``boxes_from_matches`` returns, per pair, with ``view`` the index among the pair's own views: pair b's results equal those of
    ``boxes_from_matches`` on its object's views and its frame alone, bit for bit.  A pair whose view range leaves the table,
    whose count is outside [1, V_max] or whose query row does not exist gets status 0, the empty box, view 0 and n_matches 0."""
    dev = _lib.cuda_device(matches0)
    rk, rc, rs = _ref_args(refs, dev, MAX_TABLE_VIEWS)
    n_views, cap_ref = int(rk.shape[0]), int(rk.shape[1])
    qk, qc = _query_args(query)
    n_query = int(qk.shape[0])
    if (matches0.dtype not in (torch.int32, torch.int64) or matches0.dim() != 3 or matches0.shape[0] == 0 or not 0 < matches0.shape[1] <= MAX_VIEWS
            or matches0.shape[2] != cap_ref):
        raise ValueError(f"matches0 must be int32 or int64 [B, V_max, {cap_ref}] with B >= 1 and 1 <= V_max <= {MAX_VIEWS}, got "
                         f"{matches0.dtype} {list(matches0.shape)}")
    B, V_max = int(matches0.shape[0]), int(matches0.shape[1])
    H, W = _size_args(query_size)
    vf = crop._indices(view_first, B, n_views, "view_first", dev)
    vc = crop._indices(view_count, B, V_max + 1, "view_count", dev)
    qi = crop._indices(query_index, B, n_query, "query_index", dev)
    qk = qk.to(dev, torch.float32).contiguous()
    qc = qc.to(dev, torch.int32).contiguous()
    m = matches0.contiguous()
    out = _outputs(B, dev)
    _lib.call(dev, "opb_boxes_from_matches_objects", rk, rc, rs, n_views, cap_ref, vf, vc, V_max, qk, qc, n_query, int(qk.shape[1]), qi, m,
              int(m.dtype == torch.int64), B, H, W, out["box"], out["view"], out["n_matches"], out["affine"], out["status"])
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


def detect_from_matches_objects(frames_u8: torch.Tensor, frame_index, K: torch.Tensor, refs: dict, view_first, view_count, query: dict,
                                matches0: torch.Tensor, crop_size: int = 512):
    """``detect_from_matches`` for B (frame, object) pairs: frames uint8 [F, H, W] CUDA, frame_index integer [B] (pair b's frame,
    which is also its row of ``query``: the frames' key points [F, cap, 2] and counts [F]), K [3, 3] or [B, 3, 3] per pair, refs /
    view_first / view_count / matches0 as in ``boxes_from_matches_objects``.  One detection launch and one crop launch, every
    crop cut from its frame without copying the frames.  Returns the reference's triple per pair (bbox int32 [B, 4], image_crop
    fp32 [B, 1, S, S], K_crop f64 [B, 3, 3]).  No host synchronisation with the index tensors on the device."""
    dev, F, H, W = crop._frames_args(frames_u8)
    if query["counts"].dim() != 1 or query["counts"].shape[0] != F:
        raise ValueError(f"query must hold one row per frame ({F}), got counts {list(query['counts'].shape)}")
    S = int(crop_size)
    if S <= 0 or S % 8 or S > crop.MAX_SIDE:
        raise ValueError(f"crop_size must be a positive multiple of 8 up to {crop.MAX_SIDE}, got {crop_size!r}")
    B = int(matches0.shape[0]) if matches0.dim() == 3 else 0
    if not 0 < B <= crop.MAX_FRAMES:
        raise ValueError(f"matches0 must be [B, V_max, cap_ref] with 1 <= B <= {crop.MAX_FRAMES}, got {list(matches0.shape)}")
    K = crop._per_frame(K, B, (3, 3), "K", dev)
    fi = crop._indices(frame_index, B, F, "frame_index", dev)
    bbox = boxes_from_matches_objects(refs, view_first, view_count, query, fi, matches0, (H, W))["box"]
    out = crop.crop_frames(frames_u8, bbox, K, S, fi)
    return bbox, out["image"], out["K_crop"]


def pair_table(pairs, n_frames: int, views: dict):
    """The per-pair arrays of ``boxes_from_matches_objects`` on the host: pairs, a sequence of (frame index, object id); views,
    {object id: (first view, view count)} of the table.  Returns int32 numpy arrays (frame_index, view_first, view_count), each
    [len(pairs)].  Raises ValueError for an empty pair list, a frame outside [0, n_frames) or an unknown object id."""
    pairs = [(int(f), int(o)) for f, o in pairs]
    if not 0 < len(pairs) <= crop.MAX_FRAMES:
        raise ValueError(f"1 to {crop.MAX_FRAMES} (frame, object) pairs per call, got {len(pairs)}")
    for f, o in pairs:
        if not 0 <= f < n_frames:
            raise ValueError(f"frame index {f} is outside the call's {n_frames} frames")
        if o not in views:
            raise ValueError(f"unknown object id {o}")
    fi = np.array([f for f, _ in pairs], np.int32)
    vf = np.array([views[o][0] for _, o in pairs], np.int32)
    vc = np.array([views[o][1] for _, o in pairs], np.int32)
    return fi, vf, vc


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


class ObjectDetectors:
    """``LocalFeatureObjectDetector`` for several objects in the same camera frames.  ``add_object(ref_images)`` registers an
    object's reference views (extracted once; their features stay on the device) and returns its id, as ``matcher.add_object``
    does; ``detect(frames_u8, K, pairs)`` finds object o in frame f for every (f, o) of ``pairs`` with one extractor call on the
    frames, the caller's matcher once per (pair, view), one detection launch and one crop launch."""

    def __init__(self, extractor, matcher, crop_size: int = 512, device=None):
        self.extractor, self.matcher, self.crop_size = extractor, matcher, int(crop_size)
        self.device = torch.device(device if device is not None else "cuda")
        self._objects = {}
        self._next_id = 0
        self._table = None

    def add_object(self, ref_images) -> int:
        """Register an object by its reference views (as ``LocalFeatureObjectDetector``'s ``ref_images``) and return its id."""
        self._objects[self._next_id] = LocalFeatureObjectDetector(self.extractor, self.matcher, ref_images, self.crop_size, self.device)
        self._table = None
        self._next_id += 1
        return self._next_id - 1

    def remove_object(self, object_id: int):
        """Forget a registered object."""
        if int(object_id) not in self._objects:
            raise ValueError(f"unknown object id {object_id}")
        del self._objects[int(object_id)]
        self._table = None

    def table(self):
        """(refs, views): every registered object's views in one table, in id order, and {object id: (first view, view count)}."""
        if self._table is None:
            if not self._objects:
                raise ValueError("no object registered: call add_object first")
            dets = [self._objects[i] for i in sorted(self._objects)]
            cap = max(int(d.ref["keypoints"].shape[1]) for d in dets)
            kp = torch.cat([torch.nn.functional.pad(d.ref["keypoints"], (0, 0, 0, cap - d.ref["keypoints"].shape[1])) for d in dets])
            refs = {"keypoints": kp, "counts": torch.cat([d.ref["counts"] for d in dets]), "sizes": torch.cat([d.ref["sizes"] for d in dets])}
            first = np.cumsum([0] + [len(d.views) for d in dets])
            self._table = (refs, {i: (int(first[k]), len(d.views)) for k, (i, d) in enumerate(zip(sorted(self._objects), dets))})
        return self._table

    @torch.no_grad()
    def detect(self, frames_u8: torch.Tensor, K: torch.Tensor, pairs):
        """``detect`` for B (frame, object) pairs of F frames uint8 [F, H, W] on the device: pairs is a sequence of (frame index,
        object id), K [3, 3] or [B, 3, 3] per pair.  One extractor call on the F frames (one host synchronisation, for the key-point
        counts the matcher needs at exact size), one matcher call per (pair, view), then ``detect_from_matches_objects``.  Returns
        (bbox int32 [B, 4], image_crop fp32 [B, 1, S, S], K_crop f64 [B, 3, 3]), pair b's equal to what its object's
        ``LocalFeatureObjectDetector.detect`` gives for its frame."""
        _, F, H, W = crop._frames_args(frames_u8)
        refs, views = self.table()
        pairs = list(pairs)
        fi, vf, vc = pair_table(pairs, F, views)
        dev = frames_u8.device
        det = self.extractor.forward(frames_u8[:, None].float() / 255)
        matches0 = torch.full((len(fi), int(vc.max()), int(refs["keypoints"].shape[1])), -1, dtype=torch.int64, device=dev)
        for b, (f, o) in enumerate(pairs):
            obj = self._objects[int(o)]
            kp, sc, de = det["keypoints"][int(f)], det["scores"][int(f)], det["descriptors"][int(f)]
            for v, view in enumerate(obj.views):
                m = self.matcher(obj._match_data(view, kp, sc, de, (H, W)))["matches0"][0]
                matches0[b, v, :m.shape[0]] = m
        cap_q = max(max(len(k) for k in det["keypoints"]), 1)
        query = {"keypoints": _pad(det["keypoints"], cap_q, dev),
                 "counts": torch.tensor([len(k) for k in det["keypoints"]], dtype=torch.int32).to(dev)}
        return detect_from_matches_objects(frames_u8, torch.from_numpy(fi).to(dev), K, refs, torch.from_numpy(vf).to(dev),
                                           torch.from_numpy(vc).to(dev), query, matches0, self.crop_size)

    def previous_pose_detect(self, frames_u8, K, pre_pose, bbox3d, frame_index):
        """The reference method for B objects in F frames: ``crop.previous_pose_detect(..., frame_index)``."""
        return crop.previous_pose_detect(frames_u8, K, pre_pose, bbox3d, self.crop_size, frame_index)
