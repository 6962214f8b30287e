"""The reference tracker's flow step on the GPU: an object's keyframe points followed into the next crop, and the pose from them.

With ``use_tracking`` the reference's live demo (``inference_demo.py:253-299``) runs ``BATracker.flow_track``
(``src/tracker/ba_tracker.py:295-356``): ``cv2.calcOpticalFlowPyrLK`` from the last keyframe's crop into the new one
(``kpt_flow_track``, :113-126), ``ransac_PnP`` on the tracked points and their 3D points, the mean reprojection distance and
the cm / degree distance to a reference pose, and the new keyframe when the pose passes ``<= 7 cm, <= 7 deg, < 10 px``.
``flow_track`` does that for B tracks in one call on the device, with no host synchronisation:

    kf = flow.keyframes_from_poses(res, crops_u8)                  # every 5th frame: from the matcher path's poses
    out = flow.flow_track(kf, query_u8, K_crop, pose_ref)          # the others
    kf = out["kf"]

``lk_batch`` is ``cv2.calcOpticalFlowPyrLK`` for B image pairs (``csrc/flow.cu`` behind ``opb_calc_optical_flow_pyr_lk``); its
points, status and err are OpenCV 4.13's bit for bit.  ``calc_optical_flow_pyr_lk`` is a numpy drop-in for the cv2 function.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib, pnp

TERM_COUNT, TERM_EPS = 1, 2
OPTFLOW_USE_INITIAL_FLOW, OPTFLOW_LK_GET_MIN_EIGENVALS = 4, 8
MAX_LEVEL = 4
MAX_WIN = 31
MAX_SIDE = 32767
MAX_PAIRS = 65535
# the reference's kpt_flow_track and flow_track parameters (ba_tracker.py:114-116, :322, :351)
TRACK_WIN, TRACK_LEVELS, TRACK_CRITERIA = (15, 15), 2, (TERM_EPS | TERM_COUNT, 10, 0.03)
ACCEPT_CM, ACCEPT_DEG, ACCEPT_PX = 7.0, 7.0, 10.0


def _level_dim(d: int, level: int) -> int:
    for _ in range(level):
        d = (d + 1) // 2
    return d


def _align16(v: int) -> int:
    return (v + 15) & ~15


def workspace_bytes(B: int, H: int, W: int, max_level: int) -> int:
    """Bytes of the workspace ``lk_batch`` needs for B pairs of at most H x W pixels and ``max_level``."""
    out = C.c_int64()
    _lib.check(_lib.load().opb_optical_flow_workspace_bytes(int(B), int(H), int(W), int(max_level), C.byref(out)))
    return int(out.value)


def pyramid_views(workspace: torch.Tensor, B: int, H: int, W: int, max_level: int, win_size, b: int, size=None):
    """Pair b's pyramid as ``lk_batch`` left it in ``workspace`` (the layout of include/onepose_b200.h): a list over the levels
    the pair has of (prev uint8 [h,w] or None at level 0, next uint8 [h,w] or None at level 0, prev derivatives int16 [h,w,2]).
    ``size`` is the host (h, w) of pair b when it differs from (H, W)."""
    h, w = (H, W) if size is None else (int(size[0]), int(size[1]))
    pair = workspace_bytes(B, H, W, max_level) // B
    base = workspace[b * pair:(b + 1) * pair]
    off, out = 0, []
    last = _last_level(h, w, win_size, max_level)
    for level in range(max_level + 1):
        Hl, Wl, hl, wl = _level_dim(H, level), _level_dim(W, level), _level_dim(h, level), _level_dim(w, level)
        der = base[off:off + Hl * Wl * 4].view(torch.int16).reshape(Hl, Wl, 2)[:hl, :wl]
        off = _align16(off + Hl * Wl * 4)
        ims = [None, None]
        if level > 0:
            for k in range(2):
                ims[k] = base[off:off + Hl * Wl].reshape(Hl, Wl)[:hl, :wl]
                off = _align16(off + Hl * Wl)
        if level <= last:
            out.append((ims[0], ims[1], der))
    return out


def _last_level(h, w, win, max_level):
    """The last level cv2.buildOpticalFlowPyramid builds (after level l it stops if level l + 1 has a side <= the window's)."""
    for level in range(max_level):
        w, h = (w + 1) // 2, (h + 1) // 2
        if w <= win[0] or h <= win[1]:
            return level
    return max_level


def _images(t: torch.Tensor, name: str):
    if t.dtype != torch.uint8 or t.dim() != 3:
        raise ValueError(f"{name} must be uint8 [B, H, W], got {t.dtype} {list(t.shape)}")
    B, H, W = (int(v) for v in t.shape)
    if not 0 < B <= MAX_PAIRS or not 0 < H <= MAX_SIDE or not 0 < W <= MAX_SIDE:
        raise ValueError(f"{name} must be 1..{MAX_PAIRS} images of 1..{MAX_SIDE} pixels a side, got {list(t.shape)}")
    if t.stride(2) != 1 or t.stride(1) < W or t.stride(0) < 0:
        raise ValueError(f"{name} must have unit pixel stride and rows that do not overlap, got strides {t.stride()}")
    return B, H, W


def _params(win_size, max_level, criteria, min_eig_threshold, flags=0):
    ww, wh = (int(v) for v in win_size)
    if not (3 <= ww <= MAX_WIN and 3 <= wh <= MAX_WIN and ww % 2 and wh % 2):
        raise ValueError(f"win_size must be odd, 3..{MAX_WIN}, got {tuple(win_size)}")
    if not 0 <= int(max_level) <= MAX_LEVEL:
        raise ValueError(f"max_level must be 0..{MAX_LEVEL}, got {max_level!r}")
    ty, count, eps = criteria
    ty, count, eps = int(ty), int(count), float(eps)
    if ty not in (TERM_COUNT, TERM_EPS, TERM_COUNT | TERM_EPS):
        raise ValueError(f"criteria type must be COUNT (1), EPS (2) or both, got {ty}")
    if ty & TERM_COUNT and not 1 <= count <= 100:
        raise ValueError(f"criteria count must be 1..100, got {count}")
    if ty & TERM_EPS and not eps >= 0:
        raise ValueError(f"criteria epsilon must be >= 0, got {eps}")
    if not float(min_eig_threshold) >= 0:
        raise ValueError(f"min_eig_threshold must be >= 0, got {min_eig_threshold!r}")
    if int(flags) != 0:
        raise ValueError("flags must be 0: OPTFLOW_USE_INITIAL_FLOW and OPTFLOW_LK_GET_MIN_EIGENVALS are not supported")
    return ww, wh, int(max_level), ty, count, eps, float(min_eig_threshold)


def lk_batch(prev_u8: torch.Tensor, next_u8: torch.Tensor, pts: torch.Tensor, offsets: torch.Tensor, win_size=TRACK_WIN,
             max_level: int = TRACK_LEVELS, criteria=TRACK_CRITERIA, min_eig_threshold: float = 1e-4, sizes=None,
             workspace: torch.Tensor | None = None):
    """``cv2.calcOpticalFlowPyrLK`` for B image pairs on the device: prev_u8 / next_u8 uint8 [B,H,W] CUDA (any row and image
    stride, unit pixel stride), pts fp32 [total,2], offsets int32 [B+1] (pair b owns rows offsets[b] .. offsets[b+1]-1;
    offsets[0] = 0, offsets[B] = total), ``sizes`` an optional int32 [B,2] device tensor of per-pair (h, w) <= (H, W) (the
    pair's images are the top-left corners of its slots).  win_size odd 3..31, max_level 0..4, criteria (type, count, eps) as
    cv2's.  Returns (next_pts fp32 [total,2], status uint8 [total], err fp32 [total]), cv2's bit for bit (err is 0 where
    status is 0).  ``workspace``: a contiguous uint8 CUDA tensor of at least ``workspace_bytes(B, H, W, max_level)`` bytes
    whose data starts at a multiple of 16 bytes (a misaligned one is refused with OpbError), to use (the pyramids are left in
    it, see ``pyramid_views``).  No host synchronisation."""
    dev = _lib.cuda_device(prev_u8)
    ww, wh, max_level, ty, count, eps, min_eig = _params(win_size, max_level, criteria, min_eig_threshold)
    B, H, W = _images(prev_u8, "prev_u8")
    if _images(next_u8, "next_u8") != (B, H, W) or next_u8.device != dev:
        raise ValueError(f"next_u8 must be [B, H, W] = {[B, H, W]} on {dev} like prev_u8, got {list(next_u8.shape)} on {next_u8.device}")
    if pts.dim() != 2 or pts.shape[1] != 2 or not pts.dtype.is_floating_point:
        raise ValueError(f"pts must be floating-point [total, 2], got {pts.dtype} {list(pts.shape)}")
    if offsets.dim() != 1 or offsets.shape[0] != B + 1 or offsets.dtype.is_floating_point:
        raise ValueError(f"offsets must be an integer [{B + 1}] tensor, got {offsets.dtype} {list(offsets.shape)}")
    total = int(pts.shape[0])
    pts = pts.to(device=dev, dtype=torch.float32).contiguous()
    offsets = offsets.to(device=dev, dtype=torch.int32).contiguous()
    if sizes is not None:
        if sizes.dtype != torch.int32 or tuple(sizes.shape) != (B, 2):
            raise ValueError(f"sizes must be int32 [{B}, 2], got {sizes.dtype} {list(sizes.shape)}")
        sizes = sizes.to(dev).contiguous()
    need = workspace_bytes(B, H, W, max_level)
    if workspace is None:
        workspace = torch.empty(need, dtype=torch.uint8, device=dev)
    elif workspace.dtype != torch.uint8 or workspace.device != dev or not workspace.is_contiguous() or workspace.numel() < need:
        raise ValueError(f"workspace must be a contiguous uint8 tensor of at least {need} bytes on {dev}")
    next_pts = torch.empty(total, 2, dtype=torch.float32, device=dev)
    status = torch.empty(total, dtype=torch.uint8, device=dev)
    err = torch.empty(total, dtype=torch.float32, device=dev)
    _lib.call(dev, "opb_calc_optical_flow_pyr_lk", prev_u8, prev_u8.stride(0), prev_u8.stride(1), next_u8, next_u8.stride(0), next_u8.stride(1),
              B, H, W, sizes, pts, offsets, total, ww, wh, max_level, ty, count, eps, min_eig, 0, workspace, workspace.numel(), next_pts, status, err)
    return next_pts, status, err


def calc_optical_flow_pyr_lk(prevImg, nextImg, prevPts, nextPts=None, winSize=(21, 21), maxLevel=3,
                             criteria=(TERM_COUNT | TERM_EPS, 30, 0.01), flags=0, minEigThreshold=1e-4, device=None):
    """Drop-in for ``cv2.calcOpticalFlowPyrLK`` on grey uint8 images: numpy in, numpy out, computed on the device.  Returns
    (nextPts fp32 [n,1,2], status uint8 [n,1], err fp32 [n,1]).  ``nextPts`` is only an initial guess with
    OPTFLOW_USE_INITIAL_FLOW, which is refused, as is OPTFLOW_LK_GET_MIN_EIGENVALS."""
    dev = torch.device(device if device is not None else "cuda")
    _params(winSize, maxLevel, criteria, minEigThreshold, flags)
    a, b = np.asarray(prevImg), np.asarray(nextImg)
    if a.dtype != np.uint8 or b.dtype != np.uint8 or a.ndim != 2 or a.shape != b.shape:
        raise ValueError(f"prevImg and nextImg must be uint8 [H, W] of one size, got {a.dtype} {a.shape} and {b.dtype} {b.shape}")
    p = np.asarray(prevPts, dtype=np.float32).reshape(-1, 2)
    n = p.shape[0]
    imgs = torch.from_numpy(np.stack([a, b]))[:, None].to(dev)
    pts, st, err = lk_batch(imgs[0], imgs[1], torch.from_numpy(p).to(dev), torch.tensor([0, n], dtype=torch.int32, device=dev), winSize,
                            maxLevel, criteria, minEigThreshold)
    return pts.cpu().numpy().reshape(n, 1, 2), st.cpu().numpy().reshape(n, 1), err.cpu().numpy().reshape(n, 1)


def _u8_crops(t: torch.Tensor, name: str) -> torch.Tensor:
    """uint8 [B,S,S], or the crop's fp32 [B,1,S,S] image (uint8 / 255, mapped back exactly)."""
    if t.dtype == torch.float32 and t.dim() == 4 and t.shape[1] == 1:
        t = (t[:, 0] * 255.0).round().to(torch.uint8)
    if t.dtype != torch.uint8 or t.dim() != 3:
        raise ValueError(f"{name} must be uint8 [B, S, S] or the crop's fp32 [B, 1, S, S], got {t.dtype} {list(t.shape)}")
    return t


def _check_kf(kf: dict):
    for k in ("image", "pts2d", "pts3d", "counts"):
        if k not in kf:
            raise ValueError(f"keyframe state lacks {k!r}: it needs image, pts2d, pts3d and counts")
    img, p2, p3, cnt = kf["image"], kf["pts2d"], kf["pts3d"], kf["counts"]
    if p2.dim() == 3 and p2.shape[1] == 0:
        raise ValueError("the keyframe state has no point rows (cap = 0): build it from a result with at least one pair per frame")
    dev = _lib.cuda_device(img)
    B, _, _ = _images(img, "kf['image']")
    if p2.dtype != torch.float32 or p2.dim() != 3 or p2.shape[0] != B or p2.shape[2] != 2:
        raise ValueError(f"kf['pts2d'] must be fp32 [{B}, cap, 2], got {p2.dtype} {list(p2.shape)}")
    cap = int(p2.shape[1])
    if p3.dtype != torch.float32 or tuple(p3.shape) != (B, cap, 3):
        raise ValueError(f"kf['pts3d'] must be fp32 [{B}, {cap}, 3], got {p3.dtype} {list(p3.shape)}")
    if cnt.dtype != torch.int32 or tuple(cnt.shape) != (B,):
        raise ValueError(f"kf['counts'] must be int32 [{B}], got {cnt.dtype} {list(cnt.shape)}")
    if any(t.device != dev for t in (p2, p3, cnt)):
        raise ValueError(f"the keyframe state must live on one device ({dev})")
    return dev, B, cap


def flow_track(kf: dict, query_crop: torch.Tensor, K_crop: torch.Tensor, pose_ref: torch.Tensor) -> dict:
    """``BATracker.flow_track`` (ba_tracker.py:295-356) for B tracks on the device, with no host synchronisation.

    kf          keyframe state of device tensors: image uint8 [B,S,S] (the keyframe's crop), pts2d fp32 [B,cap,2] and pts3d
                fp32 [B,cap,3] (its inlier 2D-3D pairs; rows past counts are ignored), counts int32 [B]
    query_crop  the new crop, uint8 [B,S,S] or ``crop.crop_frames``' fp32 [B,1,S,S]
    K_crop      [B,3,3] or [3,3], the new crop's intrinsics
    pose_ref    [B,3,4] or [B,4,4], the pose the flow pose is scored against.  In the reference's demo it is the frame's own
                matcher pose (``'pose_gt': pose_pred_homo``, inference_demo.py:258).

    Steps, as the reference: ``cv2.calcOpticalFlowPyrLK`` (window 15, 2 levels, (EPS|COUNT, 10, 0.03)) from the keyframe crop
    into the query crop; the status-1 points in index order (``np.where``) with their 3D points; ``ransac_PnP`` on them --
    cv2.solvePnPRansac(EPNP, 10000 iterations, 5 px, confidence 0.99, no scale) as ``ransac_pnp_batch(method="epnp",
    confidence=0.99)`` runs it, the identity pose below 4 points; kpt_dist, the fp64 mean of |project(pts3d, K_crop, pose) -
    tracked| (NaN with no tracked point); trans_dist / rot_dist to pose_ref (``cm_degree_5_metric`` = ``pnp.pose_errors``);
    accept = trans <= 7 & rot <= 7 & kpt_dist < 10.  (The reference's ``valid_ids is None`` branch, :345-349, cannot be taken
    with cv2 4.13, which always returns a status.)

    Returns a dict of device tensors: pose_init_homo f64 [B,4,4], kpt_dist / trans_dist / rot_dist f64 [B], n_tracked /
    n_inliers int32 [B], accept bool [B], and kf, the updated state: an accepted track's row becomes (query crop, tracked
    2D points, their 3D points), the others are unchanged (``last_kf_info`` of :351-354)."""
    dev, B, cap = _check_kf(kf)
    query = _u8_crops(query_crop, "query_crop").to(dev)
    if tuple(query.shape) != tuple(kf["image"].shape):
        raise ValueError(f"query_crop must match the keyframe crops {list(kf['image'].shape)}, got {list(query.shape)}")
    K = K_crop.to(device=dev, dtype=torch.float64)
    K = K.expand(B, 3, 3) if K.dim() == 2 else K
    if tuple(K.shape) != (B, 3, 3):
        raise ValueError(f"K_crop must be [3, 3] or [{B}, 3, 3], got {list(K_crop.shape)}")
    if pose_ref.dim() != 3 or pose_ref.shape[0] != B or tuple(pose_ref.shape[1:]) not in ((3, 4), (4, 4)):
        raise ValueError(f"pose_ref must be [{B}, 3, 4] or [{B}, 4, 4], got {list(pose_ref.shape)}")
    K = K.contiguous()
    offsets_lk = torch.arange(0, (B + 1) * cap, cap, dtype=torch.int32, device=dev)
    tracked, status, _ = lk_batch(kf["image"], query, kf["pts2d"].reshape(B * cap, 2), offsets_lk)
    n = max(B * cap, 1)
    p2 = torch.empty(n, 2, dtype=torch.float64, device=dev)
    p3 = torch.empty(n, 3, dtype=torch.float64, device=dev)
    pad2 = torch.empty(B, cap, 2, dtype=torch.float32, device=dev)
    pad3 = torch.empty(B, cap, 3, dtype=torch.float32, device=dev)
    offsets = torch.empty(B + 1, dtype=torch.int32, device=dev)
    n_tracked = torch.empty(B, dtype=torch.int32, device=dev)
    _lib.call(dev, "opb_flow_compact", status, tracked, kf["pts3d"].contiguous(), kf["counts"].contiguous(), B, cap, p2, p3, offsets, n_tracked,
              pad2, pad3)
    pose, _, n_inliers = pnp.ransac_pnp_batch(K, p2, p3, offsets, reproj_error=5.0, hypotheses=pnp.EPNP_HYPOTHESES, method="epnp",
                                              confidence=0.99)
    kpt_dist = torch.empty(B, dtype=torch.float64, device=dev)
    _lib.call(dev, "opb_flow_reprojection", K, pose.contiguous(), p2, p3, offsets, B, kpt_dist)
    pose_homo = torch.zeros(B, 4, 4, dtype=torch.float64, device=dev)
    pose_homo[:, :3] = pose
    pose_homo[:, 3, 3] = 1.0
    rot, trans = pnp.pose_errors(pose_homo, pose_ref.to(dev))
    accept = (trans <= ACCEPT_CM) & (rot <= ACCEPT_DEG) & (kpt_dist < ACCEPT_PX)
    a3 = accept[:, None, None]
    new_kf = {"image": torch.where(a3, query, kf["image"]), "pts2d": torch.where(a3, pad2, kf["pts2d"]),
              "pts3d": torch.where(a3, pad3, kf["pts3d"]), "counts": torch.where(accept, n_tracked, kf["counts"])}
    return {"pose_init_homo": pose_homo, "kpt_dist": kpt_dist, "trans_dist": trans, "rot_dist": rot, "n_tracked": n_tracked,
            "n_inliers": n_inliers, "accept": accept, "kf": new_kf}


def keyframes_from_poses(res: dict, crops_u8: torch.Tensor) -> dict:
    """The keyframe state ``flow_track`` takes, from a ``pnp.poses_from_matches`` / ``poses_from_matches_objects`` result and
    the B crops it was solved on (uint8 [B,S,S] or the crop's fp32 [B,1,S,S]): per frame, the inlier pairs in pair order --
    ``mkpts2d[inliers.flatten()]``, ``mkpts3d[...]`` of inference_demo.py:266-267 -- as fp32 pts2d [B,cap,2] and pts3d
    [B,cap,3] (cap = the result's pairs per frame, N; rows past counts are zero), and counts int32 [B] (= n_inliers).  The pairs
    are the result's own gathered ones (``res['pts2d']`` / ``res['pts3d']``, fp32 key points widened to f64, so the narrowing
    is exact).  No host synchronisation."""
    crops = _u8_crops(crops_u8, "crops_u8")
    dev = _lib.cuda_device(crops)
    B = int(crops.shape[0])
    off = res["offsets"].to(dev)
    mask = res["inlier_mask"].to(dev)
    if off.shape[0] != B + 1 or mask.numel() % B:
        raise ValueError(f"the result is for {off.shape[0] - 1} frames and {mask.numel()} pairs, the crops for {B} frames")
    cap = mask.numel() // B
    rows = torch.arange(B * cap, device=dev, dtype=torch.int64)
    frame = torch.searchsorted(off[1:].to(torch.int64), rows, right=True)       # B for rows past offsets[B]
    keep = mask & (frame < B)
    csum = torch.cumsum(keep.to(torch.int64), 0)
    base = torch.cat([torch.zeros(1, dtype=torch.int64, device=dev), csum])[off.to(torch.int64)]   # inliers before frame b's rows
    rank = csum - 1 - base[frame.clamp(max=B - 1)]
    dest = torch.where(keep, frame * cap + rank, torch.full_like(rows, B * cap))  # the dropped rows go to a spare row
    p2 = torch.zeros(B * cap + 1, 2, dtype=torch.float32, device=dev)
    p3 = torch.zeros(B * cap + 1, 3, dtype=torch.float32, device=dev)
    p2.index_copy_(0, dest, res["pts2d"][:B * cap].to(torch.float32))
    p3.index_copy_(0, dest, res["pts3d"][:B * cap].to(torch.float32))
    counts = (base[1:] - base[:-1]).to(torch.int32)
    return {"image": crops.contiguous(), "pts2d": p2[:-1].reshape(B, cap, 2), "pts3d": p3[:-1].reshape(B, cap, 3), "counts": counts}
