"""Object pose from the matcher's 2D-3D correspondences -- GPU RANSAC-PnP.

``ransac_PnP`` mirrors the reference's function of the same name (``src/utils/eval_utils.py:18-42``: same arguments, same
return triple ``(pose [3,4], pose_homo [4,4], inliers)`` as numpy, identity pose and ``[]`` when no pose can be estimated);
``ransac_pnp_batch`` solves many frames in one launch and keeps everything on the device.  The arithmetic is
``csrc/pnp_ransac.cu`` (P3P minimal samples, inlier counting over all correspondences, Gauss-Newton refinement on the
inliers) behind ``opb_ransac_pnp``.  The reference delegates to ``cv2.solvePnPRansac`` (EPnP, 10000 iterations, 5 px);
parity is on the pose (the reference's cm-degree metric), not on bits -- OpenCV draws its own random samples.

``gather_matches`` turns the matcher's ``matches0`` into those correspondence lists on the device (``opb_gather_matches``; the
reference's ``valid = matches > -1; mkpts2d = kpts2d[valid]; mkpts3d = kpts3d[matches[valid]]``, inference.py:147-152) and
``poses_from_matches`` chains it with the solver.  ``pose_errors`` / ``cm_degree`` are the reference's pose metric
(``query_pose_error`` and ``aggregate_metrics``, eval_utils.py:45-63, :105-120; ``cmd_evaluator.Evaluator``).
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib

DEFAULT_HYPOTHESES = 4096      # minimal samples per frame: P(no all-inlier sample) < 1e-9 down to 15 % inliers


def ransac_pnp_batch(K: torch.Tensor, pts2d: torch.Tensor, pts3d: torch.Tensor, offsets: torch.Tensor, reproj_error: float = 5.0,
                     hypotheses: int = DEFAULT_HYPOTHESES, seed: int = 0):
    """K [B,3,3], pts2d [total,2], pts3d [total,3], offsets [B+1] (frame b owns [offsets[b], offsets[b+1])) -- CUDA tensors
    (any float dtype; computed in fp64).  Returns (pose [B,3,4] f64, inlier_mask [total] bool, n_inliers [B] int32), on the device."""
    lib = _lib.load()
    dev = pts2d.device
    if dev.type != "cuda":
        raise RuntimeError("onepose_b200 has no CPU path: tensors must be on a CUDA device")
    B = int(offsets.numel()) - 1
    K = K.to(device=dev, dtype=torch.float64).reshape(B, 9).contiguous()
    p2 = pts2d.to(torch.float64).contiguous()
    p3 = pts3d.to(torch.float64).contiguous()
    off = offsets.to(device=dev, dtype=torch.int32).contiguous()
    total = int(p2.shape[0])
    ws = torch.empty(B * hypotheses * 13, dtype=torch.float64, device=dev)
    pose = torch.empty(B, 12, dtype=torch.float64, device=dev)
    mask = torch.zeros(max(total, 1), dtype=torch.int32, device=dev)
    cnt = torch.empty(B, dtype=torch.int32, device=dev)
    st = torch.cuda.current_stream(dev).cuda_stream
    with torch.cuda.device(dev):
        _lib.check(lib.opb_ransac_pnp(K.data_ptr(), p2.data_ptr(), p3.data_ptr(), off.data_ptr(), B, int(hypotheses), float(reproj_error),
                                      int(seed) & 0xFFFFFFFFFFFFFFFF, ws.data_ptr(), pose.data_ptr(), mask.data_ptr(), cnt.data_ptr(), st))
    return pose.reshape(B, 3, 4), mask[:total].bool(), cnt


def gather_matches(matches0: torch.Tensor, keypoints2d: torch.Tensor, keypoints3d: torch.Tensor,
                   matching_scores0: torch.Tensor | None = None):
    """Matched 2D-3D pairs of B frames, frame-major and in ascending query index within a frame (numpy boolean-mask order).
    matches0 int64 [B,N] (an entry outside [0, M) is not a match), keypoints2d fp32 [B,N,2] (rows of unmatched entries are never
    read), keypoints3d fp32 [M,3], matching_scores0 fp32 [B,N] or None -- CUDA tensors.  Returns a dict of device tensors with
    capacity B*N: pts2d f64 [B*N,2], pts3d f64 [B*N,3], mconf fp32 [B*N] (None without scores), query_index int32 [B*N] and
    offsets int32 [B+1]; frame b owns rows [offsets[b], offsets[b+1]), rows from offsets[B] on are unspecified.  The values are
    exactly the reference's ``kpts2d[valid]``, ``kpts3d[matches[valid]]`` after ``astype(np.float64)``.  No host synchronisation."""
    lib = _lib.load()
    dev = matches0.device
    if dev.type != "cuda":
        raise RuntimeError("onepose_b200 has no CPU path: tensors must be on a CUDA device")
    if matches0.dim() != 2:
        raise ValueError("matches0 must be [B, N]")
    B, N = matches0.shape
    m0 = matches0.to(torch.int64).contiguous()
    kp2 = keypoints2d.to(device=dev, dtype=torch.float32).contiguous()
    kp3 = keypoints3d.to(device=dev, dtype=torch.float32).contiguous()
    if tuple(kp2.shape) != (B, N, 2):
        raise ValueError(f"keypoints2d must be [B, N, 2] = {(B, N, 2)}, got {tuple(kp2.shape)}")
    if kp3.dim() != 2 or kp3.shape[1] != 3:
        raise ValueError(f"keypoints3d must be [M, 3], got {tuple(kp3.shape)}")
    sc = None
    if matching_scores0 is not None:
        sc = matching_scores0.to(device=dev, dtype=torch.float32).contiguous()
        if tuple(sc.shape) != (B, N):
            raise ValueError("matching_scores0 must be [B, N] like matches0")
    out = {"pts2d": torch.empty(B * N, 2, dtype=torch.float64, device=dev), "pts3d": torch.empty(B * N, 3, dtype=torch.float64, device=dev),
           "mconf": torch.empty(B * N, dtype=torch.float32, device=dev) if sc is not None else None,
           "query_index": torch.empty(B * N, dtype=torch.int32, device=dev), "offsets": torch.empty(B + 1, dtype=torch.int32, device=dev)}
    st = torch.cuda.current_stream(dev).cuda_stream
    with torch.cuda.device(dev):
        _lib.check(lib.opb_gather_matches(m0.data_ptr(), sc.data_ptr() if sc is not None else None, kp2.data_ptr(), kp3.data_ptr(),
                                          B, N, int(kp3.shape[0]), out["pts2d"].data_ptr(), out["pts3d"].data_ptr(),
                                          out["mconf"].data_ptr() if sc is not None else None, out["query_index"].data_ptr(),
                                          out["offsets"].data_ptr(), st))
    return out


def poses_from_matches(K: torch.Tensor, keypoints2d: torch.Tensor, keypoints3d: torch.Tensor, matches0: torch.Tensor,
                       matching_scores0: torch.Tensor | None = None, reproj_error: float = 5.0, scale: float = 1000.0,
                       hypotheses: int = DEFAULT_HYPOTHESES, seed: int = 0):
    """Object pose of B frames from the matcher's output: ``gather_matches`` then ``ransac_pnp_batch``, all on the device and with
    no host synchronisation (inference.py:147-155 for a batch).  K [3,3] (shared) or [B,3,3]; the other arguments as in
    ``gather_matches``.  ``scale`` multiplies the 3D points before the solve and divides the translation after it, as
    ``ransac_PnP(..., scale=1000)`` does in the reference.  A frame with fewer than 4 pairs, or no model, gets the identity pose
    and 0 inliers.  Returns a dict: pose [B,3,4] and pose_homo [B,4,4] f64, n_inliers int32 [B], inlier_mask bool [B*N],
    query_index, mconf and offsets (rows indexed as in ``gather_matches``)."""
    g = gather_matches(matches0, keypoints2d, keypoints3d, matching_scores0)
    B = int(matches0.shape[0])
    dev = matches0.device
    K = K.to(device=dev, dtype=torch.float64)
    if K.dim() == 2:
        K = K.expand(B, 3, 3)
    pose, mask, cnt = ransac_pnp_batch(K, g["pts2d"], g["pts3d"] * scale, g["offsets"], reproj_error=reproj_error,
                                       hypotheses=hypotheses, seed=seed)
    pose[:, :, 3] /= scale
    pose_homo = torch.zeros(B, 4, 4, dtype=torch.float64, device=dev)
    pose_homo[:, :3] = pose
    pose_homo[:, 3, 3] = 1.0
    return {"pose": pose, "pose_homo": pose_homo, "n_inliers": cnt, "inlier_mask": mask, "query_index": g["query_index"],
            "mconf": g["mconf"], "offsets": g["offsets"]}


def pose_errors(pose_pred: torch.Tensor, pose_gt: torch.Tensor):
    """(rot_err_deg [B], trans_err_cm [B]) of poses [B,3,4] or [B,4,4], in f64 on the inputs' device: the reference's
    ``query_pose_error`` (eval_utils.py:45-63) per frame.  As there, the trace is clamped above at 3 only (a trace below -1
    gives NaN, a NaN trace becomes 3) and the translation error is |dt| * 100."""
    pp = pose_pred.to(torch.float64)[..., :3, :]
    pg = pose_gt.to(device=pp.device, dtype=torch.float64)[..., :3, :]
    dt = pp[..., 3] - pg[..., 3]
    trans = torch.sqrt(dt[..., 0] * dt[..., 0] + dt[..., 1] * dt[..., 1] + dt[..., 2] * dt[..., 2]) * 100
    e = pp[..., :3] * pg[..., :3]
    d = e[..., 0] + e[..., 1] + e[..., 2]                       # diagonal of R_pred . R_gt^T, summed in index order
    trace = d[..., 0] + d[..., 1] + d[..., 2]
    trace = torch.where(trace <= 3, trace, torch.full_like(trace, 3.0))
    rot = torch.rad2deg(torch.acos((trace - 1.0) / 2.0))
    return rot, trans


def cm_degree(rot_err: torch.Tensor, trans_err: torch.Tensor, thresholds=(1, 3, 5)):
    """Fraction of frames with rot_err < thr degrees and trans_err < thr cm, {'1cm@1degree': ...} as the reference's
    ``aggregate_metrics`` (eval_utils.py:105-120); NaN fails.  The values equal ``cmd_evaluator.Evaluator.summarize``'s cmd1/3/5."""
    rot = torch.as_tensor(rot_err, dtype=torch.float64)
    trans = torch.as_tensor(trans_err, dtype=torch.float64, device=rot.device)
    return {f"{t}cm@{t}degree": float(((rot < t) & (trans < t)).double().mean()) for t in thresholds}


def ransac_PnP(K, pts_2d, pts_3d, scale=1, device=None):
    """Drop-in for the reference ``ransac_PnP`` (eval_utils.py:18-42): numpy in, numpy out.
    ``scale`` only conditions OpenCV's EPnP in the reference (points x scale, translation / scale): applied and undone here
    too so that the argument keeps its meaning.  Returns (pose [3,4], pose_homo [4,4], inliers [k,1] int32 or [])."""
    dev = torch.device(device if device is not None else "cuda")
    pts_2d = np.ascontiguousarray(np.asarray(pts_2d, dtype=np.float64)).reshape(-1, 2)
    pts_3d = np.ascontiguousarray(np.asarray(pts_3d, dtype=np.float64)).reshape(-1, 3) * scale
    n = pts_2d.shape[0]
    if n < 4:                                                   # cv2.error branch of the reference (:40-42)
        return np.eye(4)[:3], np.eye(4), []
    pose, mask, cnt = ransac_pnp_batch(torch.from_numpy(np.asarray(K, dtype=np.float64))[None].to(dev), torch.from_numpy(pts_2d).to(dev),
                                       torch.from_numpy(pts_3d).to(dev), torch.tensor([0, n], dtype=torch.int32, device=dev))
    if int(cnt[0]) == 0:
        return np.eye(4)[:3], np.eye(4), []
    pose = pose[0].cpu().numpy()
    pose[:, 3] /= scale
    pose_homo = np.concatenate([pose, np.array([[0, 0, 0, 1.0]])], axis=0)
    inliers = torch.nonzero(mask).to(torch.int32).cpu().numpy().reshape(-1, 1)
    return pose, pose_homo, inliers
