"""Object pose from the matcher's 2D-3D correspondences -- GPU RANSAC-PnP.

``ransac_PnP`` mirrors the reference's function of the same name (``src/utils/eval_utils.py:18-42``: same arguments, same
return triple ``(pose [3,4], pose_homo [4,4], inliers)`` as numpy, identity pose and ``[]`` when no pose can be estimated);
``ransac_pnp_batch`` solves many frames in one launch and keeps everything on the device.  The arithmetic is
``csrc/pnp_ransac.cu`` (P3P minimal samples, inlier counting over all correspondences, Gauss-Newton refinement on the
inliers) behind ``opb_ransac_pnp``; ``method="epnp"`` selects the reference's own estimator instead (``opb_ransac_epnp``:
five-point EPnP samples, OpenCV's inlier rule, an EPnP refit on the inliers), and ``epnp_batch`` is ``cv2.solvePnP(EPNP)``.  The reference delegates to ``cv2.solvePnPRansac`` (EPnP, 10000 iterations, 5 px);
parity is on the pose (the reference's cm-degree metric), not on bits -- OpenCV draws its own random samples.  With
``confidence=c`` as well (``opb_ransac_epnp_cv``) the loop is OpenCV's own: its sample sequence, its fp32 inlier count and its
stopping rule, so a frame stops after the samples OpenCV would draw (about 145 at 50 % inliers and c = 0.99).

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
EPNP_HYPOTHESES = 10000        # the reference's iterationsCount: five-point samples need more draws than three-point ones
METHODS = ("p3p", "epnp")
# the workspace layout of include/onepose_b200.h: per frame and hypothesis one record {count, R (9), t (3)}, and for the
# confidence mode one loop state per frame after all records
RECORD_DOUBLES = 13
CV_STATE_DOUBLES = 16


def _hypotheses(method, hypotheses, confidence=None):
    if method not in METHODS:
        raise ValueError(f"method must be one of {METHODS}, got {method!r}")
    if confidence is not None:
        if method != "epnp":
            raise ValueError("confidence is OpenCV's EPnP-RANSAC stopping rule: it needs method=\"epnp\"")
        if not 0.0 <= float(confidence) <= 1.0:
            raise ValueError(f"confidence must be in [0, 1], got {confidence!r}")
    if hypotheses is None:
        return DEFAULT_HYPOTHESES if method == "p3p" else EPNP_HYPOTHESES
    return int(hypotheses)


def _frames(K, pts2d, pts3d, offsets):
    dev = _lib.cuda_device(pts2d)
    B = int(offsets.numel()) - 1
    K = K.to(device=dev, dtype=torch.float64).reshape(B, 9).contiguous()
    p2 = pts2d.to(torch.float64).contiguous()
    p3 = pts3d.to(torch.float64).contiguous()
    off = offsets.to(device=dev, dtype=torch.int32).contiguous()
    return dev, B, K, p2, p3, off


def epnp_batch(K: torch.Tensor, pts2d: torch.Tensor, pts3d: torch.Tensor, offsets: torch.Tensor):
    """EPnP on every correspondence of each frame -- ``cv2.solvePnP(..., flags=SOLVEPNP_EPNP)`` for B frames in one launch.
    Arguments as in ``ransac_pnp_batch``.  Returns (pose [B,3,4] f64, status [B] int32) on the device: status 1 for a pose,
    0 (and the identity pose) for a frame with fewer than 4 pairs or a degenerate point set.  No host synchronisation."""
    dev, B, K, p2, p3, off = _frames(K, pts2d, pts3d, offsets)
    pose = torch.empty(B, 12, dtype=torch.float64, device=dev)
    status = torch.empty(B, dtype=torch.int32, device=dev)
    _lib.call(dev, "opb_epnp", K, p2, p3, off, B, pose, status)
    return pose.reshape(B, 3, 4), status


def ransac_pnp_batch(K: torch.Tensor, pts2d: torch.Tensor, pts3d: torch.Tensor, offsets: torch.Tensor, reproj_error: float = 5.0,
                     hypotheses: int | None = None, seed: int = 0, method: str = "p3p", confidence: float | None = None,
                     iterations_out: torch.Tensor | None = None):
    """K [B,3,3], pts2d [total,2], pts3d [total,3], offsets [B+1] (frame b owns [offsets[b], offsets[b+1])) -- CUDA tensors
    (any float dtype; computed in fp64).  Returns (pose [B,3,4] f64, inlier_mask [total] bool, n_inliers [B] int32), on the device.
    ``method`` picks the estimator: "p3p" (default: P3P samples, Gauss-Newton on the inliers; ``hypotheses=None`` = 4096) or
    "epnp" (the reference's cv2.solvePnPRansac(EPNP): five-point EPnP samples on fp32-rounded inputs, OpenCV's inlier rule, an
    EPnP refit on the best sample's inliers; ``hypotheses=None`` = 10000).  The two return different poses.
    ``confidence`` (``method="epnp"`` only; a ValueError otherwise) runs OpenCV's loop, cv2.solvePnPRansac(...,
    iterationsCount=hypotheses, confidence=confidence, flags=SOLVEPNP_EPNP): OpenCV's sample sequence (``seed`` plays no part),
    its fp32 inlier count, and a frame stops when OpenCV's would.  ``iterations_out``, an int32 [B] device tensor, then receives
    the number of samples each frame's loop ran (0 for frames of fewer than 6 pairs)."""
    hypotheses = _hypotheses(method, hypotheses, confidence)
    dev, B, K, p2, p3, off = _frames(K, pts2d, pts3d, offsets)
    total = int(p2.shape[0])
    pose = torch.empty(B, 12, dtype=torch.float64, device=dev)
    mask = torch.zeros(max(total, 1), dtype=torch.int32, device=dev)
    cnt = torch.empty(B, dtype=torch.int32, device=dev)
    if confidence is not None:
        it = iterations_out
        if it is None:
            it = torch.empty(B, dtype=torch.int32, device=dev)
        elif it.device != dev or it.dtype != torch.int32 or tuple(it.shape) != (B,) or not it.is_contiguous():
            raise ValueError(f"iterations_out must be a contiguous int32 [{B}] tensor on {dev}")
        ws = torch.empty(B * (hypotheses * RECORD_DOUBLES + CV_STATE_DOUBLES), dtype=torch.float64, device=dev)
        _lib.call(dev, "opb_ransac_epnp_cv", K, p2, p3, off, B, int(hypotheses), float(reproj_error), float(confidence), ws, pose, mask, cnt, it)
        return pose.reshape(B, 3, 4), mask[:total].bool(), cnt
    if iterations_out is not None:
        raise ValueError("iterations_out is filled by the confidence mode only")
    ws = torch.empty(B * hypotheses * RECORD_DOUBLES, dtype=torch.float64, device=dev)
    _lib.call(dev, "opb_ransac_pnp" if method == "p3p" else "opb_ransac_epnp", K, p2, p3, off, B, int(hypotheses), float(reproj_error),
              int(seed) & 0xFFFFFFFFFFFFFFFF, ws, pose, mask, cnt)
    return pose.reshape(B, 3, 4), mask[:total].bool(), cnt


def gather_matches(matches0: torch.Tensor, keypoints2d: torch.Tensor, keypoints3d: torch.Tensor,
                   matching_scores0: torch.Tensor | None = None):
    """Matched 2D-3D pairs of B frames, frame-major and in ascending query index within a frame (numpy boolean-mask order).
    matches0 int64 [B,N] (an entry outside [0, M) is not a match), keypoints2d fp32 [B,N,2] (rows of unmatched entries are never
    read), keypoints3d fp32 [M,3], matching_scores0 fp32 [B,N] or None -- CUDA tensors.  Returns a dict of device tensors with
    capacity B*N: pts2d f64 [B*N,2], pts3d f64 [B*N,3], mconf fp32 [B*N] (None without scores), query_index int32 [B*N] and
    offsets int32 [B+1]; frame b owns rows [offsets[b], offsets[b+1]), rows from offsets[B] on are unspecified.  The values are
    exactly the reference's ``kpts2d[valid]``, ``kpts3d[matches[valid]]`` after ``astype(np.float64)``.  No host synchronisation."""
    dev, B, N = _match_batch(matches0)
    kp3 = keypoints3d.to(device=dev, dtype=torch.float32).contiguous()
    if kp3.dim() != 2 or kp3.shape[1] != 3:
        raise ValueError(f"keypoints3d must be [M, 3], got {tuple(kp3.shape)}")
    return _gather(matches0, keypoints2d, matching_scores0, "opb_gather_matches", kp3, B, N, int(kp3.shape[0]))


def _match_batch(matches0):
    dev = _lib.cuda_device(matches0)
    if matches0.dim() != 2:
        raise ValueError("matches0 must be [B, N]")
    B, N = matches0.shape
    return dev, B, N


def _gather(matches0, keypoints2d, matching_scores0, name, *args):
    """What both gathers share: the keypoints2d and score checks, the outputs, and the call of entry point ``name``, whose
    arguments between keypoints2d and the outputs are ``args``."""
    dev = matches0.device
    B, N = matches0.shape
    m0 = matches0.to(torch.int64).contiguous()
    kp2 = keypoints2d.to(device=dev, dtype=torch.float32).contiguous()
    if tuple(kp2.shape) != (B, N, 2):
        raise ValueError(f"keypoints2d must be [B, N, 2] = {(B, N, 2)}, got {tuple(kp2.shape)}")
    sc = None
    if matching_scores0 is not None:
        sc = matching_scores0.to(device=dev, dtype=torch.float32).contiguous()
        if tuple(sc.shape) != (B, N):
            raise ValueError("matching_scores0 must be [B, N] like matches0")
    out = {"pts2d": torch.empty(B * N, 2, dtype=torch.float64, device=dev), "pts3d": torch.empty(B * N, 3, dtype=torch.float64, device=dev),
           "mconf": torch.empty(B * N, dtype=torch.float32, device=dev) if sc is not None else None,
           "query_index": torch.empty(B * N, dtype=torch.int32, device=dev), "offsets": torch.empty(B + 1, dtype=torch.int32, device=dev)}
    _lib.call(dev, name, m0, sc, kp2, *args, out["pts2d"], out["pts3d"], out["mconf"], out["query_index"], out["offsets"])
    return out


def gather_matches_objects(matches0: torch.Tensor, keypoints2d: torch.Tensor, keypoints3d, object_ids,
                           matching_scores0: torch.Tensor | None = None):
    """``gather_matches`` for frames of different objects (``GATsSuperGlue.match_objects``' output): frame b's matches index the
    3D key points ``keypoints3d[object_ids[b]]`` (fp32 [M_b, 3] CUDA tensors; ``keypoints3d`` maps object id -> tensor, a dict
    or a sequence indexed by id), an entry outside [0, M_b) is not a match.  ``object_ids`` is a host sequence (or CPU tensor).
    Same outputs as ``gather_matches``.  The per-frame tables go to the device from pinned memory: no host synchronisation."""
    dev, B, N = _match_batch(matches0)
    ids = [int(i) for i in (object_ids.tolist() if isinstance(object_ids, torch.Tensor) else object_ids)]
    if len(ids) != B:
        raise ValueError(f"object_ids has {len(ids)} entries for {B} frames")
    first, parts, row = {}, [], 0                       # each object's key points once, in order of first appearance
    for i in ids:
        if i not in first:
            k = keypoints3d[i].to(device=dev, dtype=torch.float32)
            if k.dim() != 2 or k.shape[1] != 3 or k.shape[0] == 0:
                raise ValueError(f"keypoints3d[{i}] must be [M, 3] with M > 0, got {tuple(k.shape)}")
            first[i] = (row, int(k.shape[0]))
            parts.append(k)
            row += int(k.shape[0])
    kp3 = torch.cat(parts, 0).contiguous()
    tab = torch.tensor([first[i][0] for i in ids] + [first[i][1] for i in ids], dtype=torch.int32).pin_memory()
    tab = tab.to(dev, non_blocking=True)
    return _gather(matches0, keypoints2d, matching_scores0, "opb_gather_matches_objects", kp3, tab, tab[B:], B, N)


def _solve(K, g, B, dev, reproj_error, scale, hypotheses, seed, method, confidence):
    K = K.to(device=dev, dtype=torch.float64)
    if K.dim() == 2:
        K = K.expand(B, 3, 3)
    its = torch.empty(B, dtype=torch.int32, device=dev) if confidence is not None else None
    pose, mask, cnt = ransac_pnp_batch(K, g["pts2d"], g["pts3d"] * scale, g["offsets"], reproj_error=reproj_error,
                                       hypotheses=hypotheses, seed=seed, method=method, confidence=confidence, iterations_out=its)
    pose[:, :, 3] /= scale
    pose_homo = torch.zeros(B, 4, 4, dtype=torch.float64, device=dev)
    pose_homo[:, :3] = pose
    pose_homo[:, 3, 3] = 1.0
    out = {"pose": pose, "pose_homo": pose_homo, "n_inliers": cnt, "inlier_mask": mask, "query_index": g["query_index"],
           "mconf": g["mconf"], "offsets": g["offsets"], "pts2d": g["pts2d"], "pts3d": g["pts3d"]}
    if its is not None:
        out["iterations"] = its
    return out


def poses_from_matches_objects(K: torch.Tensor, keypoints2d: torch.Tensor, keypoints3d, object_ids, matches0: torch.Tensor,
                               matching_scores0: torch.Tensor | None = None, reproj_error: float = 5.0, scale: float = 1000.0,
                               hypotheses: int | None = None, seed: int = 0, method: str = "p3p", confidence: float | None = None):
    """``poses_from_matches`` for frames of different objects: ``gather_matches_objects`` then ``ransac_pnp_batch``; same
    arguments and outputs, with ``keypoints3d`` / ``object_ids`` as in ``gather_matches_objects``.  No host synchronisation."""
    hypotheses = _hypotheses(method, hypotheses, confidence)
    g = gather_matches_objects(matches0, keypoints2d, keypoints3d, object_ids, matching_scores0)
    return _solve(K, g, int(matches0.shape[0]), matches0.device, reproj_error, scale, hypotheses, seed, method, confidence)


def poses_from_matches(K: torch.Tensor, keypoints2d: torch.Tensor, keypoints3d: torch.Tensor, matches0: torch.Tensor,
                       matching_scores0: torch.Tensor | None = None, reproj_error: float = 5.0, scale: float = 1000.0,
                       hypotheses: int | None = None, seed: int = 0, method: str = "p3p", confidence: float | None = None):
    """Object pose of B frames from the matcher's output: ``gather_matches`` then ``ransac_pnp_batch``, all on the device and with
    no host synchronisation (inference.py:147-155 for a batch).  K [3,3] (shared) or [B,3,3]; the other arguments as in
    ``gather_matches``.  ``scale`` multiplies the 3D points before the solve and divides the translation after it, as
    ``ransac_PnP(..., scale=1000)`` does in the reference.  A frame with fewer than 4 pairs, or no model, gets the identity pose
    and 0 inliers.  ``method`` / ``hypotheses`` / ``confidence`` as in ``ransac_pnp_batch``.  Returns a dict: pose [B,3,4] and
    pose_homo [B,4,4] f64, n_inliers int32 [B], inlier_mask bool [B*N], query_index, mconf, offsets and the gathered pairs
    pts2d / pts3d (rows indexed as in ``gather_matches``; pts3d unscaled), and with ``confidence`` also iterations int32 [B] (the samples each frame's loop ran)."""
    hypotheses = _hypotheses(method, hypotheses, confidence)
    g = gather_matches(matches0, keypoints2d, keypoints3d, matching_scores0)
    return _solve(K, g, int(matches0.shape[0]), matches0.device, reproj_error, scale, hypotheses, seed, method, confidence)


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


def ransac_PnP(K, pts_2d, pts_3d, scale=1, device=None, method="p3p", confidence=None):
    """Drop-in for the reference ``ransac_PnP`` (eval_utils.py:18-42): numpy in, numpy out.
    ``scale`` only conditions OpenCV's EPnP in the reference (points x scale, translation / scale): applied and undone here
    too so that the argument keeps its meaning.  ``method="epnp"`` runs the reference's estimator (EPnP-RANSAC, 10000
    samples), the default "p3p" the project's own; ``method="epnp", confidence=0.99`` is the reference's call itself, OpenCV's
    loop with its default confidence.  Returns (pose [3,4], pose_homo [4,4], inliers [k,1] int32 or [])."""
    _hypotheses(method, None, confidence)
    dev = torch.device(device if device is not None else "cuda")
    pts_2d = np.ascontiguousarray(np.asarray(pts_2d, dtype=np.float64)).reshape(-1, 2)
    pts_3d = np.ascontiguousarray(np.asarray(pts_3d, dtype=np.float64)).reshape(-1, 3) * scale
    n = pts_2d.shape[0]
    if n < 4:                                                   # cv2.error branch of the reference (:40-42)
        return np.eye(4)[:3], np.eye(4), []
    pose, mask, cnt = ransac_pnp_batch(torch.from_numpy(np.asarray(K, dtype=np.float64))[None].to(dev), torch.from_numpy(pts_2d).to(dev),
                                       torch.from_numpy(pts_3d).to(dev), torch.tensor([0, n], dtype=torch.int32, device=dev), method=method,
                                       confidence=confidence)
    if int(cnt[0]) == 0:
        return np.eye(4)[:3], np.eye(4), []
    pose = pose[0].cpu().numpy()
    pose[:, 3] /= scale
    pose_homo = np.concatenate([pose, np.array([[0, 0, 0, 1.0]])], axis=0)
    inliers = torch.nonzero(mask).to(torch.int32).cpu().numpy().reshape(-1, 1)
    return pose, pose_homo, inliers
