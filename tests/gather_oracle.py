"""ORACLE -- test infrastructure, NOT product code.

The hand-off from the matcher to the pose solver restated in numpy: the reference's
``valid = matches > -1; mkpts2d = kpts2d[valid]; mkpts3d = kpts3d[matches[valid]]; mconf = confidence[valid]``
(``inference.py:147-152``, ``src/utils/eval_utils.py:72-77``), applied frame by frame and concatenated in the layout
``opb_gather_matches`` writes.  An index >= M is treated as no match (the reference would raise on it).
"""
import numpy as np


def gather_matches(matches0, keypoints2d, keypoints3d, matching_scores0=None):
    """matches0 int64 [B,N], keypoints2d fp32 [B,N,2], keypoints3d fp32 [M,3], matching_scores0 fp32 [B,N] or None ->
    dict(pts2d f64 [T,2], pts3d f64 [T,3], mconf fp32 [T] or None, query_index int32 [T], offsets int32 [B+1])."""
    matches0 = np.asarray(matches0)
    M = len(keypoints3d)
    p2, p3, conf, qi, off = [], [], [], [], [0]
    for b in range(matches0.shape[0]):
        m = matches0[b]
        valid = (m > -1) & (m < M)
        p2.append(keypoints2d[b][valid].astype(np.float64))
        p3.append(keypoints3d[m[valid]].astype(np.float64))
        if matching_scores0 is not None:
            conf.append(matching_scores0[b][valid])
        qi.append(np.nonzero(valid)[0].astype(np.int32))
        off.append(off[-1] + int(valid.sum()))
    return {"pts2d": np.concatenate(p2).reshape(-1, 2), "pts3d": np.concatenate(p3).reshape(-1, 3),
            "mconf": np.concatenate(conf).astype(np.float32) if matching_scores0 is not None else None,
            "query_index": np.concatenate(qi).astype(np.int32), "offsets": np.array(off, np.int32)}


def gather_objects_numpy(matches0, keypoints2d, keypoints3d, object_ids, matching_scores0=None):
    """numpy restatement of the mixed gather (``opb_gather_matches_objects``): frame b keeps entries 0 <= m < M_b of its object
    and reads that object's key points (the reference's kpts3d[matches[valid]] per frame), frame-major, ascending query index.
    keypoints3d maps object id -> [M_b, 3]; same outputs as ``gather_matches``."""
    p2, p3, conf, qi, off = [], [], [], [], [0]
    for b, oid in enumerate(object_ids):
        kp3 = keypoints3d[oid]
        m = matches0[b]
        valid = (m > -1) & (m < len(kp3))
        p2.append(keypoints2d[b][valid].astype(np.float64))
        p3.append(kp3[m[valid]].astype(np.float64))
        if matching_scores0 is not None:
            conf.append(matching_scores0[b][valid])
        qi.append(np.nonzero(valid)[0].astype(np.int32))
        off.append(off[-1] + int(valid.sum()))
    return {"pts2d": np.concatenate(p2).reshape(-1, 2), "pts3d": np.concatenate(p3).reshape(-1, 3),
            "mconf": np.concatenate(conf).astype(np.float32) if matching_scores0 is not None else None,
            "query_index": np.concatenate(qi).astype(np.int32), "offsets": np.array(off, np.int32)}
