"""numpy model of the reference's SfM post-processing (run.py postprocess, :142-163): get_tkl, filter_3d, merge and the 3D half
of get_kpt_ann, restated step by step with the arithmetic pinned where the reference leaves it to a library:

* the box test of filter_by_3d_box in fp32, m = ((d0 v0 + d1 v1) + d2 v2) with every product and sum rounded on its own (torch's
  CPU dot may sum in another order, so fixtures keep points away from the box planes);
* scipy's pdist as s = dx*dx, s += dy*dy, s += dz*dz on the fp32 rows widened to fp64, then sqrt;
* np.mean of a group's fp32 rows (an fp32 sum in member order, an fp32 divide).

``features(seed, F, D, cap)`` makes integer-valued features (exact in fp32) that the fixture generator and the tests share.
"""
from __future__ import annotations

import numpy as np
from scipy.spatial import cKDTree


MOD = 4194301          # a prime above every F * cap the tests use (300 * 4096): each feature's values are its own


def features(seed: int, F: int, D: int, cap: int):
    """scores [F, cap] and descriptors [F, D, cap] fp32: integers below 2^22 over powers of two, exact in fp32 and fp64.  Feature
    (f, k) is numbered f * 8192 + k; its score and its descriptor's first channel are distinct for every number below MOD, so
    no two features of a model share either."""
    f = np.arange(F, dtype=np.int64)[:, None, None]
    d = np.arange(D, dtype=np.int64)[None, :, None]
    k = np.arange(cap, dtype=np.int64)[None, None, :]
    idx = f * 8192 + k
    desc = (((idx * 1299709 + d * 104729 + seed * 31) % MOD) - MOD // 2).astype(np.float32) / np.float32(1 << 20)
    sc = (((idx[:, 0] * 7919 + seed) % MOD) + 1).astype(np.float32) / np.float32(1 << 22)
    return sc, desc


def get_tkl(lens, thres: int) -> int:
    """filter_tkl.get_tkl: walk the lengths present in ascending order, subtracting each one's count from P; the first length at
    which at most ``thres`` points remain."""
    values, counts = np.unique(np.asarray(lens), return_counts=True)
    remaining = len(lens)
    for v, c in zip(values, counts):
        remaining -= int(c)
        if remaining <= thres:
            return int(v)
    raise ValueError("get_tkl: no track length brings the points below the threshold")


def box_keep(xyz, corners) -> np.ndarray:
    """filter_by_3d_box's keep mask of fp64 points [n, 3] in fp32."""
    p = np.asarray(xyz, dtype=np.float32)
    c = np.asarray(corners, dtype=np.float32)
    d = p - c[4]
    keep = np.ones(len(p), dtype=bool)
    for corner in (5, 0, 7):
        v = c[corner] - c[4]
        m = (d[:, 0] * v[0] + d[:, 1] * v[1]) + d[:, 2] * v[2]
        vv = (v[0] * v[0] + v[1] * v[1]) + v[2] * v[2]
        keep &= (np.float32(0) < m) & (m < vv)
    return keep


def filter_3d(ids, xyz, lens, track_length: int, corners):
    """filter_by_track_length (ids ascending, length >= track_length) then the box: (kept ids int64, kept xyz fp32 [n, 3])."""
    order = np.argsort(ids, kind="stable")
    ids, xyz, lens = np.asarray(ids)[order], np.asarray(xyz)[order], np.asarray(lens)[order]
    sel = lens >= track_length
    ids, xyz = ids[sel], xyz[sel]
    keep = box_keep(xyz, corners)
    return ids[keep].astype(np.int64), xyz[keep].astype(np.float32)


def pdist_pair(a, b) -> float:
    d = a.astype(np.float64) - b.astype(np.float64)
    s = d[0] * d[0]
    s = s + d[1] * d[1]
    s = s + d[2] * d[2]
    return float(np.sqrt(s))


def neighbour_lists(xyz32, threshold: float):
    """Each row's neighbours (pdist < threshold), itself included, ascending.  Candidates from a k-d tree with a margin, then the
    exact test."""
    n = len(xyz32)
    rows = [[j] for j in range(n)]
    x = xyz32.astype(np.float64)
    for i, j in sorted(cKDTree(x).query_pairs(threshold * (1 + 1e-6) + 1e-300)):
        if pdist_pair(xyz32[i], xyz32[j]) < threshold:
            rows[i].append(j)
            rows[j].append(i)
    return [np.array(sorted(r), dtype=np.int64) for r in rows]


def merge(xyz32, ids, threshold: float = 1e-3):
    """filter_points.merge: (merged xyz f64 [n, 3], [member rows of each group]).  Row j is skipped when any of its neighbours
    is recorded already; otherwise its neighbours form the next group and are recorded."""
    recorded = np.zeros(len(xyz32), dtype=bool)
    pos, groups = [], []
    for j, row in enumerate(neighbour_lists(xyz32, threshold)):
        if recorded[row].any():
            continue
        s = np.zeros(3, dtype=np.float32)
        for i in row:
            s = s + xyz32[i]
        pos.append((s / np.float32(len(row))).astype(np.float64))
        groups.append(row)
        recorded[row] = True
    return np.array(pos, dtype=np.float64).reshape(-1, 3), groups


def gather(point3d_ids, member_ids):
    """get_kpt_ann's observation order: for each group member in order, its (image, feature) pairs in image then feature order.
    point3d_ids: per image (the caller's order) int64 [n_i]; member_ids: per group the members' ids.  Raises KeyError for a member
    without an observation, as the reference does.  -> (obs int64 [total, 2], idxs int64 [n])."""
    seen = {}
    for f, p in enumerate(point3d_ids):
        for k in np.nonzero(np.asarray(p) != -1)[0]:
            seen.setdefault(int(p[k]), []).append((f, int(k)))
    obs, idxs = [], []
    for g in member_ids:
        c = 0
        for q in g:
            rows = seen[int(q)]
            obs.extend(rows)
            c += len(rows)
        idxs.append(c)
    return np.array(obs, dtype=np.int64).reshape(-1, 2), np.array(idxs, dtype=np.int64)


def postprocess(ids, xyz, lens, point3d_ids, scores, descriptors, corners, max_num_kp3d=2500, dist_threshold=1e-3) -> dict:
    """The whole step on host arrays; scores [F, cap], descriptors [F, D, cap] fp32 as the device extractor pads them."""
    if len(ids) == 0 or max_num_kp3d < 0:
        raise ValueError("postprocess: no points, or max_num_kp3d < 0")
    tl = get_tkl(lens, max_num_kp3d)
    kept_ids, kept_xyz = filter_3d(ids, xyz, lens, tl, corners)
    if len(kept_ids) == 0:
        raise ValueError("postprocess: no point passes the filters")
    merged, groups = merge(kept_xyz, kept_ids, dist_threshold)
    member_ids = [kept_ids[g] for g in groups]
    obs, idxs = gather(point3d_ids, member_ids)
    desc = descriptors[obs[:, 0], :, obs[:, 1]].astype(np.float64)          # [total, D]
    sc = scores[obs[:, 0], obs[:, 1]].astype(np.float64)[:, None]
    ends = np.cumsum(idxs)
    starts = ends - idxs
    avg_d = np.concatenate([np.mean(desc[s:e], axis=0).reshape(1, -1) for s, e in zip(starts, ends)], axis=0)
    avg_s = np.concatenate([np.mean(sc[s:e], axis=0).reshape(1, -1) for s, e in zip(starts, ends)], axis=0)
    return {"track_length": tl, "kept_ids": kept_ids, "keypoints3d": merged, "groups": member_ids, "obs": obs, "idxs": idxs,
            "descriptors3d": avg_d.T, "scores3d": avg_s, "descriptors3d_collect": desc.T, "scores3d_collect": sc}
