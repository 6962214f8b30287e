"""A model of the 2D half of the reference's get_kpt_ann (src/sfm/postprocess/feature_process.py): each image's assign matrix
(count_features :95-135 and get_assign_matrix :197-230) and the text of its annotation file (save_2d_anno_for_each_image
:233-262).

count_features keeps, per image and in feature order, {kept COLMAP point id: feature index}: a repeated id overwrites the
index (the last feature wins) but keeps the id's first position.  get_assign_matrix walks those ids in order and pairs each
with its merge group unless the group was paired before in the image.  ``first_wins`` and ``dedup=False`` plant the two
defects the tests require to break equality with the fixture.
"""
import json

import numpy as np


def group_map(group_ids, group_offsets) -> dict:
    """id_mapping (:47-56): {COLMAP point id: its group}."""
    off = np.asarray(group_offsets, np.int64)
    return {int(x): g for g in range(len(off) - 1) for x in np.asarray(group_ids, np.int64)[off[g]:off[g + 1]]}


def assign_pairs(point_ids, gmap: dict, first_wins: bool = False, dedup: bool = True) -> np.ndarray:
    """The assign matrix int64 [2, k] of one image whose features observe ``point_ids`` (-1: none)."""
    last = {}
    for k, x in enumerate(np.asarray(point_ids, np.int64).tolist()):
        if x in gmap and not (first_wins and x in last):
            last[x] = k
    seen, pairs = set(), []
    for x, k in last.items():
        g = gmap[x]
        if dedup and g in seen:
            continue
        seen.add(g)
        pairs.append((k, g))
    return np.array(pairs, np.int64).reshape(-1, 2).T.copy()


def anno_text(keypoints, descriptors, scores, assign) -> str:
    """json.dump's text of one image's file: keypoints fp32 [n, 2], descriptors fp32 [D, n], scores fp32 [n], assign [2, k]."""
    return json.dumps({"keypoints2d": np.asarray(keypoints, np.float32).tolist(), "descriptors2d": np.asarray(descriptors, np.float32).tolist(),
                       "scores2d": np.asarray(scores, np.float32).reshape(-1, 1).tolist(), "assign_matrix": np.asarray(assign).tolist(),
                       "num_matches": int(np.asarray(assign).shape[1])})


def _values(rng, shape) -> np.ndarray:
    """fp32 values over every exponent, with zeros, integers, powers of two and the fixed / exponent notation edges planted."""
    v = rng.integers(0, 2 ** 32, shape, dtype=np.uint64).astype(np.uint32).view(np.float32).copy()
    flat = v.reshape(-1)
    special = np.array([0.0, -0.0, 1.0, -2.0, 0.1, 1e-4, 9.999999e-5, 1e16, 9.99999e15, 123.0, 2.0 ** -149, 3.4028235e38, 0.5, 16777216.0],
                       np.float32)
    pick = rng.choice(flat.size, min(flat.size, 3 * special.size), replace=False)
    flat[pick] = np.resize(special, pick.size)
    nonfinite = ~np.isfinite(flat)
    flat[nonfinite] = rng.normal(size=int(nonfinite.sum())).astype(np.float32)
    return v


def features(seed: int, F: int, D: int, cap: int):
    """The planted images' features: keypoints fp32 [F, cap, 2], descriptors fp32 [F, D, cap], scores fp32 [F, cap]."""
    rng = np.random.default_rng(seed)
    kp = _values(rng, (F, cap, 2))
    kp[:, : cap // 2] = rng.uniform(0, 512, (F, cap // 2, 2)).astype(np.float32)   # pixel coordinates
    de = _values(rng, (F, D, cap))
    sc = _values(rng, (F, cap))
    sc[:, 0], sc[:, 1] = np.inf, np.nan              # json's Infinity and NaN
    return kp, de, sc
