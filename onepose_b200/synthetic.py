"""Seeded synthetic weights / objects / frames for the GATsSPG hot path.

Everything here is numpy ``RandomState`` based so that the same seed gives the
same bytes in this container, on the GPU box and inside the golden-fixture
generator (``tests/golden/make_golden.py``) -- no dependence on torch's RNG or
on the reference tree.

Recipe follows SURVEY.md section 8(d) / section 7 step 0:
  * weights: reference-shaped state dict (key names as produced by
    ``GATsSuperGlue`` -- reference ``GATs_SuperGlue.py:143-177`` and
    ``GATs.py:25-28``), optionally *damped* (``mlp[-1].weight *= 0.02``,
    ``final_proj.weight = I + 0.02 W0``) so that planted correspondences
    survive the 0.2 threshold;
  * object: unit-norm 3D descriptors ``[256, M]`` and leaves ``[256, M*L]``
    with column ``i*L + j`` = leaf j of point i (reference ``GATs.py:46``);
  * frame: unit-norm query descriptors ``[256, N]``, the first N/2 columns
    planted as noisy copies of a random subset of the 3D descriptors.
"""
from __future__ import annotations

import numpy as np

D = 256
HEADS = 4
GNN_LAYERS = ["GATs", "self", "cross"] * 4  # reference GATs_SuperGlue.py:162

DEFAULT_HPARAMS = {
    # reference configs/experiment/train_GATsSPG.yaml:44-60
    "descriptor_dim": 256,
    "keypoints_encoder": [32, 64, 128],
    "match_type": "softmax",
    "scale_factor": 0.07,
    "match_threshold": 0.2,
    "include_self": True,
    "additional": False,
    "with_linear_transform": False,
}


def _conv(rs: np.random.RandomState, cout: int, cin: int):
    """Conv1d(k=1) default init: U(-1/sqrt(fan_in), 1/sqrt(fan_in)) for both."""
    bound = 1.0 / np.sqrt(cin)
    w = rs.uniform(-bound, bound, size=(cout, cin, 1)).astype(np.float32)
    b = rs.uniform(-bound, bound, size=(cout,)).astype(np.float32)
    return w, b


def _kenc(rs, sd, prefix, inp_dim, layers, feature_dim):
    """Dead parameters (reference GATs_SuperGlue.py:131-160); present so that a
    reference checkpoint / state dict round-trips."""
    chans = [inp_dim] + list(layers) + [feature_dim]
    idx = 0
    for i in range(1, len(chans)):
        w, b = _conv(rs, chans[i], chans[i - 1])
        if i == len(chans) - 1:
            b[:] = 0.0
        sd[f"{prefix}.encoder.{idx}.weight"] = w
        sd[f"{prefix}.encoder.{idx}.bias"] = b
        idx += 1
        if i < len(chans) - 1:
            idx += 2  # InstanceNorm1d (no params) + ReLU


def make_state_dict(seed: int = 0, damped: bool = True, hparams: dict | None = None, mlp3_scale: float | None = None):
    """Reference-keyed state dict (numpy fp32 arrays).  ``mlp3_scale`` overrides the 0.02 damping of the layers' last
    convolution (1.0 = the reference initialisation) while keeping the near-identity final projection: the knob of the
    precision sweep (tools/damping_sweep.py) -- the larger it is, the larger the residual updates every GEMM error rides on."""
    hp = dict(DEFAULT_HPARAMS if hparams is None else hparams)
    d = hp["descriptor_dim"]
    rs = np.random.RandomState(seed)
    sd: dict[str, np.ndarray] = {}
    _kenc(rs, sd, "kenc_2d", 3, hp["keypoints_encoder"], d)
    _kenc(rs, sd, "kenc_3d", 4, hp["keypoints_encoder"], d)
    for i, name in enumerate(GNN_LAYERS):
        p = f"gnn.layers.{i}"
        if name == "GATs":
            std = 1.414 * np.sqrt(2.0 / (d + d))
            sd[f"{p}.W"] = (rs.randn(d, d) * std).astype(np.float32)
            std = 1.414 * np.sqrt(2.0 / (2 * d + 1))
            sd[f"{p}.a"] = (rs.randn(2 * d, 1) * std).astype(np.float32)
        else:
            w, b = _conv(rs, d, d)
            sd[f"{p}.attn.merge.weight"], sd[f"{p}.attn.merge.bias"] = w, b
            for j in range(3):
                w, b = _conv(rs, d, d)
                sd[f"{p}.attn.proj.{j}.weight"], sd[f"{p}.attn.proj.{j}.bias"] = w, b
            w, b = _conv(rs, 2 * d, 2 * d)
            sd[f"{p}.mlp.0.weight"], sd[f"{p}.mlp.0.bias"] = w, b
            w, b = _conv(rs, d, 2 * d)
            b[:] = 0.0  # reference GATs_SuperGlue.py:109
            if mlp3_scale is not None:
                w *= mlp3_scale
            elif damped:
                w *= 0.02
            sd[f"{p}.mlp.3.weight"], sd[f"{p}.mlp.3.bias"] = w, b
    w, b = _conv(rs, d, d)
    if damped or mlp3_scale is not None:
        w = (np.eye(d, dtype=np.float32)[:, :, None] + 0.02 * w).astype(np.float32)
    sd["final_proj.weight"], sd["final_proj.bias"] = w, b
    sd["bin_score"] = np.array(1.0, dtype=np.float32)
    return sd


def _unit_cols(x: np.ndarray) -> np.ndarray:
    return (x / np.linalg.norm(x, axis=0, keepdims=True)).astype(np.float32)


def make_object(object_id: int, M: int, L: int = 8, d: int = D):
    """Per-object constants: (descriptors3d_db [d, M], descriptors2d_db [d, M*L])."""
    rs = np.random.RandomState(1000 + object_id)
    db = _unit_cols(rs.randn(d, M))
    leaves = _unit_cols(np.repeat(db, L, axis=1) + 0.02 * rs.randn(d, M * L))
    return db, leaves


def make_frame(frame_id: int, db: np.ndarray, N: int):
    """Query descriptors [d, N]; first N//2 columns planted on db[:, perm]."""
    d, M = db.shape
    rs = np.random.RandomState(frame_id)
    q = rs.randn(d, N)
    n_plant = min(N // 2, M)
    perm = rs.permutation(M)[:n_plant]
    q[:, :n_plant] = db[:, perm] + 0.03 * rs.randn(d, n_plant)
    return _unit_cols(q), perm


def make_batch(object_id: int, frame_ids, N: int, M: int, L: int = 8):
    """Reference-shaped input dict (numpy, batch-first, channel-first descriptors;
    reference inference.py:80-94) for frames of ONE object."""
    db, leaves = make_object(object_id, M, L)
    qs = [make_frame(f, db, N)[0] for f in frame_ids]
    B = len(qs)
    return {
        "keypoints2d": np.zeros((B, N, 2), np.float32),
        "keypoints3d": np.zeros((B, M, 3), np.float32),
        "descriptors2d_query": np.stack(qs, 0),
        "descriptors3d_db": np.repeat(db[None], B, 0),
        "descriptors2d_db": np.repeat(leaves[None], B, 0),
    }


def make_tracks(seed: int, M: int, d: int = D, max_len: int = 12):
    """Variable-length multi-view tracks for the offline segmented mean
    (reference feature_process.py:297-305): (descriptors [sum_len, d] f64, idxs [M])."""
    rs = np.random.RandomState(seed)
    idxs = rs.randint(1, max_len + 1, size=M).astype(np.int64)
    desc = rs.randn(int(idxs.sum()), d)
    return desc, idxs


def make_track_scores(seed: int, idxs: np.ndarray):
    """Per-observation detection scores [sum_len, 1] f64 for ``mean_scores`` (reference feature_process.py:308-317);
    wide dynamic range so that the summation order matters."""
    rs = np.random.RandomState(seed + 7919)
    n = int(np.sum(idxs))
    return rs.rand(n, 1) * np.exp(3.0 * rs.randn(n, 1))


def make_sfm_features(seed: int, n_points: int, d: int = D, max_len: int = 14):
    """Stand-in for the per-object SfM feature files (reference feature_process.py:191-194, :357-363): unit-norm fp32
    observation descriptors [d, sum_len], scores [sum_len, 1], track lengths idxs [n_points], and the per-point averages
    (descriptors3d [d, n_points], scores3d [n_points, 1]) -- inputs of pad_features3d_random / build_features3d_leaves."""
    rs = np.random.RandomState(seed)
    idxs = rs.randint(1, max_len + 1, size=n_points).astype(np.int64)
    centers = _unit_cols(rs.randn(d, n_points))
    obs = _unit_cols(np.repeat(centers, idxs, axis=1) + 0.02 * rs.randn(d, int(idxs.sum())))
    obs_scores = rs.rand(int(idxs.sum()), 1).astype(np.float32)
    ends = np.cumsum(idxs)
    starts = ends - idxs
    avg = np.stack([obs[:, s:e].mean(axis=1) for s, e in zip(starts, ends)], 1).astype(np.float32)
    avg_scores = np.stack([obs_scores[s:e].mean(axis=0) for s, e in zip(starts, ends)], 0).astype(np.float32)
    return obs, obs_scores, idxs, avg, avg_scores


def make_pnp_scene(seed: int, n: int, outlier_frac: float = 0.4, noise_px: float = 0.5, size: int = 512):
    """Matched 2D-3D correspondences of one frame for the pose solver (reference eval_utils.py:18-42): an object of ~10 cm
    about 50-80 cm in front of a 512 x 512 crop camera, pixel noise on the inliers, uniformly random 2D positions for the
    outliers.  Returns (K [3,3], pts2d [n,2], pts3d [n,3], pose_gt [3,4]) as float64 (3D points in metres)."""
    rs = np.random.RandomState(seed)
    K = np.array([[600.0 + 50 * rs.rand(), 0, size / 2 + 5 * rs.randn()], [0, 600.0 + 50 * rs.rand(), size / 2 + 5 * rs.randn()], [0, 0, 1.0]])
    w = rs.randn(3)
    th = np.linalg.norm(w)
    k = w / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    R = np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx
    t = np.array([0.03 * rs.randn(), 0.03 * rs.randn(), 0.5 + 0.3 * rs.rand()])
    P = 0.05 * rs.randn(n, 3)
    X = P @ R.T + t
    uv = X[:, :2] / X[:, 2:3] * np.array([K[0, 0], K[1, 1]]) + np.array([K[0, 2], K[1, 2]])
    uv += noise_px * rs.randn(n, 2)
    out = rs.rand(n) < outlier_frac
    uv[out] = rs.rand(int(out.sum()), 2) * size
    return K, uv, P, np.concatenate([R, t[:, None]], 1)


def make_planted_scene(object_id: int, frame_ids, N: int, M: int, L: int = 8, unplanted=(), noise_px: float = 0.5, size: int = 512):
    """An object and B frames that the matcher and the pose solver can both get right: ``make_object`` descriptors, M 3D points
    (metres, ~10 cm across; keypoints3d fp32 [M,3]) and per frame a camera K, a ground-truth pose and ``make_frame`` query
    descriptors whose planted column i sits at the projection of 3D point perm[i] (plus ``noise_px`` of pixel noise); unplanted
    columns have key points uniform in the size x size crop.  Frames listed in ``unplanted`` get random descriptors only.
    Returns a dict of numpy arrays: desc3d [256,M], desc2d_db [256,M*L], keypoints3d [M,3] f32, K [B,3,3] f64,
    descriptors2d [B,256,N] f32, keypoints2d [B,N,2] f32, pose_gt [B,3,4] f64, n_planted [B]."""
    db, leaves = make_object(object_id, M, L)
    rs = np.random.RandomState(5000 + object_id)
    P = (0.05 * rs.randn(M, 3)).astype(np.float32)
    Ks, qs, kps, gts, npl = [], [], [], [], []
    for f in frame_ids:
        if f in unplanted:
            q, perm = _unit_cols(np.random.RandomState(f).randn(db.shape[0], N)), np.zeros(0, np.int64)
        else:
            q, perm = make_frame(f, db, N)
        frs = np.random.RandomState(7000 + f)
        K = np.array([[600.0 + 50 * frs.rand(), 0, size / 2 + 5 * frs.randn()], [0, 600.0 + 50 * frs.rand(), size / 2 + 5 * frs.randn()],
                      [0, 0, 1.0]])
        w = frs.randn(3)
        th = np.linalg.norm(w)
        k = w / th
        Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
        R = np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx
        t = np.array([0.03 * frs.randn(), 0.03 * frs.randn(), 0.5 + 0.3 * frs.rand()])
        kp = frs.rand(N, 2) * size
        X = P[perm].astype(np.float64) @ R.T + t
        kp[:len(perm)] = X[:, :2] / X[:, 2:3] * np.array([K[0, 0], K[1, 1]]) + np.array([K[0, 2], K[1, 2]]) + noise_px * frs.randn(len(perm), 2)
        Ks.append(K); qs.append(q); kps.append(kp.astype(np.float32)); gts.append(np.concatenate([R, t[:, None]], 1)); npl.append(len(perm))
    return {"desc3d": db, "desc2d_db": leaves, "keypoints3d": P, "K": np.stack(Ks), "descriptors2d": np.stack(qs),
            "keypoints2d": np.stack(kps), "pose_gt": np.stack(gts), "n_planted": np.array(npl)}


# ---------------------------------------------------------------------------------------------
# SuperPoint extractor (SURVEY 8f N4): reference-shaped state dict and seeded grey images
# ---------------------------------------------------------------------------------------------
SUPERPOINT_LAYERS = [
    # name, C_out, C_in, kernel  (reference src/models/extractors/SuperPoint/superpoint.py:111-126)
    ("conv1a", 64, 1, 3), ("conv1b", 64, 64, 3), ("conv2a", 64, 64, 3), ("conv2b", 64, 64, 3),
    ("conv3a", 128, 64, 3), ("conv3b", 128, 128, 3), ("conv4a", 128, 128, 3), ("conv4b", 128, 128, 3),
    ("convPa", 256, 128, 3), ("convPb", 65, 256, 1), ("convDa", 256, 128, 3), ("convDb", 256, 256, 1),
]

# the extractor configuration inference.py runs with (src/sfm/extract_features.py:19-24).  NB the key 'keypoints_threshold'
# is NOT the key SuperPoint reads ('keypoint_threshold', superpoint.py:99,164): the default 0.005 stays in force.
SUPERPOINT_CONF = {"descriptor_dim": 256, "nms_radius": 3, "max_keypoints": 4096, "keypoints_threshold": 0.6}


def make_superpoint_state_dict(seed: int = 0, score_gain: float = 6.0):
    """He-initialised conv stack (activations stay O(1) through the ReLUs); the score head's last layer is scaled by
    ``score_gain`` so that the 65-way softmax is peaked and the 0.005 threshold actually separates pixels."""
    rs = np.random.RandomState(7000 + seed)
    sd = {}
    for name, cout, cin, k in SUPERPOINT_LAYERS:
        fan_in = cin * k * k
        w = (rs.standard_normal((cout, cin, k, k)) * np.sqrt(2.0 / fan_in)).astype(np.float32)
        b = rs.uniform(-0.05, 0.05, size=(cout,)).astype(np.float32)
        if name == "convPb":
            w *= np.float32(score_gain)
        sd[name + ".weight"] = w
        sd[name + ".bias"] = b
    return sd


def make_image(seed: int, H: int, W: int):
    """Grey image in [0, 1], fp32 [1, H, W]: a few smooth blobs and edges plus fine texture (corners for the detector)."""
    rs = np.random.RandomState(9000 + seed)
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float64)
    img = np.zeros((H, W))
    for _ in range(12):
        cy, cx = rs.uniform(0, H), rs.uniform(0, W)
        sy, sx = rs.uniform(H / 20, H / 4), rs.uniform(W / 20, W / 4)
        img += rs.uniform(-1, 1) * np.exp(-(((yy - cy) / sy) ** 2 + ((xx - cx) / sx) ** 2))
    for _ in range(6):   # rectangles: sharp corners
        y0, x0 = int(rs.uniform(0, H * 0.8)), int(rs.uniform(0, W * 0.8))
        y1, x1 = y0 + int(rs.uniform(8, H * 0.3)), x0 + int(rs.uniform(8, W * 0.3))
        img[y0:y1, x0:x1] += rs.uniform(-0.6, 0.6)
    img += 0.15 * rs.standard_normal((H, W))
    img = (img - img.min()) / (img.max() - img.min())
    return img.astype(np.float32)[None]
