"""Per-object 3D feature construction on the GPU -- the producers of the tensors the matcher consumes.

Mirrors the reference functions (same names, arguments, results):

* ``pad_features3d_random`` / ``build_features3d_leaves``  -- reference ``src/utils/data_utils.py:143-160`` / ``:163-205``
  (what ``inference.py:113-130`` calls once per sequence to build ``descriptors3d_db`` and ``descriptors2d_db``);
* ``mean_descriptors`` / ``mean_scores``                   -- reference ``src/sfm/postprocess/feature_process.py:297-317``
  (the offline step that writes ``anno_3d_average.npz``).

The leaf selection of ``build_features3d_leaves`` is defined by numpy's global RNG (one ``np.random.permutation`` per 3D
point, reference ``:182-192``); the index list is drawn on the host with exactly those calls -- so that the same
``np.random.seed`` gives byte-identical tensors -- and the column gather / dustbin / padding run in one CUDA kernel
(``opb_gather_features3d``).  The segmented means run in fp64 on the device and reproduce numpy's summation order
(sequential over rows for the [len, 256] descriptors, pairwise for the [len, 1] scores), bit for bit.

There is no CPU path: results are CUDA tensors (``inference.py``'s later ``.cuda()`` calls are no-ops on them).
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib


def _dev(device):
    d = torch.device(device if device is not None else "cuda")
    if d.type != "cuda":
        raise RuntimeError("onepose_b200 has no CPU path: device must be a CUDA device")
    return d


def _as_f32(x, device):
    # reference: torch.Tensor(x) -> float32 (data_utils.py:148-151, :165-168)
    if not isinstance(x, torch.Tensor):
        x = torch.from_numpy(np.ascontiguousarray(np.asarray(x, dtype=np.float32)))
    return x.to(device=device, dtype=torch.float32).contiguous()


def _gather(desc, scores, idx, n_out, device):
    dim, n_src = desc.shape
    out_d = torch.empty(dim, n_out, dtype=torch.float32, device=device)
    out_s = torch.empty(n_out, 1, dtype=torch.float32, device=device)
    n_idx = min(int(idx.numel()) if idx is not None else n_src, n_out)
    _lib.call(device, "opb_gather_features3d", desc, scores, dim, n_src, idx, n_idx, out_d, out_s, n_out)
    return out_d, out_s


def pad_features3d_random(descriptors, scores, n_target_shape, device=None):
    """Pad (all-ones descriptors, zero scores) or truncate the averaged 3D features to ``n_target_shape`` points.
    descriptors [dim, n], scores [n, 1] -> ([dim, n_target], [n_target, 1]) fp32.  Reference data_utils.py:143-160."""
    device = _dev(device)
    d = _as_f32(descriptors, device)
    s = _as_f32(scores, device).reshape(-1)
    return _gather(d, s, None, int(n_target_shape), device)


def build_features3d_leaves(descriptors, scores, idxs, n_target_shape, num_leaf, device=None):
    """Fix the number of 2D leaf features per 3D point to ``num_leaf``: points with fewer observations are filled with the
    dustbin (all-ones descriptor, zero score), points with more keep a random subset; then pad / truncate to
    ``n_target_shape`` points.  descriptors [dim, sum(idxs)], scores [sum(idxs), 1], idxs [n_points] track lengths
    -> ([dim, num_leaf * n_target], [num_leaf * n_target, 1]) fp32.  Reference data_utils.py:163-205."""
    device = _dev(device)
    d = _as_f32(descriptors, device)
    s = _as_f32(scores, device).reshape(-1)
    idxs = np.asarray(idxs)
    n_src = d.shape[1]
    dustbin = n_src                                     # index of the appended dustbin column (:175-177)
    ends = np.cumsum(idxs, axis=0)
    starts = np.insert(ends[:-1], 0, 0)
    picks = []
    for lo, hi in zip(starts, ends):                    # one RNG draw per point, same calls as the reference (:182-192)
        n_obs = hi - lo
        if num_leaf > n_obs:
            cand = np.arange(lo, hi).tolist() + [dustbin] * (num_leaf - n_obs)
            picks.append(np.random.permutation(np.array(cand)))
        else:
            picks.append(np.random.permutation(np.arange(lo, hi))[:num_leaf])
    sel = np.concatenate(picks, axis=0).astype(np.int64)
    assert sel.shape[0] == idxs.shape[0] * num_leaf
    sel_dev = torch.from_numpy(sel).to(device)
    return _gather(d, s, sel_dev, int(num_leaf) * int(n_target_shape), device)


def _segmented(name, values, idxs, D, device, *dims):
    """Entry point ``name`` over the segments of ``values`` -> f64 [n_points, D]; ``dims`` are its arguments after M."""
    device = _dev(device)
    v = torch.as_tensor(np.ascontiguousarray(np.asarray(values, dtype=np.float64)) if not isinstance(values, torch.Tensor) else values)
    v = v.to(device=device, dtype=torch.float64).contiguous()
    lens = torch.as_tensor(np.asarray(idxs, dtype=np.int64)).to(device)
    M = int(lens.numel())
    out = torch.empty(M, D, dtype=torch.float64, device=device)
    _lib.call(device, name, v, lens, M, *dims, out)
    return out


def mean_descriptors(descriptors, idxs, device=None):
    """Average the leaf descriptors of every 3D point: descriptors [sum(idxs), D] fp64 -> [n_points, D] fp64
    (np.mean over each track's rows).  Reference feature_process.py:297-305."""
    D = int(descriptors.shape[1])
    return _segmented("opb_segmented_mean_f64", descriptors, idxs, D, device, D)


def mean_scores(scores, idxs, device=None):
    """Average the leaf scores of every 3D point: scores [sum(idxs), 1] fp64 -> [n_points, 1] fp64.
    Reference feature_process.py:308-317."""
    return _segmented("opb_segmented_mean_scores_f64", scores, idxs, 1, device)
