"""Per-object 3D feature construction on the GPU -- the producers of the tensors the matcher consumes.

Mirrors the reference functions (same names, arguments, results):

* ``pad_features3d_random`` / ``build_features3d_leaves``  -- reference ``src/utils/data_utils.py:143-160`` / ``:163-205``
  (what ``inference.py:113-130`` calls once per sequence to build ``descriptors3d_db`` and ``descriptors2d_db``);
* ``mean_descriptors`` / ``mean_scores``                   -- reference ``src/sfm/postprocess/feature_process.py:297-317``
  (the offline step that writes ``anno_3d_average.npz``).

The leaf selection of ``build_features3d_leaves`` is defined by numpy's global RNG (one ``np.random.permutation`` per 3D
point, reference ``:182-192``); the index list is drawn on the host with exactly those calls -- so that the same
``np.random.seed`` gives byte-identical tensors -- and the column gather / dustbin / padding run in one CUDA kernel
(``opb_gather_features3d``).  The segmented means run in fp64 on the device and reproduce numpy's result bit for bit,
summation order included; ``_mean`` states the rule.

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


def _mean(name, values, idxs, device):
    """np.mean(values[s:e], axis=0) of every track [s, e) of ``idxs``, bit for bit -> f64 [n_points, D] on the device.

    numpy's reduction loop runs along the axis of ``values`` with the smaller stride, and that sets the summation order:
      * rows contiguous (a C-ordered [sum(idxs), D] array, or a row-strided or column-sliced view of one), D > 1: numpy adds the
        rows in order, one running sum per channel;
      * the reduced axis contiguous (an F-ordered array such as ``obs.T`` of channel-first [D, sum(idxs)] features, a strided
        view of one, or D = 1): numpy sums each channel's track pairwise.
    Both sums start from numpy's identity +0.0, so an all -0.0 track gives +0.0; a zero-length track gives NaN.  The layout is
    read here, before anything is made contiguous, and the device gets the rows (first case) or the channels (second) in
    order.  Only fp64 is accepted: the reference's producer builds these arrays in fp64 (``np.empty`` / ``np.append``,
    feature_process.py:143-188), and np.mean of fp32 input accumulates in fp32, which this port does not reproduce."""
    device = _dev(device)
    x = values if isinstance(values, torch.Tensor) else np.asarray(values)
    if x.dtype != (torch.float64 if isinstance(x, torch.Tensor) else np.float64):
        raise ValueError(f"{name}: values must be fp64 (the reference's feature files hold fp64 arrays), got {x.dtype}")
    if x.ndim == 1:
        x = x[:, None]
    D = int(x.shape[1])
    s0, s1 = x.stride() if isinstance(x, torch.Tensor) else x.strides
    pairwise = D == 1 or abs(s0) < abs(s1)
    if isinstance(x, torch.Tensor):
        v = (x.T if pairwise else x).to(device).contiguous()
    else:
        v = torch.from_numpy(np.ascontiguousarray(x.T if pairwise else x)).to(device)
    lens = torch.as_tensor(np.asarray(idxs, dtype=np.int64)).to(device)
    M = int(lens.numel())
    out = torch.empty(M, D, dtype=torch.float64, device=device)
    _lib.call(device, "opb_segmented_mean_channels_f64" if pairwise else "opb_segmented_mean_f64", v, lens, M, D, out)
    return out


def mean_descriptors(descriptors, idxs, device=None):
    """Average the leaf descriptors of every 3D point: descriptors [sum(idxs), D] fp64 -> [n_points, D] fp64
    (np.mean over each track's rows, in numpy's summation order for the layout given).  Reference feature_process.py:297-305."""
    return _mean("mean_descriptors", descriptors, idxs, device)


def mean_scores(scores, idxs, device=None):
    """Average the leaf scores of every 3D point: scores [sum(idxs), 1] fp64 -> [n_points, 1] fp64.
    Reference feature_process.py:308-317."""
    return _mean("mean_scores", scores, idxs, device)
