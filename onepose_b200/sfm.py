"""An object's SfM post-processing on the GPU: the reference's ``run.py postprocess`` (:142-163) from COLMAP's model and the
images' device features to the arrays of ``anno_3d_average.npz``, ``anno_3d_collect.npz`` and ``idxs.npy``.

    get_tkl + filter_3d      filter_tkl.py:35-52, filter_points.py:8-83    opb_sfm_filter_points
    merge                    filter_points.py:86-117                       opb_sfm_merge_points
    get_kpt_ann (3D half)    feature_process.py:95-188, :320-363           opb_sfm_gather_observations, opb_sfm_gather_features,
                                                                           then features3d.mean_descriptors / mean_scores

The readers parse COLMAP's binary model on the host (its documented layout).  ``postprocess`` runs the steps on the caller's
stream; the counts stay on the device until one read, after the last step that sizes an output, brings the counts, ``idxs`` and
the groups to the host in one copy.

The 2D half of get_kpt_ann (feature_process.py:95-135, :197-294) follows from ``postprocess``'s groups:

    count_features + get_assign_matrix     opb_sfm_assign_pairs                             assign_matrices
    save_2d_anno (per-image JSON text)     opb_anno2d_text_lengths, opb_anno2d_text_write   save_anno_2d

COLMAP triangulation and the PLY visualisation are not part of it.
"""
from __future__ import annotations

import ctypes
import json
import os
import struct

import numpy as np
import torch

from . import _lib, features3d

INT32_MAX = 2 ** 31 - 1


def _model_bytes(path) -> bytes:
    with open(path, "rb") as f:
        return f.read()


class _Cursor:
    def __init__(self, data: bytes, path):
        self.data, self.pos, self.path = data, 0, str(path)

    def take(self, fmt: str):
        n = struct.calcsize(fmt)
        if self.pos + n > len(self.data):
            raise ValueError(f"{self.path}: truncated at byte {self.pos} (needs {n} more bytes, has {len(self.data) - self.pos})")
        v = struct.unpack_from(fmt, self.data, self.pos)
        self.pos += n
        return v

    def array(self, dtype, count: int) -> np.ndarray:
        dt = np.dtype(dtype)
        n = dt.itemsize * count
        if count < 0 or self.pos + n > len(self.data):
            raise ValueError(f"{self.path}: truncated at byte {self.pos} (a record of {count} entries does not fit)")
        v = np.frombuffer(self.data, dtype=dt, count=count, offset=self.pos)
        self.pos += n
        return v

    def end(self):
        if self.pos != len(self.data):
            raise ValueError(f"{self.path}: {len(self.data) - self.pos} bytes after the last record")


def read_points3d_bin(path):
    """COLMAP's points3D.bin -> (ids int64 [P], xyz f64 [P, 3], track lengths int64 [P]) in file order.  Layout: uint64 P, then
    per point uint64 id, 3 f64 xyz, 3 uint8 rgb, f64 error, uint64 track length L, L x (int32 image id, int32 point2D idx)."""
    c = _Cursor(_model_bytes(path), path)
    (P,) = c.take("<Q")
    if P > len(c.data):
        raise ValueError(f"{path}: header claims {P} points in {len(c.data)} bytes")
    ids = np.empty(P, np.int64)
    xyz = np.empty((P, 3), np.float64)
    lens = np.empty(P, np.int64)
    for i in range(P):
        rec = c.take("<Q3d3BdQ")
        ids[i] = np.uint64(rec[0]).astype(np.int64)
        xyz[i] = rec[1:4]
        lens[i] = rec[8]
        c.array("<i4", 2 * rec[8])
    c.end()
    return ids, xyz, lens


def read_images_bin(path):
    """COLMAP's images.bin -> [(name, point3D_ids int64 [n_i])] in file order, -1 for a feature without a 3D point.  Layout:
    uint64 count, then per image uint32 id, 4 f64 qvec, 3 f64 tvec, uint32 camera id, a NUL-terminated name, uint64 n_i,
    n_i x (f64 x, f64 y, int64 point3D id)."""
    c = _Cursor(_model_bytes(path), path)
    (n,) = c.take("<Q")
    if n > len(c.data):
        raise ValueError(f"{path}: header claims {n} images in {len(c.data)} bytes")
    out = []
    for _ in range(n):
        c.take("<I7dI")
        end = c.data.find(b"\x00", c.pos)
        if end < 0:
            raise ValueError(f"{path}: image name without its terminating NUL at byte {c.pos}")
        name = c.data[c.pos:end].decode("utf-8")
        c.pos = end + 1
        (k,) = c.take("<Q")
        rows = c.array(np.dtype([("x", "<f8"), ("y", "<f8"), ("id", "<i8")]), k)
        out.append((name, rows["id"].astype(np.int64)))
    c.end()
    return out


def _ws(dev, name: str, *args) -> torch.Tensor:
    """A workspace of the size that the query ``name`` gives for ``args`` (torch's allocations are 256-byte aligned)."""
    b = ctypes.c_int64()
    _lib.check(getattr(_lib.load(), name)(*args, ctypes.byref(b)))
    return torch.empty(max(int(b.value), 1), dtype=torch.uint8, device=dev)


def _device_features(features, F: int):
    sc, de = features.get("scores"), features.get("descriptors")
    for name, t, nd in (("scores", sc, 2), ("descriptors", de, 3)):
        if not isinstance(t, torch.Tensor) or t.device.type != "cuda" or t.dtype != torch.float32 or t.dim() != nd:
            raise ValueError(f"opb_sfm_gather_features: features[{name!r}] must be a CUDA fp32 tensor of {nd} dimensions "
                             f"(forward_padded's), got {getattr(t, 'dtype', type(t))} {list(getattr(t, 'shape', []))}")
    if sc.shape[0] != F or de.shape[0] != F or de.shape[2] != sc.shape[1]:
        raise ValueError(f"opb_sfm_gather_features: scores [F, cap] and descriptors [F, D, cap] must hold the {F} images with one cap, "
                         f"got {list(sc.shape)} and {list(de.shape)}")
    if de.device != sc.device:
        raise ValueError("opb_sfm_gather_features: scores and descriptors must be on one device")
    return sc.contiguous(), de.contiguous()


def _point_id_table(images, n_obs, cap: int) -> np.ndarray:
    """Image f's COLMAP point ids in row f of an int64 [F, cap] table, -1 past its count."""
    F = len(images)
    flat = np.concatenate([np.asarray(p, np.int64) for _, p in images])
    starts = np.cumsum(n_obs) - n_obs
    pid = np.full((F, cap), -1, np.int64)
    pid[np.repeat(np.arange(F), n_obs), np.arange(len(flat)) - np.repeat(starts, n_obs)] = flat
    return pid


def _images(images, image_names):
    if isinstance(images, (str, os.PathLike)):
        images = read_images_bin(os.path.join(images, "images.bin"))
    if image_names is not None:
        by_name = dict(images)
        missing = [n for n in image_names if n not in by_name]
        if missing:
            raise ValueError(f"images {missing[:3]} are not in the model")
        images = [(n, by_name[n]) for n in image_names]
    return images


def postprocess(points3d, images, features, box_corners, max_num_kp3d: int = 2500, dist_threshold: float = 1e-3,
                image_names=None) -> dict:
    """run.py postprocess on the device.

    points3d      read_points3d_bin's (ids, xyz, track lengths), or a model directory (``sfm_ws/model``) holding points3D.bin
    images        read_images_bin's [(name, point3D_ids)], or a model directory holding images.bin
    features      SuperPoint.forward_padded's dict for the same images in the same order: scores [F, cap], descriptors
                  [F, D, cap] (fp32, CUDA); image f's features are 0 .. len(point3D_ids) - 1.  get_kpt_ann walks run.py's
                  img_lists, which generate_empty sorted in place by frame index, so pass the images in that order
    image_names   the names of the images in the features' order, picked from ``images`` by name; None: ``images`` as given
    box_corners   [8, 3], e.g. scan.read_box(...)[0] or np.loadtxt(box3d_corners.txt)

    Returns the reference's arrays, CUDA tensors unless stated: keypoints3d [n, 3] f64; descriptors3d [D, n] and scores3d [n, 1]
    f64, the averages; descriptors3d_collect [D, total] and scores3d_collect [total, 1] f64; idxs int64 [n] (numpy); track_length
    (int); group_offsets int64 [n + 1] and group_ids int64 [sum]: group g's COLMAP point ids are group_ids[group_offsets[g] :
    group_offsets[g + 1]] (numpy)."""
    if isinstance(points3d, (str, os.PathLike)):
        points3d = read_points3d_bin(os.path.join(points3d, "points3D.bin"))
    if isinstance(images, (str, os.PathLike)):
        images = read_images_bin(os.path.join(images, "images.bin"))
    if image_names is not None:
        by_name = dict(images)
        missing = [n for n in image_names if n not in by_name]
        if missing:
            raise ValueError(f"postprocess: images {missing[:3]} are not in the model")
        images = [(n, by_name[n]) for n in image_names]
    ids, xyz, lens = (np.asarray(a) for a in points3d)
    P = int(ids.shape[0])
    if P == 0:
        raise ValueError("postprocess: the model has no 3D points")
    if ids.shape != (P,) or xyz.shape != (P, 3) or lens.shape != (P,) or P > INT32_MAX:
        raise ValueError(f"postprocess: points3d must be ids [P], xyz [P, 3] and track lengths [P], got {ids.shape}, {xyz.shape}, {lens.shape}")
    if int(max_num_kp3d) < 0 or int(max_num_kp3d) > INT32_MAX:
        raise ValueError(f"postprocess: max_num_kp3d must be >= 0, got {max_num_kp3d}")
    if not dist_threshold > 0:
        raise ValueError(f"postprocess: dist_threshold must be > 0, got {dist_threshold}")
    corners = np.asarray(box_corners, dtype=np.float64)
    if corners.shape != (8, 3):
        raise ValueError(f"postprocess: box_corners must be [8, 3], got {list(corners.shape)}")
    F = len(images)
    if F == 0:
        raise ValueError("postprocess: no images")
    sc, de = _device_features(features, F)
    dev = sc.device
    cap, D = int(sc.shape[1]), int(de.shape[1])
    n_obs = np.array([len(p) for _, p in images], np.int64)
    if n_obs.max() > cap:
        raise ValueError(f"opb_sfm_gather_observations: an image has {n_obs.max()} features, above the features' cap {cap}")
    if F * cap > INT32_MAX:
        raise ValueError(f"opb_sfm_gather_observations: F * cap = {F * cap} is above {INT32_MAX}")
    pid = _point_id_table(images, n_obs, cap)

    order = np.argsort(ids, kind="stable")        # filter_by_track_length walks the ids sorted
    with torch.cuda.device(dev):
        # pinned, stream-ordered uploads: the host does not wait for work already queued on the caller's stream
        up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory().to(dev, non_blocking=True)  # noqa: E731
        d_ids, d_xyz, d_len = up(ids[order].astype(np.int64)), up(xyz[order].astype(np.float64)), up(lens[order].astype(np.int64))
        d_corners, d_pid = up(corners), up(pid)
        d_counts = up(n_obs.astype(np.int32))
        # everything the host needs, read in one copy: the counts, then idxs [P], member ids [P] and group offsets [P + 1]
        blk = torch.zeros(6 + 3 * P + 1, dtype=torch.int64, device=dev)
        t_len, n_kept, n_groups, n_members, total, missing = (blk[i:i + 1] for i in range(6))
        idxs, member_ids, offsets64 = blk[6:6 + P], blk[6 + P:6 + 2 * P], blk[6 + 2 * P:]
        kept_ids = torch.empty(P, dtype=torch.int64, device=dev)
        kept_xyz = torch.empty(P, 3, dtype=torch.float32, device=dev)
        ws = _ws(dev, "opb_sfm_filter_workspace_bytes", P)
        _lib.call(dev, "opb_sfm_filter_points", d_ids, d_xyz, d_len, P, int(max_num_kp3d), d_corners, ws, ws.numel(), kept_ids, kept_xyz,
                  t_len, n_kept)
        merged = torch.empty(P, 3, dtype=torch.float64, device=dev)
        offsets = torch.empty(P + 1, dtype=torch.int32, device=dev)
        member_index = torch.empty(P, dtype=torch.int32, device=dev)
        slot_of = torch.empty(P, dtype=torch.int32, device=dev)
        ws = _ws(dev, "opb_sfm_merge_workspace_bytes", P)
        _lib.call(dev, "opb_sfm_merge_points", kept_xyz, kept_ids, n_kept, P, float(dist_threshold), ws, ws.numel(), merged, offsets, member_ids,
                  member_index, slot_of, n_groups, n_members)
        obs_order = torch.empty(F * cap, dtype=torch.int32, device=dev)
        ws = _ws(dev, "opb_sfm_gather_workspace_bytes", F, cap, P)
        _lib.call(dev, "opb_sfm_gather_observations", d_pid, d_counts, F, cap, kept_ids, n_kept, P, slot_of, offsets, n_groups, ws, ws.numel(),
                  obs_order, idxs, total, missing)
        offsets64.copy_(offsets)      # rows past the group count are unwritten and never read
        h = blk.cpu().numpy()                                           # the one synchronisation
        track_length, nk, n, nm, tot, miss = (int(v) for v in h[:6])
        if nk == 0:
            raise ValueError(f"postprocess: no point passes the track-length ({track_length}) and box filters")
        idxs_h, ids_h, offsets_h = h[6:6 + n].copy(), h[6 + P:6 + P + nm].copy(), h[6 + 2 * P:6 + 2 * P + n + 1].copy()
        if miss < nm:
            raise ValueError(f"opb_sfm_gather_observations: point {int(ids_h[miss])} belongs to a group but no image observes it")
        out_desc = torch.empty(tot, D, dtype=torch.float64, device=dev)
        out_scores = torch.empty(tot, 1, dtype=torch.float64, device=dev)
        _lib.call(dev, "opb_sfm_gather_features", obs_order, tot, F, cap, D, sc, de, out_desc, out_scores)
        avg_desc = features3d.mean_descriptors(out_desc, idxs_h, dev)
        avg_scores = features3d.mean_scores(out_scores, idxs_h, dev)
        return {
            "keypoints3d": merged[:n],
            "descriptors3d": avg_desc.T,
            "scores3d": avg_scores,
            "descriptors3d_collect": out_desc.T,
            "scores3d_collect": out_scores,
            "idxs": idxs_h,
            "track_length": track_length,
            "group_offsets": offsets_h,
            "group_ids": ids_h,
        }


def save_anno(anno_dir, result: dict) -> None:
    """Write ``anno_3d_average.npz``, ``anno_3d_collect.npz`` and ``idxs.npy`` as save_3d_anno does (feature_process.py:191-194,
    :357-363): keypoints3d [n, 3], descriptors3d [D, n] or [D, total], scores3d [n, 1] or [total, 1], all f64; idxs int64 [n]."""
    os.makedirs(anno_dir, exist_ok=True)
    host = lambda t: t.cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)  # noqa: E731
    xyz = host(result["keypoints3d"])
    np.savez(os.path.join(anno_dir, "anno_3d_average.npz"), keypoints3d=xyz, descriptors3d=host(result["descriptors3d"]),
             scores3d=host(result["scores3d"]))
    np.savez(os.path.join(anno_dir, "anno_3d_collect.npz"), keypoints3d=xyz, descriptors3d=host(result["descriptors3d_collect"]),
             scores3d=host(result["scores3d_collect"]))
    np.save(os.path.join(anno_dir, "idxs.npy"), np.asarray(result["idxs"], dtype=np.int64))


ANNO2D_CHUNK_BYTES = 1 << 30       # the default bound of save_anno_2d's device text buffer
_ITEM_BOUND = 27                   # bytes of an item at most: ", " or "], [" and a 23-character float repr
_OBJECT_BOUND = 128                # the section keys, their brackets and num_matches' closing brace


def _assign_device(result: dict, images, features, image_names):
    """opb_sfm_assign_pairs on postprocess's groups: (device, pairs int64 [2, F * cap] on the device, offsets [F + 1] and
    num_matches [F] on the host, the number of features of each image, cap)."""
    images = _images(images, image_names)
    F = len(images)
    if F == 0:
        raise ValueError("opb_sfm_assign_pairs: no images")
    sc, _ = _device_features(features, F)
    dev, cap = sc.device, int(sc.shape[1])
    n_obs = np.array([len(p) for _, p in images], np.int64)
    if n_obs.max() > cap:
        raise ValueError(f"opb_sfm_assign_pairs: an image has {n_obs.max()} features, above the features' cap {cap}")
    ids = np.asarray(result["group_ids"], np.int64)
    off = np.asarray(result["group_offsets"], np.int64)
    if ids.size == 0 or off.shape != (off.size,) or off[0] != 0 or off[-1] != ids.size or (np.diff(off) < 0).any():
        raise ValueError("opb_sfm_assign_pairs: result must hold postprocess's group_ids and group_offsets")
    group = np.repeat(np.arange(off.size - 1, dtype=np.int32), np.diff(off))
    order = np.argsort(ids, kind="stable")          # id_mapping's table, searched by id
    kept, kept_group = ids[order], group[order]
    if (np.diff(kept) == 0).any():
        raise ValueError("opb_sfm_assign_pairs: a COLMAP point id is in two groups")
    pid = _point_id_table(images, n_obs, cap)
    with torch.cuda.device(dev):
        up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory().to(dev, non_blocking=True)  # noqa: E731
        d_pid, d_counts, d_kept, d_group = up(pid), up(n_obs.astype(np.int32)), up(kept), up(kept_group)
        pairs = torch.empty(2, F * cap, dtype=torch.int64, device=dev)
        counts = torch.empty(2 * F + 1, dtype=torch.int64, device=dev)     # offsets [F + 1], then num_matches [F]: one read
        ws = _ws(dev, "opb_sfm_assign_workspace_bytes", F, cap)
        _lib.call(dev, "opb_sfm_assign_pairs", d_pid, d_counts, F, cap, d_kept, d_group, int(kept.size), ws, ws.numel(), pairs,
                  counts[:F + 1], counts[F + 1:])
        h = counts.cpu().numpy()
    return dev, pairs, h[:F + 1].copy(), h[F + 1:].copy(), n_obs, cap


def assign_matrices(result: dict, images, features, image_names=None):
    """count_features + get_assign_matrix (feature_process.py:95-135, :197-230) on the device.

    result        postprocess's result (its group_ids and group_offsets)
    images, features, image_names   as given to postprocess, in the same order

    Returns (the assign matrices, num_matches int64 [F]): image f's matrix is int64 [2, k_f], row 0 its features and row 1 their
    groups (the rows of keypoints3d), one pair per group seen in the image, in the order of the group's first feature; the
    feature is the last one with that first feature's COLMAP point id.  An image without a kept point has a [2, 0] matrix."""
    dev, pairs, offsets, num, _, _ = _assign_device(result, images, features, image_names)
    h = pairs[:, :int(offsets[-1])].cpu().numpy()
    return [h[:, offsets[f]:offsets[f + 1]].copy() for f in range(len(num))], num


def _chunks(bounds: np.ndarray, limit: int):
    """Runs of consecutive images whose text bounds sum to at most ``limit`` bytes."""
    out, start, total = [], 0, 0
    for i, b in enumerate(bounds):
        if b > limit:
            raise ValueError(f"save_anno_2d: one image's text may take {int(b)} bytes, above max_chunk_bytes = {limit}")
        if total + b > limit:
            out.append((start, i))
            start, total = i, 0
        total += int(b)
    out.append((start, len(bounds)))
    return out


def save_anno_2d(anno_dir, img_paths, result: dict, images, features, image_names=None, detection: str = "superpoint",
                 max_chunk_bytes: int = ANNO2D_CHUNK_BYTES) -> list:
    """save_2d_anno (feature_process.py:233-294) on the device: for every image with a pair, ``anno_<detection>/<name>.json``
    beside the image's directory (<dirname(dirname(img_path))>/anno_<detection>/, .png -> .json), byte for byte as json.dump
    writes {"keypoints2d", "descriptors2d", "scores2d", "assign_matrix", "num_matches"}; then ``<anno_dir>/anno_2d.json``, the
    list of {"anno_id", "anno_file", "img_file", "pose_file"} (/color/ -> /poses_ba/, .png -> .txt) over the written images.

    img_paths     the images' paths in the features' order (run.py's img_lists)
    features      forward_padded's dict: keypoints [F, cap, 2], scores [F, cap], descriptors [F, D, cap] (fp32, CUDA)
    max_chunk_bytes   the bound of the device text buffer: the images go in chunks whose text fits it, one host read each

    Returns the index list that anno_2d.json holds."""
    img_paths = [str(p) for p in img_paths]
    dev, pairs, offsets, num, n_obs, cap = _assign_device(result, images, features, image_names)
    F = len(num)
    if len(img_paths) != F:
        raise ValueError(f"save_anno_2d: {len(img_paths)} image paths for {F} images")
    sc, de = _device_features(features, F)
    kp = features.get("keypoints")
    if not isinstance(kp, torch.Tensor) or kp.device != sc.device or kp.dtype != torch.float32 or tuple(kp.shape) != (F, cap, 2):
        raise ValueError(f"save_anno_2d: features['keypoints'] must be a CUDA fp32 tensor [{F}, {cap}, 2] on the scores' device")
    kp = kp.contiguous()
    D = int(de.shape[1])
    written = np.nonzero(num > 0)[0]
    items = 3 * n_obs[written] + D * n_obs[written] + 2 * num[written] + 1
    files = []
    for f in written:
        p = img_paths[f]
        d = os.path.join(os.path.dirname(os.path.dirname(p)), f"anno_{detection}")
        os.makedirs(d, exist_ok=True)
        files.append(os.path.join(d, os.path.basename(p).replace(".png", ".json")))
    if int(max_chunk_bytes) <= 0:
        raise ValueError(f"save_anno_2d: max_chunk_bytes must be > 0, got {max_chunk_bytes}")
    with torch.cuda.device(dev):
        for c0, c1 in (_chunks(_ITEM_BOUND * items + _OBJECT_BOUND, int(max_chunk_bytes)) if written.size else []):
            Fc = c1 - c0
            w = written[c0:c1]
            desc = np.stack([w, n_obs[w], num[w], offsets[w]], axis=1).astype(np.int64)
            item_off = np.concatenate([[0], np.cumsum(items[c0:c1])]).astype(np.int64)
            up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory().to(dev, non_blocking=True)  # noqa: E731
            d_desc, d_item_off = up(desc), up(item_off)
            n_items, max_items = int(item_off[-1]), int(items[c0:c1].max())
            ws = _ws(dev, "opb_anno2d_text_workspace_bytes", Fc, n_items)
            text_off = torch.empty(Fc + 1, dtype=torch.int64, device=dev)
            _lib.call(dev, "opb_anno2d_text_lengths", d_desc, d_item_off, Fc, n_items, max_items, D, cap, kp, de, sc, pairs, F * cap, ws,
                      ws.numel(), text_off)
            t = text_off.cpu().numpy()                                   # the chunk's one synchronisation
            text = torch.empty(max(int(t[-1]), 1), dtype=torch.uint8, device=dev)
            _lib.call(dev, "opb_anno2d_text_write", d_desc, d_item_off, Fc, max_items, D, cap, kp, de, sc, pairs, F * cap, ws, text_off,
                      text)
            host = torch.empty(text.numel(), dtype=torch.uint8, pin_memory=True)
            host.copy_(text, non_blocking=True)
            torch.cuda.current_stream(dev).synchronize()
            buf = memoryview(host.numpy())
            for i in range(Fc):
                with open(files[c0 + i], "wb") as fh:
                    fh.write(buf[t[i]:t[i + 1]])
    annotations = [{"anno_id": i + 1, "anno_file": files[i], "img_file": img_paths[f],
                    "pose_file": img_paths[f].replace("/color/", "/poses_ba/").replace(".png", ".txt")} for i, f in enumerate(written)]
    os.makedirs(anno_dir, exist_ok=True)
    with open(os.path.join(anno_dir, "anno_2d.json"), "w") as fh:
        json.dump(annotations, fh)
    return annotations
