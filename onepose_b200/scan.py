"""An annotated scan's object poses, boxes and colour crops on the GPU: ``parse_scanned_data.py``'s ``data_process_anno``.

The reference turns each ``*-annotate`` sequence of an ARKit scan into what ``inference.py`` evaluates against
(``parse_scanned_data.py:184-240`` and ``parse_video``, ``:129-181``): the object pose ``T_oc`` of every frame (``poses/``), the
512 x 512 colour crop around the object's projected box (``color/``, which the evaluation's ``GT_box`` mode and the SfM read),
its ``K_crop`` (``intrin/``), the crop-to-frame transform (``M/``) and the box in crop coordinates (``bbox/``).  The readers here
parse the scan's text files on the host; ``object_poses`` and ``annotate`` do the rest on the device with no host
synchronisation (``csrc/scan.cu`` behind ``opb_scan_poses`` / ``opb_scan_crop_geometry``, and ``crop.crop_frames_colour``):

    K = scan.read_intrinsics("Frames.txt")
    bbox3d, T_ow = scan.read_box("Box.txt")
    arposes = scan.read_arposes("ARposes.txt")
    ann = scan.annotate(frames_bgr, K, arposes, T_ow, bbox3d)          # frames_bgr: the decoded video, uint8 [F, H, W, 3] CUDA

The crops are cut from the colour frames and stay colour, as the reference writes them; the evaluation makes them grey with
``frames.grey_frames(ann["image"])``, the pixels ``cv2.imread(..., IMREAD_GRAYSCALE)`` reads back (INTEGRATION.md).
Decoding the video and writing files are the caller's.
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib, crop

FLOAT_EPS = float(np.finfo(np.float64).eps)
MAX_CORNERS = 1024
MAX_ROWS = (1 << 31) - 1


# ---- transforms3d's two functions the reference calls, in full ----

def quat2mat(q) -> np.ndarray:
    """``transforms3d.quaternions.quat2mat``: q = (w, x, y, z) -> [3, 3] f64 with its non-normalising formula, s = 2 / (w² + x² +
    y² + z²); the identity when that norm is below float64 eps.  Equal to the rotation of q / |q| for any larger q."""
    w, x, y, z = (float(v) for v in q)
    Nq = w * w + x * x + y * y + z * z
    if Nq < FLOAT_EPS:
        return np.eye(3)
    s = 2.0 / Nq
    X, Y, Z = x * s, y * s, z * s
    wX, wY, wZ = w * X, w * Y, w * Z
    xX, xY, xZ = x * X, x * Y, x * Z
    yY, yZ, zZ = y * Y, y * Z, z * Z
    return np.array([[1.0 - (yY + zZ), xY - wZ, xZ + wY],
                     [xY + wZ, 1.0 - (xX + zZ), yZ - wX],
                     [xZ - wY, yZ + wX, 1.0 - (xX + yY)]])


def compose(t, R) -> np.ndarray:
    """``transforms3d.affines.compose(t, R, np.ones(3))``: [R t; 0 1], f64 [4, 4]."""
    A = np.eye(4)
    A[:3, :3] = np.asarray(R, np.float64)
    A[:3, 3] = np.asarray(t, np.float64)
    return A


# ---- the scan's text files (host: they are file formats) ----

def _text(path) -> str:
    with open(path, "r") as f:
        return f.read()


def read_intrinsics(frames_txt) -> np.ndarray:
    """``Frames.txt`` -> K f64 [3, 3], as ``data_process_anno`` (``:186-192``) averages it: lines starting with ``#`` skipped,
    columns 2-5 (fx, fy, cx, cy) of the rest averaged by ``np.average``.  Blank lines are skipped too (the reference's
    ``len(l) > 0`` test sees their newline and fails on them)."""
    lines = [ln.strip() for ln in _text(frames_txt).splitlines(keepends=True) if len(ln) > 0 and ln[0] != "#"]
    rows = [[float(e) for e in ln.split(",")] for ln in lines if ln]
    if not rows or any(len(r) != len(rows[0]) or len(r) < 6 for r in rows):
        raise ValueError("Frames.txt must hold rows of at least 6 comma-separated numbers, all of one length")
    fx, fy, cx, cy = np.average(np.array(rows), axis=0)[2:6]
    return np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float64)


def _box_values(box_txt) -> list:
    lines = _text(box_txt).splitlines(keepends=True)
    if len(lines) < 2:
        raise ValueError("Box.txt must hold a header line and a data line")
    data = [float(e) for e in lines[1].strip().split(",")]
    if len(data) != 10:
        raise ValueError(f"Box.txt's data line must hold 10 numbers (position, extent, quaternion), got {len(data)}")
    return data


def read_box(box_txt):
    """``Box.txt`` -> (bbox3d f64 [8, 3], T_ow f64 [4, 4]): ``get_bbox3d``'s corners (``:88-105``, its order, ``* 0.5`` of the
    extents) and ``parse_box``'s object-to-world transform (``:107-115``, ``compose(position, quat2mat(quaternion))``).  Its second
    line is read, as there."""
    data = _box_values(box_txt)
    ex, ey, ez = data[3:6]
    bbox3d = np.array([[-ex, -ey, -ez], [ex, -ey, -ez], [ex, -ey, ez], [-ex, -ey, ez],
                       [-ex, ey, -ez], [ex, ey, -ez], [ex, ey, ez], [-ex, ey, ez]]) * 0.5
    return bbox3d, compose(data[:3], quat2mat(data[6:]))


def read_arposes(arposes_txt) -> np.ndarray:
    """``ARposes.txt`` -> f64 [n, 8] rows (timestamp, x, y, z, qw, qx, qy, qz), skipping what ``data_process_anno`` skips
    (``:205-207``): lines empty after stripping, or starting with ``#``."""
    rows = []
    for ln in _text(arposes_txt).splitlines():
        ln = ln.strip()
        if len(ln) == 0 or ln[0] == "#":
            continue
        r = [float(e) for e in ln.split(",")]
        if len(r) != 8:
            raise ValueError(f"an ARposes row must hold 8 numbers (timestamp, position, quaternion w-first), got {len(r)}: {ln!r}")
        rows.append(r)
    return np.array(rows, np.float64).reshape(-1, 8)


# ---- on the device ----

def _f64(t, shape: tuple, name: str, dev) -> torch.Tensor:
    t = torch.as_tensor(t)
    if not (t.dtype.is_floating_point or t.dtype in (torch.int32, torch.int64)) or tuple(t.shape) != shape:
        raise ValueError(f"{name} must be a real {list(shape)} array or tensor, got {t.dtype} {list(t.shape)}")
    return t.to(device=dev, dtype=torch.float64).contiguous()


def _scan_args(K, arposes, T_ow, bbox3d, dev):
    rows = torch.as_tensor(arposes)
    if rows.dim() != 2 or rows.shape[1] != 8 or not 0 < rows.shape[0] <= MAX_ROWS:
        raise ValueError(f"arposes must be [n, 8] with n >= 1 (read_arposes' rows), got {list(rows.shape)}")
    corners = torch.as_tensor(bbox3d)
    if corners.dim() != 2 or corners.shape[1] != 3 or not 0 < corners.shape[0] <= MAX_CORNERS:
        raise ValueError(f"bbox3d must be [n, 3] with 1 <= n <= {MAX_CORNERS}, got {list(corners.shape)}")
    n, nc = int(rows.shape[0]), int(corners.shape[0])
    return (_f64(K, (3, 3), "K", dev), _f64(rows, (n, 8), "arposes", dev), _f64(T_ow, (4, 4), "T_ow", dev), _f64(corners, (nc, 3), "bbox3d", dev),
            n, nc)


def _poses(dev, K, rows, T_ow, corners, n, nc, n_out):
    out = {"pose": torch.empty(n_out, 4, 4, dtype=torch.float64, device=dev), "proj": torch.empty(n_out, nc, 2, dtype=torch.float64, device=dev),
           "box": torch.empty(n_out, 4, dtype=torch.int32, device=dev), "row": torch.empty(n_out, dtype=torch.int32, device=dev),
           "keep": torch.empty(n, dtype=torch.int32, device=dev), "count": torch.empty(1, dtype=torch.int32, device=dev)}
    _lib.call(dev, "opb_scan_poses", K, rows, n, T_ow, corners, nc, n_out, out["pose"], out["proj"], out["box"], out["row"], out["keep"],
              out["count"])
    return out


def _device(device, *args) -> torch.device:
    for a in args:
        if isinstance(a, torch.Tensor) and a.device.type == "cuda":
            return a.device
    dev = torch.device(device if device is not None else "cuda")
    if dev.type != "cuda":
        raise RuntimeError("onepose_b200 has no CPU path: tensors must be on a CUDA device")
    return dev


def object_poses(K, arposes, T_ow, bbox3d, device=None) -> dict:
    """``data_process_anno``'s loop over the ARposes rows (``:202-238``, downsample_rate 1) in one launch: K [3,3] (from
    ``read_intrinsics``), arposes [n,8] (``read_arposes``), T_ow [4,4] and bbox3d [8,3] (``read_box``), as arrays or tensors;
    computed on the device of the first CUDA tensor among them, else on ``device`` (default the current CUDA device).

    Per row: quat2mat, the flip ``diag(1, -1, -1)``, ``T_cw = [R p; 0 1]``, ``T_oc = inv(T_cw) @ T_ow``, the corners' projection
    ``K_homo @ T_oc @ corners_homo`` (``reproj``, ``:118-126``), and the skip rule ``x0 < -1000 or y0 < -1000 or x1 > 3000 or y1 >
    3000`` on its min / max.

    The pairing is the reference's: a skipped row does not advance its ``index`` (``:233-238``), so the kept rows are numbered
    0, 1, ... in file order; ``parse_video`` then gives video frame i the i-th kept row, and stops at the first frame without one
    (``:145-146``: its ``continue`` does not advance ``index`` either), so frames past the kept count get nothing.  The kept rows
    are compacted on the device.  Returns device tensors, slot i being the i-th kept row (video frame i):

    - pose f64 [n,4,4]: T_oc (``poses/i.txt``); zeros in the slots past the kept count
    - proj f64 [n,8,2]: the projected corners (``reproj_box/i.txt``); zeros past the kept count
    - box int32 [n,4]: ``[x0, y0, x1, y1]`` of ``astype(int)`` of proj, truncation towards zero; [0,0,0,0] past the kept count
    - row int32 [n]: the ARposes row of the slot (index into arposes); -1 past the kept count
    - keep int32 [n]: per ARposes row, 1 if kept, 0 if skipped
    - count int32 [1]: the number of kept rows

    No host synchronisation."""
    dev = _device(device, K, arposes, T_ow, bbox3d)
    K, rows, T_ow, corners, n, nc = _scan_args(K, arposes, T_ow, bbox3d, dev)
    return _poses(dev, K, rows, T_ow, corners, n, nc, n)


def annotate(frames_bgr: torch.Tensor, K, arposes, T_ow, bbox3d, crop_size: int = 512) -> dict:
    """``data_process_anno`` for F decoded video frames: the poses of ``object_poses`` paired with the frames as the reference
    pairs them, then ``parse_video``'s two crops of each frame (``:147-178``).  frames_bgr uint8 [F,H,W,3] (or [F,H,W,4]) CUDA,
    packed pixels at any row and frame stride, as ``cv2.VideoCapture`` decodes them; K, arposes, T_ow, bbox3d as in
    ``object_poses``; crop_size S (512 in the reference; S % 8 == 0).

    Returns device tensors per frame f:

    - pose f64 [F,4,4]: T_oc of the f-th kept row; zeros where there is none
    - box int32 [F,4]: the projected box, ``astype(int)`` min / max
    - image uint8 [F,S,S,C]: the crop written to ``color/f.png``, colour in the frames' channel order, ``cv2.warpAffine``'s pixels
    - K_crop f64 [F,3,3] (``intrin/``), M f64 [F,3,3] = ``inv(T2 @ T1)`` (``M/``)
    - box_crop f64 [F,4]: min / max of the corners projected with ``K_crop_homo`` (``bbox/``), not truncated
    - status int32 [F]: 1, or 0 for a frame with no kept row or an unusable box (empty, or beyond what the crop addresses),
      where image, M and box_crop are zero

    One call, four launches on the current stream, no host synchronisation."""
    dev, F = crop._colour_frames_args(frames_bgr)[:2]
    K, rows, T_ow, corners, n, nc = _scan_args(K, arposes, T_ow, bbox3d, dev)
    S = int(crop_size)
    if S <= 0 or S % 8 or S > crop.MAX_SIDE:
        raise ValueError(f"crop_size must be a positive multiple of 8 up to {crop.MAX_SIDE}, got {crop_size!r}")
    p = _poses(dev, K, rows, T_ow, corners, n, nc, F)
    c = crop.crop_frames_colour(frames_bgr, p["box"], K, S)
    out = {"pose": p["pose"], "box": p["box"], "image": c["image"], "K_crop": c["K_crop"],
           "M": torch.empty(F, 3, 3, dtype=torch.float64, device=dev), "box_crop": torch.empty(F, 4, dtype=torch.float64, device=dev),
           "status": c["status"]}
    _lib.call(dev, "opb_scan_crop_geometry", c["trans"], c["K_crop"], p["pose"], corners, nc, c["status"], F, out["M"], out["box_crop"])
    return out
