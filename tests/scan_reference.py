"""Numpy and cv2 model of the reference's processing of an annotated scan (parse_scanned_data.py's data_process_anno, :184-240,
and parse_video, :129-181): the test oracle of ``onepose_b200/scan.py`` and ``csrc/scan.cu``.  Each function restates the
reference's lines with the file reads, writes and the video decode taken out; ``transforms3d``'s ``quat2mat`` and
``affines.compose`` are stated in full (tests/test_scan_reference_cpu.py pins them).

The pairing of rows and frames follows the reference's two loops: a skipped ARposes row does not advance ``index``, and
parse_video's ``continue`` at a missing box file does not either, so video frame i gets the i-th kept row and no frame after
the first one without a kept row gets anything."""
import cv2
import numpy as np

FLIP = np.array([[1, 0, 0], [0, -1, 0], [0, 0, -1]])


def quat2mat(q):
    """transforms3d.quaternions.quat2mat: w-first, s = 2 / |q|^2, the identity below float64 eps."""
    w, x, y, z = q
    Nq = w * w + x * x + y * y + z * z
    if Nq < np.finfo(np.float64).eps:
        return np.eye(3)
    s = 2.0 / Nq
    X, Y, Z = x * s, y * s, z * s
    wX, wY, wZ = w * X, w * Y, w * Z
    xX, xY, xZ = x * X, x * Y, x * Z
    yY, yZ, zZ = y * Y, y * Z, z * Z
    return np.array([[1.0 - (yY + zZ), xY - wZ, xZ + wY],
                     [xY + wZ, 1.0 - (xX + zZ), yZ - wX],
                     [xZ - wY, yZ + wX, 1.0 - (xX + yY)]])


def compose(T, R, Z):
    """transforms3d.affines.compose without shears."""
    A = np.eye(4)
    A[:3, :3] = np.asarray(R) @ np.diag(Z)
    A[:3, 3] = T
    return A


def intrinsics(frames_txt_lines):
    """data_process_anno :186-190 on the file's lines (readlines(), newlines kept) -> fx, fy, cx, cy."""
    lines = [l.strip() for l in frames_txt_lines if len(l) > 0 and l[0] != '#']
    eles = [[float(e) for e in l.split(',')] for l in lines]
    data = np.array(eles)
    fx, fy, cx, cy = np.average(data, axis=0)[2:]
    return fx, fy, cx, cy


def get_bbox3d(box_lines):
    box_data = [float(e) for e in box_lines[1].strip().split(',')]
    ex, ey, ez = box_data[3:6]
    bbox_3d = np.array([[-ex, -ey, -ez], [ex, -ey, -ez], [ex, -ey, ez], [-ex, -ey, ez],
                        [-ex, ey, -ez], [ex, ey, -ez], [ex, ey, ez], [-ex, ey, ez]]) * 0.5
    return bbox_3d, np.concatenate([bbox_3d, np.ones((8, 1))], axis=1)


def parse_box(box_lines):
    data = [float(e) for e in box_lines[1].strip().split(',')]
    return compose(data[:3], quat2mat(data[6:]), np.ones(3))


def reproj(K_homo, pose, points3d_homo):
    reproj_points = K_homo @ pose @ points3d_homo
    reproj_points = reproj_points[:] / reproj_points[2:]
    return reproj_points[:2, :].T


def skipped(reproj_box3d):
    x0, y0 = reproj_box3d.min(0)
    x1, y1 = reproj_box3d.max(0)
    return bool(x0 < -1000 or y0 < -1000 or x1 > 3000 or y1 > 3000)


def process_poses(K, box_lines, arposes_lines, corners=None):
    """data_process_anno's loop (:202-238, downsample_rate 1) -> ({index: (T_oc, reproj_box3d, row)}, keep per data row), where
    row counts the data rows (comment and blank lines removed) as read_arposes does.  corners [n, 3] replaces get_bbox3d's 8
    corners in reproj and the skip rule (opb_scan_poses takes any n up to 1024)."""
    fx, fy, cx, cy = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
    _, bbox_3d_homo = get_bbox3d(box_lines)
    if corners is not None:
        bbox_3d_homo = np.concatenate([np.asarray(corners, np.float64).reshape(-1, 3), np.ones((len(corners), 1))], axis=1)
    K_homo = np.array([[fx, 0, cx, 0], [0, fy, cy, 0], [0, 0, 1, 0]])
    saved, keep = {}, []
    lines = [l.strip() for l in arposes_lines]
    index = 0
    for line in lines:
        if len(line) == 0 or line[0] == '#':
            continue
        data = [float(e) for e in line.split(',')]
        position, quaternion = data[1:4], data[4:]
        rot_mat = quat2mat(quaternion) @ FLIP
        T_ow = parse_box(box_lines)
        T_cw = compose(position, rot_mat, np.ones(3))
        T_wc = np.linalg.inv(T_cw)
        T_oc = T_wc @ T_ow
        reproj_box3d = reproj(K_homo, T_oc, bbox_3d_homo.T)
        if skipped(reproj_box3d):
            keep.append(0)
            continue
        keep.append(1)
        saved[index] = (T_oc, reproj_box3d, len(keep) - 1)
        index += 1
    return saved, np.array(keep, np.int32)


def get_affine_transform(center, scale, output_size):
    """data_utils.get_affine_transform with rot = 0, no shift."""
    src_w, dst_w, dst_h = scale[0], output_size[0], output_size[1]
    src_dir = [0, src_w * -0.5]
    dst_dir = np.array([0, dst_w * -0.5], np.float32)
    src = np.zeros((3, 2), dtype=np.float32)
    dst = np.zeros((3, 2), dtype=np.float32)
    src[0, :] = center
    src[1, :] = center + np.asarray(src_dir)
    dst[0, :] = [dst_w * 0.5, dst_h * 0.5]
    dst[1, :] = np.array([dst_w * 0.5, dst_h * 0.5], np.float32) + dst_dir
    for p in (src, dst):
        direct = p[0] - p[1]
        p[2:, :] = p[1] + np.array([-direct[1], direct[0]], dtype=np.float32)
    return cv2.getAffineTransform(np.float32(src), np.float32(dst))


def _trans(box, resize_shape):
    center = np.array([(box[0] + box[2]) / 2., (box[1] + box[3]) / 2.])
    scale = np.array([box[2] - box[0], box[3] - box[1]])
    resize_h, resize_w = resize_shape
    return get_affine_transform(center, scale, [resize_w, resize_h]), resize_w, resize_h


def get_image_crop_resize(image, box, resize_shape):
    trans_crop, w, h = _trans(box, resize_shape)
    image_crop = cv2.warpAffine(image, trans_crop, (w, h), flags=cv2.INTER_LINEAR)
    return image_crop, np.concatenate([trans_crop, np.array([[0, 0, 1]])], axis=0)


def get_K_crop_resize(box, K_orig, resize_shape):
    trans_crop, _, _ = _trans(box, resize_shape)
    trans_crop_homo = np.concatenate([trans_crop, np.array([[0, 0, 1]])], axis=0)
    K_orig_homo = np.concatenate([K_orig, np.zeros((3, 1))], axis=-1) if K_orig.shape == (3, 3) else K_orig.copy()
    K_crop_homo = trans_crop_homo @ K_orig_homo
    return K_crop_homo[:3, :3], K_crop_homo


def crop_frame(image, reproj_box3d, K, hw):
    """parse_video's body for one frame (:147-172) -> dict(box, image, K_crop, M, box_crop-less).  image is the decoded frame."""
    rb = reproj_box3d.astype(int)
    x0, y0 = rb.min(0)
    x1, y1 = rb.max(0)
    box = np.array([x0, y0, x1, y1])
    resize_shape = np.array([y1 - y0, x1 - x0])
    K_crop, K_crop_homo = get_K_crop_resize(box, K, resize_shape)
    image_crop, trans1 = get_image_crop_resize(image, box, resize_shape)
    box_new = np.array([0, 0, x1 - x0, y1 - y0])
    resize_shape = np.array([hw, hw])
    K_crop, K_crop_homo = get_K_crop_resize(box_new, K_crop, resize_shape)
    image_crop, trans2 = get_image_crop_resize(image_crop, box_new, resize_shape)
    return {"box": box, "image": image_crop, "K_crop": K_crop, "K_crop_homo": K_crop_homo, "M": np.linalg.inv(trans2 @ trans1),
            "T1": trans1[:2], "T2": trans2[:2]}


def parse_video(frames, saved, K, bbox_3d_homo, hw=512):
    """parse_video's loop over decoded frames -> list, per frame, of its outputs or None.  A box whose crop cv2 cannot make
    (an empty side) is None too; the reference stops there with an exception."""
    out = [None] * len(frames)
    index = 0
    for f, image in enumerate(frames):
        if index not in saved:
            continue
        T_oc, reproj_box3d, row = saved[index]
        rb = reproj_box3d.astype(int)
        if not (rb.max(0) > rb.min(0)).all():
            index += 1
            continue
        r = crop_frame(image, reproj_box3d, K, hw)
        reproj_crop = reproj(r["K_crop_homo"], T_oc, bbox_3d_homo.T)
        r["box_crop"] = np.concatenate([reproj_crop.min(0), reproj_crop.max(0)])
        r.update(pose=T_oc, proj=reproj_box3d, row=row, index=index)
        out[f] = r
        index += 1
    return out


def png_grey(crop_bgr):
    """The evaluation's read of a crop: cv2.imwrite then cv2.imread(IMREAD_GRAYSCALE), in memory."""
    ok, buf = cv2.imencode('.png', crop_bgr)
    assert ok
    return cv2.imdecode(buf, cv2.IMREAD_GRAYSCALE)


def colour_frame(h, w, seed, c=3):
    """A colour frame made of integers only: tests/crop_reference.py's grey frame for each channel, with its own seed."""
    from tests.crop_reference import synthetic_frame
    return np.stack([synthetic_frame(h, w, seed * 7 + k) for k in range(c)], axis=-1)
