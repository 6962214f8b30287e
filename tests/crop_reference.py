"""Numpy model of the reference's pose-guided crop (local_feature_2D_detector.py:160-186, :232-259): the test oracle of
``onepose_b200/csrc/crop.cu``.  Plain numpy and Python floats (IEEE doubles, no fused multiply-add), no cv2 import.

``affine_transform`` is ``data_utils.get_affine_transform`` with ``rot = 0`` and no shift: three float32 point pairs, then
``cv2.getAffineTransform``'s 6x6 solve in fp64 by LU with partial pivoting.  ``warp_affine_u8`` is ``cv2.warpAffine(...,
INTER_LINEAR)`` on 8-bit data with a constant zero border, which is integer arithmetic throughout (DESIGN, "The crop").
Both are bit-exact against OpenCV 4.13 (tests/test_crop_reference_cpu.py)."""
import numpy as np

F32 = np.float32
AB_BITS, INTER_BITS = 10, 5
MAX_COORD, MAX_SIDE = 1 << 20, 32767     # the boxes opb_crop_resize accepts (include/onepose_b200.h)


def synthetic_frame(h, w, seed=0):
    """A grey camera frame made of integers only (the same on every platform): two triangle waves plus hashed noise."""
    y, x = np.mgrid[0:h, 0:w].astype(np.int64)
    tri = lambda v, p: np.abs((v % (2 * p)) - p) * 255 // p          # noqa: E731
    smooth = (tri(3 * x + y + 17 * seed, 97) + tri(2 * y - x + 5 * seed, 61)) // 2
    n = (x * 73856093) ^ (y * 19349663) ^ ((seed + 1) * 83492791)
    n = ((n ^ (n >> 13)) * 1274126177) & 0xFFFFFFFF
    return np.clip(smooth * 3 // 4 + ((n >> 16) & 63), 0, 255).astype(np.uint8)


def weight_table():
    """cv2's bilinear table: int16 rint(w * 32768) of the float32 products (1 - fx/32 | fx/32) * (1 - fy/32 | fy/32), each entry
    fixed up to sum to 32768.  [fy, fx, 4] in the order (y0 x0, y0 x1, y1 x0, y1 x1)."""
    t = np.zeros((32, 32, 4), np.int32)
    for fy in range(32):
        for fx in range(32):
            ax, ay = F32(fx / 32.0), F32(fy / 32.0)
            wx = np.array([F32(1) - ax, ax], F32)
            wy = np.array([F32(1) - ay, ay], F32)
            w = (wy[:, None] * wx[None, :]).astype(F32).reshape(-1)
            iw = np.clip(np.rint(w.astype(np.float64) * 32768), -32768, 32767).astype(np.int32)
            d = 32768 - int(iw.sum())
            if d:
                iw[np.argmax(iw) if d < 0 else np.argmin(iw)] += d
            t[fy, fx] = iw
    return t


def closed_form_weights(fx, fy):
    """What crop.cu computes instead of reading the table: the products are exact in float32, so every entry is an integer."""
    return np.array([32 * (32 - fx) * (32 - fy), 32 * fx * (32 - fy), 32 * (32 - fx) * fy, 32 * fx * fy], np.int32)


_TABLE = weight_table()


def _lu_solve(a, b):
    """OpenCV's LUImpl for one right-hand side: partial pivoting (first largest magnitude), d = -1 / pivot, row += alpha * pivot
    row, then back substitution."""
    m = len(b)
    a = [[float(v) for v in row] for row in a]
    b = [float(v) for v in b]
    for i in range(m):
        k = i
        for j in range(i + 1, m):
            if abs(a[j][i]) > abs(a[k][i]):
                k = j
        if abs(a[k][i]) < 2.220446049250313e-16 * 100:
            return None
        if k != i:
            a[i], a[k] = a[k], a[i]
            b[i], b[k] = b[k], b[i]
        d = -1.0 / a[i][i]
        for j in range(i + 1, m):
            alpha = a[j][i] * d
            for c in range(i + 1, m):
                a[j][c] += alpha * a[i][c]
            b[j] += alpha * b[i]
    for i in range(m - 1, -1, -1):
        s = b[i]
        for c in range(i + 1, m):
            s -= a[i][c] * b[c]
        b[i] = s / a[i][i]
    return b


def affine_transform(center, src_w, dst_w, dst_h, points=F32):
    """get_affine_transform(center, [src_w, .], 0, [dst_w, dst_h]) -> 2x3 f64.  Both axes scale by dst_w / src_w.  ``points``
    is the dtype of the three point pairs (float32 in the reference; float64 only as a planted variant)."""
    src = np.zeros((3, 2), points)
    dst = np.zeros((3, 2), points)
    center = np.asarray(center, np.float64)
    src[0] = center
    src[1] = center + np.array([0.0, float(src_w) * -0.5])
    dst[0] = [dst_w * 0.5, dst_h * 0.5]
    dst[1] = np.array([dst_w * 0.5, dst_h * 0.5], points) + np.array([0, dst_w * -0.5], points)
    for p in (src, dst):
        direct = p[0] - p[1]
        p[2] = p[1] + np.array([-direct[1], direct[0]], points)
    a = np.zeros((6, 6))
    b = np.zeros(6)
    for i in range(3):
        a[2 * i, 0:3] = [src[i, 0], src[i, 1], 1]
        a[2 * i + 1, 3:6] = [src[i, 0], src[i, 1], 1]
        b[2 * i], b[2 * i + 1] = dst[i]
    x = _lu_solve(a, b)
    if x is None:
        return np.zeros((2, 3))
    return np.array(x).reshape(2, 3)


def box_transform(box, out_h, out_w, points=F32):
    """The transform both get_image_crop_resize and get_K_crop_resize build for (box, [out_h, out_w])."""
    x0, y0, x1, y1 = (int(v) for v in box)
    return affine_transform([(x0 + x1) / 2.0, (y0 + y1) / 2.0], x1 - x0, out_w, out_h, points)


def _rint(v):
    return np.rint(v).astype(np.int64)


def warp_affine_u8(img, M, w, h):
    """cv2.warpAffine(img, M, (w, h), flags=INTER_LINEAR) for uint8 [H, W], constant zero border."""
    M = np.asarray(M, np.float64).reshape(-1).copy()
    D = M[0] * M[4] - M[1] * M[3]
    D = 1.0 / D if D != 0 else 0.0
    A11, A22 = M[4] * D, M[0] * D
    M[0], M[4] = A11, A22
    M[1] *= -D
    M[3] *= -D
    b1 = -M[0] * M[2] - M[1] * M[5]
    b2 = -M[3] * M[2] - M[4] * M[5]
    M[2], M[5] = b1, b2
    x = np.arange(w, dtype=np.float64)
    y = np.arange(h, dtype=np.float64)
    scale = float(1 << AB_BITS)
    half = (1 << AB_BITS) // (1 << INTER_BITS) // 2
    ad, bd = _rint(M[0] * x * scale), _rint(M[3] * x * scale)
    X0 = _rint((M[1] * y + M[2]) * scale) + half
    Y0 = _rint((M[4] * y + M[5]) * scale) + half
    X = (X0[:, None] + ad[None, :]) >> (AB_BITS - INTER_BITS)
    Y = (Y0[:, None] + bd[None, :]) >> (AB_BITS - INTER_BITS)
    sx = np.clip(X >> INTER_BITS, -32768, 32767)
    sy = np.clip(Y >> INTER_BITS, -32768, 32767)
    H, W = img.shape

    def px(yy, xx):
        ok = (yy >= 0) & (yy < H) & (xx >= 0) & (xx < W)
        return np.where(ok, img[np.clip(yy, 0, H - 1), np.clip(xx, 0, W - 1)].astype(np.int64), 0)

    wt = _TABLE[Y & 31, X & 31]
    s = px(sy, sx) * wt[..., 0] + px(sy, sx + 1) * wt[..., 1] + px(sy + 1, sx) * wt[..., 2] + px(sy + 1, sx + 1) * wt[..., 3]
    return np.clip((s + (1 << 14)) >> 15, 0, 255).astype(np.uint8)


def get_image_crop_resize(image, box, resize_shape):
    h, w = (int(v) for v in resize_shape)
    T = box_transform(box, h, w)
    return warp_affine_u8(image, T, w, h), np.concatenate([T, [[0.0, 0.0, 1.0]]], axis=0)


def get_K_crop_resize(box, K, resize_shape):
    h, w = (int(v) for v in resize_shape)
    T = np.concatenate([box_transform(box, h, w), [[0.0, 0.0, 1.0]]], axis=0)
    K_homo = T @ np.concatenate([np.asarray(K, np.float64), np.zeros((3, 1))], axis=1)
    return K_homo[:3, :3], K_homo


def box_ok(box):
    x0, y0, x1, y1 = (int(v) for v in box)
    return 0 < x1 - x0 <= MAX_SIDE and 0 < y1 - y0 <= MAX_SIDE and max(abs(x0), abs(y0), abs(x1), abs(y1)) <= MAX_COORD


def crop_img_by_bbox(image, box, K, crop_size):
    """The body of crop_img_by_bbox -> (stage-1 image, stage-2 image, T1, T2, K_crop)."""
    x0, y0, x1, y1 = (int(v) for v in box)
    K1, _ = get_K_crop_resize(box, K, [y1 - y0, x1 - x0])
    im1, T1 = get_image_crop_resize(image, box, [y1 - y0, x1 - x0])
    box2 = [0, 0, x1 - x0, y1 - y0]
    K2, _ = get_K_crop_resize(box2, K1, [crop_size, crop_size])
    im2, T2 = get_image_crop_resize(im1, box2, [crop_size, crop_size])
    return im1, im2, T1[:2], T2[:2], K2


# ---- the same warps per output pixel: for outputs and boxes too large for the array model ----

# Planted slips, one per part of the fixed-point warp; ``variant=`` in the functions below.  The suite requires that each one
# changes a pixel or a transform of sweep_cases(), or that it cannot change any (tests/test_crop_reference_cpu.py).
VARIANTS = ("tie_floor",          # round-half-even replaced by floor on the ties (__double2ll_rn -> _rd where it matters)
            "no_round_delta",     # X0, Y0 without the + 16
            "table_unfixed",      # cv2's table without its fx = fy = 0 fix-up: (32767, 0, 0, 0)
            "no_saturation",      # sx, sy not saturated to int16
            "f64_points",         # get_affine_transform's point pairs in float64 instead of float32
            "stage1_unrounded")   # stage 1 not rounded to uint8 before stage 2

_TABLE_UNFIXED = _TABLE.copy()
_TABLE_UNFIXED[0, 0] = (32767, 0, 0, 0)


def _round(v, variant):
    r = np.rint(v)
    if variant == "tie_floor":
        r = np.where(v - np.floor(v) == 0.5, np.floor(v), r)
    return r.astype(np.int64)


def inverse_transform(M):
    """warpAffine's inversion of the forward 2x3 matrix M: m maps an output pixel to its source position."""
    M = [float(v) for v in np.asarray(M, np.float64).reshape(-1)]
    D = M[0] * M[4] - M[1] * M[3]
    D = 1.0 / D if D != 0 else 0.0
    m = [M[4] * D, M[1] * -D, 0.0, M[3] * -D, M[0] * D, 0.0]
    m[2] = -m[0] * M[2] - m[1] * M[5]
    m[5] = -m[3] * M[2] - m[4] * M[5]
    return m


def fixed_point_terms(m, xs, ys, variant=None):
    """The four rounded terms of warpAffine's 1/1024 source coordinates: adelta(x), bdelta(x), X0(y), Y0(y) (before the round
    delta), and the unrounded values they come from."""
    xs, ys = np.asarray(xs, np.float64), np.asarray(ys, np.float64)
    raw = ((m[0] * xs) * 1024.0, (m[3] * xs) * 1024.0, (m[1] * ys + m[2]) * 1024.0, (m[4] * ys + m[5]) * 1024.0)
    return tuple(_round(v, variant) for v in raw), raw


def _warp_at(src, sw, sh, m, xs, ys, variant, rounded=True):
    """Warped pixels at integer positions (xs, ys), int64: src is an image, or src(u, v) gives the source's pixels at in-range
    positions.  rounded=False returns the exact weighted sums / 32768 instead (the stage1_unrounded variant's first stage)."""
    (ad, bd, X0, Y0), _ = fixed_point_terms(m, xs, ys, variant)
    half = 0 if variant == "no_round_delta" else (1 << AB_BITS) // (1 << INTER_BITS) // 2
    X = (X0 + half + ad) >> (AB_BITS - INTER_BITS)
    Y = (Y0 + half + bd) >> (AB_BITS - INTER_BITS)
    sx, sy = X >> INTER_BITS, Y >> INTER_BITS
    if variant != "no_saturation":
        sx, sy = np.clip(sx, -32768, 32767), np.clip(sy, -32768, 32767)
    wt = (_TABLE_UNFIXED if variant == "table_unfixed" else _TABLE)[Y & 31, X & 31]
    acc = np.zeros(sx.shape, np.float64 if variant == "stage1_unrounded" or not rounded else np.int64)
    for k, (dx, dy) in enumerate(((0, 0), (1, 0), (0, 1), (1, 1))):
        u, v = sx + dx, sy + dy
        ok = (u >= 0) & (u < sw) & (v >= 0) & (v < sh)
        acc[ok] += (src(u[ok], v[ok]) if callable(src) else src[v[ok], u[ok]]) * wt[ok, k]
    if not rounded:
        return acc / (1 << 15)
    if acc.dtype == np.float64:
        return np.clip(np.floor((acc + (1 << 14)) / (1 << 15)), 0, 255).astype(np.int64)
    return np.clip((acc + (1 << 14)) >> 15, 0, 255)


def warp_pixels(img, M, xs, ys, variant=None):
    """cv2.warpAffine(img, M, ..., INTER_LINEAR) at output positions (xs, ys) only: uint8, the shape of xs.  img uint8 [H, W]."""
    img = np.asarray(img)
    xs, ys = np.broadcast_arrays(np.asarray(xs, np.int64), np.asarray(ys, np.int64))
    return _warp_at(img, img.shape[1], img.shape[0], inverse_transform(M), xs, ys, variant).astype(np.uint8)


def crop_transforms(box, S, variant=None):
    """crop_img_by_bbox's T1 (box -> its own size) and T2 (its own size -> S x S), 2x3 each."""
    x0, y0, x1, y1 = (int(v) for v in box)
    pts = np.float64 if variant == "f64_points" else F32
    return box_transform(box, y1 - y0, x1 - x0, pts), box_transform([0, 0, x1 - x0, y1 - y0], S, S, pts)


def crop_pixels(frame, box, S, xs, ys, variant=None, chunk=1 << 20):
    """crop_img_by_bbox's stage-2 pixels at output positions (xs, ys), uint8 of the shape of xs: each needs four stage-1
    pixels, each of them the warp of the frame rounded to uint8 -- the integer steps of ``warp_affine_u8``, without building the
    stage-1 image (which has the box's size)."""
    frame = np.asarray(frame)
    x0, y0, x1, y1 = (int(v) for v in box)
    T1, T2 = crop_transforms(box, S, variant)
    m1, m2 = inverse_transform(T1), inverse_transform(T2)
    H, W = frame.shape
    unrounded = variant == "stage1_unrounded"
    stage1 = lambda u, v: _warp_at(frame, W, H, m1, u, v, None if unrounded else variant, rounded=not unrounded)  # noqa: E731
    xs, ys = np.broadcast_arrays(np.asarray(xs, np.int64), np.asarray(ys, np.int64))
    fx, fy = xs.reshape(-1), ys.reshape(-1)
    out = np.empty(fx.shape, np.uint8)
    for s in range(0, len(fx), chunk):
        out[s:s + chunk] = _warp_at(stage1, x1 - x0, y1 - y0, m2, fx[s:s + chunk], fy[s:s + chunk], variant)
    return out.reshape(xs.shape)


# The GPU sweep's boxes (tests/test_crop_domain_gpu.py), defined once so that the CPU suite can show what they catch: boxes
# inside, crossing, outside and larger than each frame, sides 1 .. 1200 (log-uniform), S = 8 .. 512 in steps of 8.  No
# rounding tie occurs at S <= 512: with rot = 0 the inverse maps are x * w / S and y * w / S + (h - w) / 2 in stage 2 and
# integer shifts in stage 1, so adelta and Y0 meet ties only where S has a factor 2048.  Two 2048 crops of small boxes
# close the list for that reason.
SWEEP_FRAMES = ((1, 1), (1, 640), (480, 1), (37, 53), (480, 640), (1440, 1920))
SWEEP_TIE_CASES = ((4, (300, 200, 301, 201), 2048), (3, (-1, 30, 2, 35), 2048))


def sweep_cases(n=1000, seed=2026):
    """-> list of (frame index into SWEEP_FRAMES, box int32 [4], S, K f64 [3, 3]): n random boxes, then SWEEP_TIE_CASES."""
    rng = np.random.default_rng(seed)
    cases = []

    def extent(size):
        kind = rng.integers(4)
        side = int(np.exp(rng.uniform(0, np.log(1201))))
        if kind == 0:                                            # inside where the frame allows it, else crossing
            lo = int(rng.integers(0, max(size - side, 0) + 1)) if side <= size else int(rng.integers(size - side, 1))
        elif kind == 1:                                          # crossing an edge
            lo = int(rng.integers(-side + 1, size))
        elif kind == 2:                                          # wholly outside, before or after
            lo = int(rng.integers(-side - 400, -side + 1)) if rng.random() < 0.5 else int(rng.integers(size, size + 400))
        else:                                                    # larger than the frame, covering it
            side = size + int(rng.integers(1, 1201))
            lo = int(rng.integers(size - side, 1))
        return lo, lo + side

    for i in range(n):
        f = i % len(SWEEP_FRAMES)
        H, W = SWEEP_FRAMES[f]
        (x0, x1), (y0, y1) = extent(W), extent(H)
        S = 8 * int(rng.integers(1, 65))
        fo = rng.uniform(300, 1500)
        K = np.array([[fo, 0, rng.uniform(0, W)], [0, fo * rng.uniform(0.9, 1.1), rng.uniform(0, H)], [0, 0, 1]])
        cases.append((f, np.array([x0, y0, x1, y1], np.int32), S, K))
    for f, box, S in SWEEP_TIE_CASES:
        cases.append((f, np.array(box, np.int32), S, np.array([[500.0, 0, 20.5], [0, 505.0, 16.25], [0, 0, 1]])))
    return cases


def reproj(K, pose, pts_3d):
    """vis_utils.reproj: K [3,3], pose [3,4] or [4,4], pts [n,3] -> [n,2]."""
    K_homo = np.concatenate([np.asarray(K, np.float64), np.zeros((3, 1))], axis=1)
    pose = np.asarray(pose, np.float64)
    if pose.shape == (3, 4):
        pose = np.concatenate([pose, [[0.0, 0.0, 0.0, 1.0]]], axis=0)
    pts = np.asarray(pts_3d, np.float64).reshape(-1, 3)
    p = K_homo @ pose @ np.concatenate([pts, np.ones((len(pts), 1))], axis=1).T
    return (p / p[2:])[:2].T


def box_from_pose(K, pose, corners):
    """previous_pose_detect's box: min / max of the projected corners, truncated towards zero; the empty box where numpy's cast
    is undefined (a non-finite value or one outside int32)."""
    p = reproj(K, pose, corners)
    v = np.concatenate([p.min(axis=0), p.max(axis=0)])
    if not np.all(np.isfinite(v)) or np.any(v <= -2147483649.0) or np.any(v >= 2147483648.0):
        return np.zeros(4, np.int32)
    return np.trunc(v).astype(np.int32)
