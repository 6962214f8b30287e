"""numpy restatement of ``cv2.calcOpticalFlowPyrLK`` (OpenCV 4.13, 8-bit grey images, no flags) -- the model that
``csrc/flow.cu`` is checked against, and that ``test_lk_reference_cpu.py`` pins to live cv2.

Every step was confirmed by black-box comparison with cv2 (pyramids, derivatives, points, status and err; see the tests):

pyramid      level l+1 = cv2.pyrDown(level l): the 5x5 [1 4 6 4 1]^2 / 256 kernel, (sum + 128) >> 8, BORDER_REFLECT_101 on the
             source.  Levels stop early: after level l, if the next size ((w+1)//2, (h+1)//2) has a side <= the window's, l
             is the last level (``cv2.buildOpticalFlowPyramid``'s return value).
derivatives  Scharr on each prev level, int16 (dx, dy): [3 10 3] across, [-1 0 1] along, REFLECT_101 rows and columns.
borders      a window reads the image levels through REFLECT_101 and the derivatives through a zero border.
per point    from the coarsest level down (``_track_level``): fixed-point bilinear weights (14 bits, cvRound of fp32
             products), the window of prev and its derivatives descaled to 1/32 of a grey level and to integers, the
             structure tensor and the mismatch vector as fp32 sums in OpenCV's SIMD order (``_sum_tensor``,
             ``_sum_mismatch``: four lanes over the first 8*floor(w/8) columns of each row, the rest of each row in order into
             the scalar sum, the lanes added last as (l0 + l2) + (l1 + l3)), the minimum-eigenvalue test, Newton steps with
             OpenCV's stop rules, the guess doubled between levels.
"""
from __future__ import annotations

import numpy as np

W_BITS = 14
FLT_SCALE = np.float32(1.0 / (1 << 20))
F32 = np.float32
TERM_COUNT, TERM_EPS = 1, 2


def _reflect101(i: np.ndarray, n: int) -> np.ndarray:
    """cv::borderInterpolate(i, n, BORDER_REFLECT_101) elementwise."""
    i = np.asarray(i, dtype=np.int64).copy()
    if n == 1:
        return np.zeros_like(i)
    while True:
        lo, hi = i < 0, i >= n
        if not (lo.any() or hi.any()):
            return i
        i[lo] = -i[lo]
        i[hi] = 2 * n - 2 - i[hi]


def pyr_down(img: np.ndarray) -> np.ndarray:
    """cv2.pyrDown of a uint8 [h, w] image: [(h+1)//2, (w+1)//2]."""
    h, w = img.shape
    oh, ow = (h + 1) // 2, (w + 1) // 2
    k = np.array([1, 4, 6, 4, 1], dtype=np.int64)
    ys = _reflect101(2 * np.arange(oh)[:, None] + np.arange(-2, 3)[None], h)    # [oh, 5]
    xs = _reflect101(2 * np.arange(ow)[:, None] + np.arange(-2, 3)[None], w)    # [ow, 5]
    src = img.astype(np.int64)
    rows = (src[ys] * k[None, :, None]).sum(1)                                   # [oh, w]
    tot = (rows[:, xs] * k[None, None, :]).sum(2)                                # [oh, ow]
    return ((tot + 128) >> 8).astype(np.uint8)


def scharr(img: np.ndarray) -> np.ndarray:
    """int16 [h, w, 2] = (dx, dy) of a uint8 [h, w] image (calcScharrDeriv)."""
    h, w = img.shape
    s = img.astype(np.int64)
    ym, yp = _reflect101(np.arange(h) - 1, h), _reflect101(np.arange(h) + 1, h)
    xm, xp = _reflect101(np.arange(w) - 1, w), _reflect101(np.arange(w) + 1, w)
    t0 = (s[ym] + s[yp]) * 3 + s * 10
    t1 = s[yp] - s[ym]
    dx = t0[:, xp] - t0[:, xm]
    dy = (t1[:, xp] + t1[:, xm]) * 3 + t1 * 10
    return np.stack([dx, dy], -1).astype(np.int16)


def n_levels(h: int, w: int, win, max_level: int) -> int:
    """The last level cv2.buildOpticalFlowPyramid builds for an [h, w] image (its return value)."""
    ww, wh = win
    for level in range(max_level + 1):
        w, h = (w + 1) // 2, (h + 1) // 2
        if w <= ww or h <= wh:
            return level
    return max_level


def build_pyramid(img: np.ndarray, win, max_level: int):
    """(images, derivatives) of the levels cv2 builds: uint8 [h_l, w_l] and int16 [h_l, w_l, 2] lists."""
    last = n_levels(*img.shape, win, max_level)
    levels = [np.ascontiguousarray(img)]
    for _ in range(last):
        levels.append(pyr_down(levels[-1]))
    return levels, [scharr(x) for x in levels]


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def _weights(a: np.ndarray, b: np.ndarray):
    """cvRound of the fp32 bilinear products, the fourth weight making up 1 << 14.  a, b fp32 [n] -> int64 [n] x 4."""
    one = F32(1.0)
    s = F32(1 << W_BITS)
    w00 = np.rint((one - a) * (one - b) * s).astype(np.int64)
    w01 = np.rint(a * (one - b) * s).astype(np.int64)
    w10 = np.rint((one - a) * b * s).astype(np.int64)
    return w00, w01, w10, (1 << W_BITS) - w00 - w01 - w10


def _window(pad: np.ndarray, off, iy, ix, wh, ww, w, shift):
    """The bilinear window (int64 [n, wh, ww, ...]) at integer corners (iy, ix) of a padded plane with weights w."""
    ys = iy[:, None] + off[0] + np.arange(wh + 1)[None]
    xs = ix[:, None] + off[1] + np.arange(ww + 1)[None]
    p = pad[ys[:, :, None], xs[:, None, :]].astype(np.int64)
    ex = (slice(None),) + (None,) * (p.ndim - 1)
    v = p[:, :-1, :-1] * w[0][ex] + p[:, :-1, 1:] * w[1][ex] + p[:, 1:, :-1] * w[2][ex] + p[:, 1:, 1:] * w[3][ex]
    return _descale(v, shift)


def _sum_tensor(prod: np.ndarray) -> np.ndarray:
    """fp32 sum of int products [n, wh, ww] in the order of OpenCV's structure-tensor loop: per row, column x < 8*floor(w/8)
    into lane x % 4, the remaining columns one by one into the scalar sum."""
    n, wh, ww = prod.shape
    xa = ww // 8 * 8
    f = prod.astype(F32)
    lanes = [np.zeros(n, F32) for _ in range(4)]
    tail = np.zeros(n, F32)
    for y in range(wh):
        for x in range(xa):
            lanes[x % 4] = lanes[x % 4] + f[:, y, x]
        for x in range(xa, ww):
            tail = tail + f[:, y, x]
    return tail + ((lanes[0] + lanes[2]) + (lanes[1] + lanes[3]))


def _sum_mismatch(diff: np.ndarray, d: np.ndarray) -> np.ndarray:
    """fp32 sum of diff * d [n, wh, ww] in the order of OpenCV's mismatch loop: per row, blocks of 8 columns whose products
    k and k+4 are added as integers, then converted and added into lane k; the remaining columns one by one."""
    n, wh, ww = diff.shape
    xb = ww // 8 * 8
    p = diff * d
    lanes = [np.zeros(n, F32) for _ in range(4)]
    tail = np.zeros(n, F32)
    for y in range(wh):
        for x0 in range(0, xb, 8):
            for k in range(4):
                lanes[k] = lanes[k] + (p[:, y, x0 + k] + p[:, y, x0 + k + 4]).astype(F32)
        for x in range(xb, ww):
            tail = tail + p[:, y, x].astype(F32)
    return tail + ((lanes[0] + lanes[2]) + (lanes[1] + lanes[3]))


def _track_level(I, dI, J, win, level, top, prev_pts, next_pts, status, err, count, eps2, min_eig):
    """One level of LKTrackerInvoker for every point; updates next_pts, status and err in place."""
    ww, wh = win
    h, w = I.shape
    Ipad = np.pad(I, ((wh, wh), (ww, ww)), mode="reflect")      # numpy's "reflect" is REFLECT_101
    Jpad = np.pad(J, ((wh, wh), (ww, ww)), mode="reflect")
    dpad = np.pad(dI, ((wh, wh), (ww, ww), (0, 0)))
    off = (wh, ww)
    half = np.array([(ww - 1) * 0.5, (wh - 1) * 0.5], F32)
    n = prev_pts.shape[0]
    prev = prev_pts * F32(1.0 / (1 << level))
    nxt = prev.copy() if level == top else next_pts * F32(2.0)
    next_pts[:] = nxt
    prev = prev - half
    ip = np.floor(prev).astype(np.int64)
    live = ~((ip[:, 0] < -ww) | (ip[:, 0] >= w) | (ip[:, 1] < -wh) | (ip[:, 1] >= h))
    if level == 0:
        status[~live] = 0
        err[~live] = 0
    idx = np.nonzero(live)[0]
    if idx.size == 0:
        return
    ab = (prev[idx] - ip[idx]).astype(F32)
    wts = _weights(ab[:, 0], ab[:, 1])
    Iw = _window(Ipad, off, ip[idx, 1], ip[idx, 0], wh, ww, wts, W_BITS - 5)
    dW = _window(dpad, off, ip[idx, 1], ip[idx, 0], wh, ww, wts, W_BITS)
    ix, iy = dW[..., 0], dW[..., 1]
    A11 = _sum_tensor(ix * ix) * FLT_SCALE
    A12 = _sum_tensor(ix * iy) * FLT_SCALE
    A22 = _sum_tensor(iy * iy) * FLT_SCALE
    D = A11 * A22 - A12 * A12
    eig = ((A22 + A11) - np.sqrt((A11 - A22) * (A11 - A22) + F32(4.0) * A12 * A12)) / F32(2 * ww * wh)
    ok = ~((eig < F32(min_eig)) | (D < np.finfo(F32).eps))
    if level == 0:
        status[idx[~ok]] = 0
    idx, Iw, ix, iy, A11, A12, A22, D = idx[ok], Iw[ok], ix[ok], iy[ok], A11[ok], A12[ok], A22[ok], D[ok]
    D = F32(1.0) / D
    pt = next_pts[idx] - half
    prev_delta = np.zeros_like(pt)
    run = np.ones(idx.size, bool)
    for j in range(count):
        r = np.nonzero(run)[0]
        if r.size == 0:
            break
        ij = np.floor(pt[r]).astype(np.int64)
        out = (ij[:, 0] < -ww) | (ij[:, 0] >= w) | (ij[:, 1] < -wh) | (ij[:, 1] >= h)
        if level == 0:
            status[idx[r[out]]] = 0
        run[r[out]] = False
        r, ij = r[~out], ij[~out]
        if r.size == 0:
            break
        ab = (pt[r] - ij).astype(F32)
        Jw = _window(Jpad, off, ij[:, 1], ij[:, 0], wh, ww, _weights(ab[:, 0], ab[:, 1]), W_BITS - 5)
        diff = Jw - Iw[r]
        b1 = _sum_mismatch(diff, ix[r]) * FLT_SCALE
        b2 = _sum_mismatch(diff, iy[r]) * FLT_SCALE
        delta = np.stack([(A12[r] * b2 - A22[r] * b1) * D[r], (A12[r] * b1 - A11[r] * b2) * D[r]], 1).astype(F32)
        pt[r] = pt[r] + delta
        next_pts[idx[r]] = pt[r] + half
        d64 = delta.astype(np.float64)
        small = d64[:, 0] * d64[:, 0] + d64[:, 1] * d64[:, 1] <= eps2
        osc = np.zeros(r.size, bool)
        if j > 0:
            s = (delta + prev_delta[r]).astype(np.float64)
            osc = ~small & (np.abs(s[:, 0]) < 0.01) & (np.abs(s[:, 1]) < 0.01)
            next_pts[idx[r[osc]]] -= delta[osc] * F32(0.5)
        run[r[small | osc]] = False
        prev_delta[r] = delta
    if level == 0:
        k = idx[status[idx] == 1]
        if k.size == 0:
            return
        q = next_pts[k] - half
        iq = np.floor(q).astype(np.int64)
        out = (iq[:, 0] < -ww) | (iq[:, 0] >= w) | (iq[:, 1] < -wh) | (iq[:, 1] >= h)
        status[k[out]] = 0
        m = ~out
        k, q, iq = k[m], q[m], iq[m]
        if k.size == 0:
            return
        ab = (q - iq).astype(F32)
        Jw = _window(Jpad, off, iq[:, 1], iq[:, 0], wh, ww, _weights(ab[:, 0], ab[:, 1]), W_BITS - 5)
        rows = np.searchsorted(idx, k)
        e = np.abs(Jw - Iw[rows]).reshape(k.size, -1).sum(1)       # integers below 2^24: exact in fp32 in any order
        err[k] = e.astype(F32) / F32(32 * ww * wh)


def criteria_params(criteria):
    """(max_count, eps^2) as calcOpticalFlowPyrLK derives them from (type, count, eps)."""
    ty, count, eps = criteria
    count = min(max(int(count), 0), 100) if ty & TERM_COUNT else 30
    eps = min(max(float(eps), 0.0), 10.0) if ty & TERM_EPS else 0.01
    return count, eps * eps


def calc_optical_flow_pyr_lk(prev: np.ndarray, nxt: np.ndarray, pts: np.ndarray, win=(21, 21), max_level=3,
                             criteria=(TERM_COUNT | TERM_EPS, 30, 0.01), min_eig=1e-4):
    """(next_pts fp32 [n, 2], status uint8 [n], err fp32 [n]) as cv2.calcOpticalFlowPyrLK(prev, nxt, pts, None, ...) gives
    them for status-1 points.  For a status-0 point err is 0 (cv2 leaves it unset unless the point starts outside the image)."""
    pts = np.asarray(pts, F32).reshape(-1, 2)
    count, eps2 = criteria_params(criteria)
    P, dP = build_pyramid(prev, win, max_level)
    N, _ = build_pyramid(nxt, win, max_level)
    top = min(len(P), len(N)) - 1
    n = pts.shape[0]
    next_pts = np.zeros((n, 2), F32)
    status = np.ones(n, np.uint8)
    err = np.zeros(n, F32)
    for level in range(top, -1, -1):
        _track_level(P[level], dP[level], N[level], win, level, top, pts, next_pts, status, err, count, eps2, min_eig)
    return next_pts, status, err
