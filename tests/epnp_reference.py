"""fp64 numpy EPnP (Lepetit, Moreno-Noguer, Fua, "EPnP: An Accurate O(n) Solution to the PnP Problem", IJCV 2009) and the
five-index sampler of csrc/pnp_ransac.cu's EPnP-RANSAC -- test infrastructure, not product code.

Every stage is a function of its own, so that a test can look at any of them:
- ``control_points``  centroid c0 plus the principal axes of the point set scaled by sqrt(lambda / n) (largest first), each
                      with its largest-magnitude component positive; a planar set's flat axis gets the first axis's length;
- ``alphas``          barycentric coordinates of every point in the four control points (they sum to 1);
- ``mtm``             M^T M of the 2n x 12 projection system M x = 0, x = the control points' camera coordinates;
- ``null_vectors``    the eigenvectors of M^T M for its 4 smallest eigenvalues (ascending), with the eigenvalues;
- ``l6x10`` / ``rho`` the distance constraints |c_a - c_b|^2 in the betas (six pairs, ten products) and their world values;
- ``betas_approx``    the linearised solutions for N = 1, 2, 3 null vectors; ``gauss_newton`` refines all four betas;
- ``pose_from_betas`` camera coordinates of the points (depth sign made positive), then R, t by absolute orientation (SVD);
- ``epnp``            all of the above; the candidate with the lowest mean reprojection error wins, the first one on ties.
The device code takes different routes where it can (Jacobi eigen-solvers, Householder least squares, Horn's quaternion for
the rotation, sums over the control points instead of the points), so agreement is a check of both.
"""
from __future__ import annotations

import numpy as np

from tests.pnp_reference import MASK64, mix64

PAIRS = ((0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3))
GN_ITERS = 5


def sample_indices5(seed: int, b: int, h: int, n: int):
    """The five distinct correspondence indices hypothesis h of frame b draws from a frame of n >= 5 points: the k-th draw is
    taken modulo n - k from the next splitmix64 state and shifted past every earlier index, in ascending order of those."""
    r = mix64((seed & MASK64) ^ (b << 40) ^ h)
    idx = [r % n]
    for k in range(1, 5):
        r = mix64(r)
        v = r % (n - k)
        for e in sorted(idx):
            if v >= e:
                v += 1
        idx.append(v)
    return tuple(idx)


FLAT = 1e-10          # an axis whose eigenvalue is below this fraction of the largest is flat


def axis_sign(v):
    """The sign that makes the largest-magnitude component of v positive (the first such component on ties)."""
    return -1.0 if v[int(np.argmax(np.abs(v)))] < 0 else 1.0


def control_points(Pw, signs=None):
    """(cw [4,3], planar).  Axes in descending eigenvalue order, each with ``axis_sign``'s sign (or ``signs[k]`` times it:
    the eight choices are all valid EPnPs that differ on noisy data); a flat third axis gets the first axis's length.
    None for coincident or collinear points."""
    Pw = np.asarray(Pw, np.float64)
    n = len(Pw)
    c0 = Pw.mean(0)
    D = Pw - c0
    lam, V = np.linalg.eigh(D.T @ D)
    order = np.argsort(lam)[::-1]
    lam, V = lam[order], V[:, order]
    if not (lam[0] > 0 and lam[1] > FLAT * lam[0]):
        return None, False
    planar = not lam[2] > FLAT * lam[0]
    cw = np.empty((4, 3))
    cw[0] = c0
    for k in range(3):
        s = axis_sign(V[:, k]) * (1.0 if signs is None else signs[k])
        lk = lam[0] if (k == 2 and planar) else lam[k]
        cw[k + 1] = c0 + s * np.sqrt(lk / n) * V[:, k]
    return cw, planar


def alphas(Pw, cw):
    """The axes are orthogonal, so the inverse is the projection on each axis over its squared length."""
    D = np.asarray(Pw, np.float64) - cw[0]
    a = np.stack([D @ (cw[k + 1] - cw[0]) / np.sum((cw[k + 1] - cw[0]) ** 2) for k in range(3)], 1)
    return np.concatenate([1.0 - a.sum(1, keepdims=True), a], 1)


def m_matrix(K, uv, al):
    fu, fv, uc, vc = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
    n = len(uv)
    M = np.zeros((2 * n, 12))
    for j in range(4):
        M[0::2, 3 * j] = al[:, j] * fu
        M[0::2, 3 * j + 2] = al[:, j] * (uc - uv[:, 0])
        M[1::2, 3 * j + 1] = al[:, j] * fv
        M[1::2, 3 * j + 2] = al[:, j] * (vc - uv[:, 1])
    return M


def mtm(K, uv, al):
    M = m_matrix(K, np.asarray(uv, np.float64), al)
    return M.T @ M


def null_vectors(MtM, planar=False):
    """(eigenvalues [4], vectors [4,12]) for the four smallest eigenvalues, ascending.  For a planar set three of them live on
    the flat axis's control point (its columns are (near) zero) and tie with the true one: the four are then ordered by their
    weight on those columns (stable), the least first."""
    lam, V = np.linalg.eigh(MtM)
    lam, v = lam[:4], V[:, :4].T
    if planar:
        o = np.argsort(np.sum(v[:, 9:] ** 2, 1), kind="stable")
        lam, v = lam[o], v[o]
    return lam, v


def l6x10(v):
    """v [4,12] null vectors -> L [6,10]: |sum_k beta_k dv_k|^2 = L . (b00, b01, b11, b02, b12, b22, b03, b13, b23, b33)."""
    L = np.empty((6, 10))
    for r, (a, b) in enumerate(PAIRS):
        dv = [v[k].reshape(4, 3)[a] - v[k].reshape(4, 3)[b] for k in range(4)]
        L[r] = [dv[0] @ dv[0], 2 * dv[0] @ dv[1], dv[1] @ dv[1], 2 * dv[0] @ dv[2], 2 * dv[1] @ dv[2], dv[2] @ dv[2],
                2 * dv[0] @ dv[3], 2 * dv[1] @ dv[3], 2 * dv[2] @ dv[3], dv[3] @ dv[3]]
    return L


def rho(cw):
    return np.array([np.sum((cw[a] - cw[b]) ** 2) for a, b in PAIRS])


def _products(be):
    b0, b1, b2, b3 = be
    return np.array([b0 * b0, b0 * b1, b1 * b1, b0 * b2, b1 * b2, b2 * b2, b0 * b3, b1 * b3, b2 * b3, b3 * b3])


def betas_approx(L, rh):
    """Initial betas of the N = 1, 2, 3 candidates (each a length-4 array)."""
    out = []
    x = np.linalg.lstsq(L[:, [0, 1, 3, 6]], rh, rcond=None)[0]          # b00 b01 b02 b03
    b0 = np.sqrt(abs(x[0]))                                             # the sign of b00 is the quadratic form's
    sg = 1.0 if x[0] >= 0 else -1.0
    out.append(np.array([b0, sg * x[1] / b0, sg * x[2] / b0, sg * x[3] / b0]))
    x = np.linalg.lstsq(L[:, [0, 1, 2]], rh, rcond=None)[0]             # b00 b01 b11
    out.append(_two(x[0], x[1], x[2]) + [0.0, 0.0])
    x = np.linalg.lstsq(L[:, [0, 1, 2, 3, 4]], rh, rcond=None)[0]       # b00 b01 b11 b02 b12
    b = _two(x[0], x[1], x[2])
    out.append(b + [x[3] / b[0] if b[0] != 0 else 0.0, 0.0])
    return [np.array(o, np.float64) for o in out]


def _two(b00, b01, b11):
    """beta0, beta1 from the linearised b00, b01, b11 (the sign of b00 taken as the overall sign of the quadratic form)."""
    if b00 < 0:
        b0, b1 = np.sqrt(-b00), (np.sqrt(-b11) if b11 < 0 else 0.0)
    else:
        b0, b1 = np.sqrt(b00), (np.sqrt(b11) if b11 > 0 else 0.0)
    if b01 < 0:
        b0 = -b0
    return [b0, b1]


def gauss_newton(L, rh, be, iters=GN_ITERS):
    be = np.array(be, np.float64)
    for _ in range(iters):
        b0, b1, b2, b3 = be
        J = np.stack([2 * L[:, 0] * b0 + L[:, 1] * b1 + L[:, 3] * b2 + L[:, 6] * b3,
                      L[:, 1] * b0 + 2 * L[:, 2] * b1 + L[:, 4] * b2 + L[:, 7] * b3,
                      L[:, 3] * b0 + L[:, 4] * b1 + 2 * L[:, 5] * b2 + L[:, 8] * b3,
                      L[:, 6] * b0 + L[:, 7] * b1 + L[:, 8] * b2 + 2 * L[:, 9] * b3], 1)
        r = rh - L @ _products(be)
        be = be + np.linalg.lstsq(J, r, rcond=None)[0]
    return be


def pose_from_betas(v, be, al, Pw):
    cc = sum(be[k] * v[k] for k in range(4)).reshape(4, 3)
    pc = al @ cc
    if pc[:, 2].sum() < 0:
        pc = -pc
    Pw = np.asarray(Pw, np.float64)
    pm, xm = Pw.mean(0), pc.mean(0)
    H = (Pw - pm).T @ (pc - xm)
    U, _, Vt = np.linalg.svd(H)
    D = np.diag([1.0, 1.0, np.sign(np.linalg.det(Vt.T @ U.T))])
    R = Vt.T @ D @ U.T
    return R, xm - R @ pm


def mean_reprojection_error(K, uv, Pw, R, t):
    X = np.asarray(Pw, np.float64) @ R.T + t
    du = K[0, 0] * X[:, 0] / X[:, 2] + K[0, 2] - uv[:, 0]
    dv = K[1, 1] * X[:, 1] / X[:, 2] + K[1, 2] - uv[:, 1]
    return float(np.mean(np.sqrt(du * du + dv * dv)))


def epnp(K, uv, Pw, signs=None):
    """Every stage of EPnP on one point set: a dict with cw, planar, alphas, MtM, null_values, v, L, rho, betas0 / betas
    (before and after Gauss-Newton, N = 1, 2, 3), candidates [(R, t)], errors [3], best (0-based candidate), R, t, pose [3,4].
    ``signs`` flips control-point axes (see ``control_points``).  None for coincident or collinear points."""
    K = np.asarray(K, np.float64)
    uv = np.asarray(uv, np.float64).reshape(-1, 2)
    Pw = np.asarray(Pw, np.float64).reshape(-1, 3)
    cw, planar = control_points(Pw, signs)
    if cw is None:
        return None
    al = alphas(Pw, cw)
    A = mtm(K, uv, al)
    lam, v = null_vectors(A, planar)
    L = l6x10(v)
    rh = rho(cw)
    b0 = betas_approx(L, rh)
    bs = [gauss_newton(L, rh, b) for b in b0]
    cands = [pose_from_betas(v, b, al, Pw) for b in bs]
    errs = [mean_reprojection_error(K, uv, Pw, R, t) for R, t in cands]
    best = 0
    for c in (1, 2):
        if errs[c] < errs[best]:
            best = c
    R, t = cands[best]
    return {"cw": cw, "planar": planar, "alphas": al, "MtM": A, "null_values": lam, "v": v, "L": L, "rho": rh, "betas0": b0, "betas": bs,
            "candidates": cands, "errors": errs, "best": best, "R": R, "t": t, "pose": np.concatenate([R, t[:, None]], 1)}


def count_inliers(pose, K, uv, Pw, thr):
    """OpenCV's RANSAC inlier rule in fp64: squared reprojection error <= thr^2, no depth test.  Returns (inlier bool [n],
    border bool [n]: within 1e-6 px^2 of thr^2, where rounding may put a point on either side)."""
    pose = np.asarray(pose, np.float64)
    X = np.asarray(Pw, np.float64) @ pose[:, :3].T + pose[:, 3]
    with np.errstate(divide="ignore", invalid="ignore"):
        du = K[0, 0] * X[:, 0] / X[:, 2] + K[0, 2] - uv[:, 0]
        dv = K[1, 1] * X[:, 1] / X[:, 2] + K[1, 2] - uv[:, 1]
        e2 = du * du + dv * dv
    thr2 = thr * thr
    return e2 <= thr2, np.abs(e2 - thr2) <= 1e-6


def round_f32(x):
    return np.asarray(x, np.float64).astype(np.float32).astype(np.float64)
