"""CPU references for the stages of csrc/pnp_ransac.cu -- test infrastructure, not product code.

- ``sample_indices``  the kernel's minimal-sample draw (splitmix64, three distinct indices), in exact Python integers;
- ``p3p_all``          every real P3P solution of three points, by a route of its own: a resultant eliminates the depth ratio
                       y = s2/s0 from two law-of-cosines equations and leaves a quartic in x = s1/s0 (the kernel's Grunert
                       quartic is in s2/s0 and back-substitutes linearly); s2 comes from the quadratic of the b^2 equation,
                       the c^2 equation's root that satisfies the a^2 equation is kept, and every solution is polished by
                       Newton on the three distance equations in long double.  The three choices of base point are all
                       solved and merged, so a root that one elimination renders badly is found by another;
- ``classify``         the fp64 inlier test (z > 1e-9, squared reprojection error < thr^2) plus a mask of points within 1e-6
                       px^2 of the threshold, where rounding may put them on either side;
- ``refine_lsq``       scipy's Levenberg-Marquardt on the reprojection error of a given point set, from a given pose.
"""
from __future__ import annotations

import numpy as np

MASK64 = (1 << 64) - 1
BORDER_PX2 = 1e-6


def mix64(z: int) -> int:
    """splitmix64 finaliser, as the kernel's mix64."""
    z = (z + 0x9E3779B97F4A7C15) & MASK64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & MASK64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & MASK64
    return z ^ (z >> 31)


def sample_indices(seed: int, b: int, h: int, n: int):
    """The three distinct correspondence indices hypothesis h of frame b draws from a frame of n >= 3 points."""
    r = mix64((seed & MASK64) ^ (b << 40) ^ h)
    i0 = r % n
    r = mix64(r)
    i1 = r % (n - 1)
    if i1 >= i0:
        i1 += 1
    r = mix64(r)
    i2 = r % (n - 2)
    lo, hi = min(i0, i1), max(i0, i1)
    if i2 >= lo:
        i2 += 1
    if i2 >= hi:
        i2 += 1
    return i0, i1, i2


def bearings(K, pts2d):
    """Unit viewing rays of pixels, computed as the kernel does: ((u - cx) / fx, (v - cy) / fy, 1) normalised."""
    pts2d = np.asarray(pts2d, np.float64).reshape(-1, 2)
    j = np.stack([(pts2d[:, 0] - K[0, 2]) / K[0, 0], (pts2d[:, 1] - K[1, 2]) / K[1, 1], np.ones(len(pts2d))], 1)
    return j / np.linalg.norm(j, axis=1, keepdims=True)


def _sides_and_cosines(P, j):
    a2 = np.sum((P[1] - P[2]) ** 2)
    b2 = np.sum((P[0] - P[2]) ** 2)
    c2 = np.sum((P[0] - P[1]) ** 2)
    return a2, b2, c2, float(j[1] @ j[2]), float(j[0] @ j[2]), float(j[0] @ j[1])


def distance_residuals(s, a2, b2, c2, ca, cb, cg):
    s0, s1, s2 = s
    return np.array([s1 * s1 + s2 * s2 - 2 * s1 * s2 * ca - a2, s0 * s0 + s2 * s2 - 2 * s0 * s2 * cb - b2,
                     s0 * s0 + s1 * s1 - 2 * s0 * s1 * cg - c2])


def distance_jacobian(s, ca, cb, cg):
    """d(residuals)/d(s0, s1, s2) of the a^2, b^2, c^2 equations."""
    s0, s1, s2 = s
    z = 0 * s0
    return np.array([[z, 2 * (s1 - s2 * ca), 2 * (s2 - s1 * ca)],
                     [2 * (s0 - s2 * cb), z, 2 * (s2 - s0 * cb)],
                     [2 * (s0 - s1 * cg), 2 * (s1 - s0 * cg), z]])


def _solve3(A, r):
    """Cramer's rule, so that long double stays long double."""
    def det(M):
        return (M[0][0] * (M[1][1] * M[2][2] - M[1][2] * M[2][1]) - M[0][1] * (M[1][0] * M[2][2] - M[1][2] * M[2][0])
                + M[0][2] * (M[1][0] * M[2][1] - M[1][1] * M[2][0]))
    d = det(A)
    if d == 0:
        return None
    out = []
    for c in range(3):
        M = [[r[i] if k == c else A[i][k] for k in range(3)] for i in range(3)]
        out.append(det(M) / d)
    return np.array(out, dtype=A.dtype)


def _polish(s, a2, b2, c2, ca, cb, cg, iters=20):
    L = np.longdouble
    s = np.array(s, dtype=L)
    a2, b2, c2, ca, cb, cg = (L(v) for v in (a2, b2, c2, ca, cb, cg))
    for _ in range(iters):
        step = _solve3(distance_jacobian(s, ca, cb, cg).astype(L), distance_residuals(s, a2, b2, c2, ca, cb, cg))
        if step is None or not np.all(np.isfinite(step)):
            break
        s = s - step
    return s


def _depth_candidates(a2, b2, c2, ca, cb, cg):
    """Depth triples (s0, s1, s2) from the quartic in x = s1/s0; unpolished, possibly spurious."""
    P = np.polynomial.Polynomial
    q = P([1.0, -2.0 * cg, 1.0])                        # 1 + x^2 - 2 x cg
    # E1 = b2 q(x) - c2 (1 + y^2 - 2 y cb),  E2 = a2 q(x) - c2 (x^2 + y^2 - 2 x y ca): quadratics in y
    A1, B1, C1 = P([-c2]), P([2.0 * c2 * cb]), b2 * q - c2
    A2, B2, C2 = P([-c2]), P([0.0, 2.0 * c2 * ca]), a2 * q - P([0.0, 0.0, c2])
    res = (A1 * C2 - A2 * C1) ** 2 - (A1 * B2 - A2 * B1) * (B1 * C2 - B2 * C1)
    coef = res.coef
    if not np.any(np.abs(coef) > 0):
        return []
    roots = np.roots(coef[::-1])
    out = []
    for x in roots:
        if abs(x.imag) > 1e-4 * max(1.0, abs(x.real)):      # near-double roots come back as close complex pairs
            continue
        x = x.real
        den = 1 + x * x - 2 * x * cg
        if not (x > 0 and den > 0):
            continue
        s0 = np.sqrt(c2 / den)
        s1 = x * s0
        disc = s0 * s0 * (cb * cb - 1) + b2               # s2^2 - 2 s0 cb s2 + s0^2 - b2 = 0
        if disc < 0:
            if disc < -1e-6 * b2:
                continue
            disc = 0.0
        for s2 in (s0 * cb + np.sqrt(disc), s0 * cb - np.sqrt(disc)):
            if s2 > 0 and abs(s1 * s1 + s2 * s2 - 2 * s1 * s2 * ca - a2) <= 1e-3 * a2:
                out.append((s0, s1, s2))
    return out


def _pose_from_points(P, X):
    """R, t with X = R P + t for three exact correspondences (Kabsch; the reflection is excluded)."""
    pm, xm = P.mean(0), X.mean(0)
    H = (P - pm).T @ (X - xm)
    U, _, Vt = np.linalg.svd(H)
    D = np.diag([1.0, 1.0, np.sign(np.linalg.det(Vt.T @ U.T))])
    R = Vt.T @ D @ U.T
    return R, xm - R @ pm


def p3p_all(P, j):
    """Every real P3P solution of world points P [3,3] seen along unit bearings j [3,3] (camera frame).  Returns a list of
    dicts {R [3,3], t [3], depths [3], cond}: cond is the condition number of the distance equations' Jacobian at the
    solution (the sensitivity of the depths to the data)."""
    P = np.asarray(P, np.float64)
    j = np.asarray(j, np.float64)
    a2, b2, c2, ca, cb, cg = _sides_and_cosines(P, j)
    if not (a2 > 0 and b2 > 0 and c2 > 0) or np.linalg.norm(np.cross(P[1] - P[0], P[2] - P[0])) <= 1e-12 * max(a2, b2, c2):
        return []
    sols = []
    for perm in ((0, 1, 2), (1, 2, 0), (2, 0, 1)):        # each point as the base of the depth ratios
        pa2, pb2, pc2, pca, pcb, pcg = _sides_and_cosines(P[list(perm)], j[list(perm)])
        for d in _depth_candidates(pa2, pb2, pc2, pca, pcb, pcg):
            s = np.empty(3)
            s[list(perm)] = d
            s = _polish(s, a2, b2, c2, ca, cb, cg)
            r = distance_residuals(s, np.longdouble(a2), np.longdouble(b2), np.longdouble(c2), np.longdouble(ca),
                                   np.longdouble(cb), np.longdouble(cg))
            scale = max(a2, b2, c2)
            if not (np.all(s > 0) and np.all(np.abs(r) <= 1e-12 * scale)):
                continue
            s64 = s.astype(np.float64)
            if any(np.max(np.abs(s64 - o["depths"])) <= 1e-9 * np.max(s64) for o in sols):
                continue
            R, t = _pose_from_points(P, s64[:, None] * j)
            cond = float(np.linalg.cond(distance_jacobian(s64, ca, cb, cg)))
            sols.append({"R": R, "t": t, "depths": s64, "cond": cond})
    return sols


def min_angle_deg(P):
    """Smallest interior angle of the triangle P [3,3]."""
    P = np.asarray(P, np.float64)
    out = []
    for k in range(3):
        u, v = P[(k + 1) % 3] - P[k], P[(k + 2) % 3] - P[k]
        out.append(np.degrees(np.arctan2(np.linalg.norm(np.cross(u, v)), u @ v)))
    return min(out)


def danger_cylinder_distance(P, R, t):
    """Distance of the camera centre of pose (R, t) from the danger cylinder of triangle P [3,3] (the cylinder through the
    triangle's circumcircle, perpendicular to its plane), relative to the circumradius.  On the cylinder two P3P solutions
    coincide and the depths' Jacobian is singular."""
    P = np.asarray(P, np.float64)
    C = -np.asarray(R).T @ np.asarray(t)
    a, b = P[1] - P[0], P[2] - P[0]
    nrm = np.cross(a, b)
    O = P[0] + np.cross(a @ a * b - b @ b * a, nrm) / (2 * (nrm @ nrm))     # circumcentre
    rho = np.linalg.norm(P[0] - O)
    d = C - O
    d_in_plane = d - (d @ nrm) / (nrm @ nrm) * nrm
    return abs(np.linalg.norm(d_in_plane) - rho) / rho


def pose_error(R, t, R_ref, t_ref):
    """max(|R - R_ref|, |t - t_ref| / |t_ref|): rotation entries absolute, translation relative."""
    return max(float(np.max(np.abs(np.asarray(R) - R_ref))), float(np.linalg.norm(np.asarray(t) - t_ref) / np.linalg.norm(t_ref)))


def classify(pose, K, pts2d, pts3d, thr):
    """fp64 inlier test of all points under pose [3,4]: (inlier bool [n], border bool [n]).  A point is an inlier when its
    depth is > 1e-9 and its squared reprojection error is < thr^2; it is a border point when it is in front of the camera and
    its squared error is within 1e-6 px^2 of thr^2."""
    pose = np.asarray(pose, np.float64)
    X = np.asarray(pts3d, np.float64) @ pose[:, :3].T + pose[:, 3]
    z = X[:, 2]
    front = z > 1e-9
    with np.errstate(divide="ignore", invalid="ignore"):
        du = K[0, 0] * X[:, 0] / z + K[0, 2] - pts2d[:, 0]
        dv = K[1, 1] * X[:, 1] / z + K[1, 2] - pts2d[:, 1]
        e2 = du * du + dv * dv
    thr2 = thr * thr
    inl = front & (e2 < thr2)
    border = front & (np.abs(e2 - thr2) <= BORDER_PX2)
    return inl, border


def _rodrigues(w):
    th = np.linalg.norm(w)
    W = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
    if th < 1e-12:
        return np.eye(3) + W + 0.5 * W @ W
    return np.eye(3) + np.sin(th) / th * W + (1 - np.cos(th)) / (th * th) * W @ W


def reprojection_residuals(pose, K, pts2d, pts3d):
    X = pts3d @ pose[:, :3].T + pose[:, 3]
    u = K[0, 0] * X[:, 0] / X[:, 2] + K[0, 2] - pts2d[:, 0]
    v = K[1, 1] * X[:, 1] / X[:, 2] + K[1, 2] - pts2d[:, 1]
    return np.concatenate([u, v])


def refine_lsq(pose, K, pts2d, pts3d):
    """The least-squares pose of the given correspondences (all of them are used), found by scipy's Levenberg-Marquardt from
    ``pose`` with tolerances 1e-15; parameters are a left rotation update and the translation, central-difference Jacobian.
    The solve is restarted from its result (the rotation update re-centred at 0) until it stops moving, so that the answer
    does not depend on how far the start was.  Returns (pose [3,4], result of the last solve)."""
    from scipy.optimize import least_squares
    pose = np.asarray(pose, np.float64)
    pts2d = np.asarray(pts2d, np.float64)
    pts3d = np.asarray(pts3d, np.float64)
    for _ in range(5):
        R0 = pose[:, :3]

        def unpack(x):
            return np.concatenate([_rodrigues(x[:3]) @ R0, x[3:, None]], 1)

        x0 = np.concatenate([np.zeros(3), pose[:, 3]])
        r = least_squares(lambda x: reprojection_residuals(unpack(x), K, pts2d, pts3d), x0, jac="3-point", method="lm",
                          xtol=1e-15, ftol=1e-15, gtol=1e-15, x_scale="jac")
        new = unpack(r.x)
        moved = np.max(np.abs(new - pose) / np.maximum(1.0, np.abs(pose)))
        pose = new
        if moved < 1e-14:
            break
    return pose, r
