"""opb_ransac_pnp stage by stage against the fp64 references of tests/pnp_reference.py.

The tests call the C ABI with a workspace they own and read its per-hypothesis records (13 doubles per frame and hypothesis,
frame-major: inlier count, R row-major, t; see include/onepose_b200.h):
- hypotheses: every stored R is a rotation; the stored pose reprojects the three CPU-drawn sample points (which pins the
  sampler); its count is the CPU recount; on noise-free scenes a well-conditioned sample's count is the best over every P3P
  solution of that sample, and without outliers it is n with the ground-truth pose -- on generic, planar, head-on grid
  (symmetric samples), far and mm-scale scenes;
- refinement and outputs: the pose is the least-squares optimum of the reported inliers, inlier_mask is the fp64 test under
  the pose, n_inliers its sum, and the answer does not depend on the unit of length;
- edges in one batch (empty, 3, 4, 5 points, coincident, collinear, behind the camera) and more than 65535 frames.
A sample is well-conditioned when its triangle's smallest angle is at least 10 degrees, every P3P solution's distance
equations have a Jacobian with condition number below 1e6 (poses are compared to max(1e-8, 1e-13 cond)), and no camera
centre of a solution (the reference's or the kernel's) is within 1 % of the circumradius of the danger cylinder: there two
solutions merge, and rounding in the data moves them by about its square root (a grid camera above the circumcircle of three
grid points is such a case).  Points within 1e-6 px^2 of the threshold are
not compared."""
import numpy as np
import pytest
import torch

from onepose_b200 import _lib, synthetic
from tests import pnp_reference as ref

pytestmark = pytest.mark.gpu

THR = 5.0
SEED = 0x5EED


def _call(frames, H, thr=THR, seed=SEED, read_hyp=True):
    """frames: list of (K [3,3], pts2d [n,2], pts3d [n,3]).  Returns numpy hyp [B,H,13] (NaN where the kernel wrote nothing),
    pose [B,3,4], mask [total], n_inliers [B], offsets [B+1]."""
    lib = _lib.load()
    B = len(frames)
    off = np.concatenate([[0], np.cumsum([len(f[1]) for f in frames])]).astype(np.int32)
    total = int(off[-1])
    K = torch.from_numpy(np.stack([np.asarray(f[0], np.float64).reshape(9) for f in frames])).cuda()
    p2 = np.zeros((max(total, 1), 2))
    p3 = np.zeros((max(total, 1), 3))
    if total:
        p2[:total] = np.concatenate([np.asarray(f[1], np.float64).reshape(-1, 2) for f in frames])
        p3[:total] = np.concatenate([np.asarray(f[2], np.float64).reshape(-1, 3) for f in frames])
    p2, p3 = torch.from_numpy(p2).cuda(), torch.from_numpy(p3).cuda()
    offs = torch.from_numpy(off).cuda()
    ws = torch.full((B * H * 13,), float("nan"), dtype=torch.float64, device="cuda")
    pose = torch.full((B, 12), float("nan"), dtype=torch.float64, device="cuda")
    mask = torch.full((max(total, 1),), -1, dtype=torch.int32, device="cuda")
    cnt = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    _lib.check(lib.opb_ransac_pnp(K.data_ptr(), p2.data_ptr(), p3.data_ptr(), offs.data_ptr(), B, H, float(thr), seed, ws.data_ptr(),
                                  pose.data_ptr(), mask.data_ptr(), cnt.data_ptr(), torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return {"hyp": ws.cpu().numpy().reshape(B, H, 13) if read_hyp else None, "pose": pose.cpu().numpy().reshape(B, 3, 4),
            "mask": mask[:total].cpu().numpy(), "cnt": cnt.cpu().numpy(), "off": off}


def _project(K, P, R, t):
    X = P @ R.T + t
    return X[:, :2] / X[:, 2:3] * np.array([K[0, 0], K[1, 1]]) + K[:2, 2]


def _rot(w):
    return ref._rodrigues(np.asarray(w, np.float64))


# ---- scene families: (K, pts2d, pts3d, R_gt, t_gt); noise-free and outlier-free unless said otherwise
def _generic(seed, n, scale=1.0):
    K, uv, P, gt = synthetic.make_pnp_scene(seed, n, outlier_frac=0.0, noise_px=0.0)
    return K, uv, P * scale, gt[:, :3], gt[:, 3] * scale


def _planar(seed, n):
    rs = np.random.RandomState(seed)
    K = np.array([[620.0, 0, 250], [0, 630.0, 262], [0, 0, 1]])
    P = np.concatenate([rs.uniform(-0.06, 0.06, size=(n, 2)), np.zeros((n, 1))], 1)
    R = _rot(rs.uniform(-0.6, 0.6, 3))
    t = np.array([0.02, -0.01, 0.6])
    return K, _project(K, P, R, t), P, R, t


def _grid(scale=1.0):
    """A 7 x 7 grid of 20 mm pitch faced head-on, centred on the optical axis: many samples are isosceles triangles seen from
    their symmetry plane."""
    K = np.array([[600.0, 0, 256], [0, 600.0, 256], [0, 0, 1]])
    g = np.arange(-3, 4) * 0.02
    P = np.stack(np.meshgrid(g, g, indexing="ij"), -1).reshape(-1, 2)
    P = np.concatenate([P, np.zeros((len(P), 1))], 1) * scale
    R, t = np.eye(3), np.array([0.0, 0.0, 0.6]) * scale
    return K, _project(K, P, R, t), P, R, t


def _far(seed, n):
    rs = np.random.RandomState(seed)
    K = np.array([[1500.0, 0, 256], [0, 1500.0, 256], [0, 0, 1]])
    P = 0.05 * rs.randn(n, 3)
    R = _rot(rs.randn(3))
    t = np.array([0.05, -0.03, 4.0])
    return K, _project(K, P, R, t), P, R, t


def _hyp_pose(rec):
    return np.concatenate([rec[1:10].reshape(3, 3), rec[10:13, None]], 1)


def _count_bounds(pose, K, uv, P, thr):
    inl, border = ref.classify(pose, K, uv, P, thr)
    lo = int((inl & ~border).sum())
    return lo, lo + int(border.sum())


def _check_hypotheses(tag, frame, recs, b, thr, noise_free, gt=None):
    """Per-hypothesis checks of frame b (recs [H,13]).  Returns (well-conditioned samples, worst ground-truth error over the
    other samples)."""
    K, uv, P = frame
    n = len(uv)
    j = ref.bearings(K, uv)
    n_wc, worst_other = 0, 0.0
    for h, rec in enumerate(recs):
        c = int(rec[0])
        assert c == rec[0] and 0 <= c <= n, (tag, h, rec[0])
        idx = list(ref.sample_indices(SEED, b, h, n))
        sols = ref.p3p_all(P[idx], j[idx])
        centres = [(s["R"], s["t"]) for s in sols] + ([(rec[1:10].reshape(3, 3), rec[10:13])] if c > 0 else [])
        wc = (bool(sols) and ref.min_angle_deg(P[idx]) >= 10 and max(s["cond"] for s in sols) < 1e6
              and min(ref.danger_cylinder_distance(P[idx], Rc, tc) for Rc, tc in centres) > 1e-2)
        n_wc += wc
        tol = max(1e-8, 1e-13 * max(s["cond"] for s in sols)) if wc else None   # data rounding, amplified
        if c > 0:
            pose = _hyp_pose(rec)
            R = pose[:, :3]
            assert np.max(np.abs(R @ R.T - np.eye(3))) <= 1e-12 and np.linalg.det(R) > 0, (tag, h)
            lo, hi = _count_bounds(pose, K, uv, P, thr)
            assert lo <= c <= hi, (tag, h, c, lo, hi)
            e = np.abs(_project(K, P[idx], R, pose[:, 3]) - uv[idx]).max()
            assert e <= (1e-6 if wc else 1e-3), (tag, h, idx, e)
            if wc:                             # one of the reference's solutions
                d = min(ref.pose_error(R, pose[:, 3], s["R"], s["t"]) for s in sols)
                assert d <= tol, (tag, h, idx, d, tol)
        if noise_free and wc:
            bounds = [_count_bounds(np.concatenate([s["R"], s["t"][:, None]], 1), K, uv, P, thr) for s in sols]
            assert max(lo for lo, _ in bounds) <= c <= max(hi for _, hi in bounds), (tag, h, c, bounds)
        if gt is not None:
            err = ref.pose_error(rec[1:10].reshape(3, 3), rec[10:13], *gt) if c > 0 else np.inf
            if wc:
                assert c == n and err <= tol, (tag, h, idx, c, err, tol)
            elif err > worst_other:
                worst_other = err
    return n_wc, worst_other


def test_hypotheses_against_p3p_reference():
    """Noise-free frames use a 0.05 px threshold, so that only an exact solution explains every point and a pose the planar
    ambiguity brings within a few pixels cannot tie with the true one; the noisy frame uses the usual 5 px."""
    scenes = {"generic": _generic(11, 200), "planar": _planar(12, 150), "grid": _grid(), "far": _far(13, 100),
              "generic_mm": _generic(14, 200, 1000.0), "grid_mm": _grid(1000.0)}
    frames = [s[:3] for s in scenes.values()]
    gts = [s[3:] for s in scenes.values()]
    K, uv, P, _ = synthetic.make_pnp_scene(15, 300, outlier_frac=0.4, noise_px=0.0)      # noise-free, 40 % outliers
    frames.append((K, uv, P))
    tags = list(scenes) + ["outliers"]
    thr = 0.05
    full = _call(frames, 512, thr=thr)
    for H in (1, 127, 129):                    # a record depends on (frame, hypothesis) only, not on the grid shape
        part = _call(frames, H, thr=thr)
        np.testing.assert_array_equal(part["hyp"], full["hyp"][:, :H])
    noisy = synthetic.make_pnp_scene(16, 300)[:3]                                      # 0.5 px noise, 40 % outliers
    cases = [(tag, frames[b], full["hyp"][b], b, thr, True, gts[b] if b < len(gts) else None) for b, tag in enumerate(tags)]
    cases.append(("noisy", noisy, _call([noisy], 512)["hyp"][0], 0, THR, False, None))
    for tag, frame, recs, b, t, noise_free, gt in cases:
        n_wc, worst = _check_hypotheses(tag, frame, recs, b, t, noise_free, gt)
        print(f"{tag}: {n_wc} of 512 samples well-conditioned; worst ground-truth error of the others {worst:.3g}")
        if tag.startswith("grid"):
            assert n_wc >= 100, n_wc


@pytest.mark.parametrize("scale", [1.0, 1000.0])
def test_refined_pose_is_least_squares_optimum_of_reported_inliers(scale):
    combos = [(n, f) for n in (30, 100, 400, 1500) for f in (0.2, 0.5, 0.85)]
    frames = []
    for i, (n, f) in enumerate(combos):
        K, uv, P, _ = synthetic.make_pnp_scene(100 + i, n, outlier_frac=f)
        frames.append((K, uv, P * scale))
    out = _call(frames, 4096, read_hyp=False)
    for b, (K, uv, P) in enumerate(frames):
        o0, o1 = out["off"][b], out["off"][b + 1]
        mask = out["mask"][o0:o1]
        pose = out["pose"][b]
        assert set(np.unique(mask)) <= {0, 1}
        assert out["cnt"][b] == mask.sum(), (b, out["cnt"][b], mask.sum())
        inl, border = ref.classify(pose, K, uv, P, THR)
        assert np.array_equal(mask.astype(bool)[~border], inl[~border]), (b, combos[b])
        assert mask.sum() >= 4, (b, combos[b])
        m = mask.astype(bool)
        opt, _ = ref.refine_lsq(pose, K, uv[m], P[m])
        err = ref.pose_error(pose[:, :3], pose[:, 3], opt[:, :3], opt[:, 3])
        assert err <= 1e-8, (b, combos[b], err)
    if scale == 1.0:
        return
    base = _call([(K, uv, P / scale) for K, uv, P in frames], 4096, read_hyp=False)
    for b in range(len(frames)):
        p1, pk = base["pose"][b], out["pose"][b]
        o0, o1 = out["off"][b], out["off"][b + 1]
        assert np.array_equal(base["mask"][o0:o1], out["mask"][o0:o1]), (b, combos[b])
        err = ref.pose_error(pk[:, :3], pk[:, 3] / scale, p1[:, :3], p1[:, 3])
        assert err <= 1e-8, (b, combos[b], err)


def test_edge_frames_in_one_batch():
    rs = np.random.RandomState(7)
    big = [synthetic.make_pnp_scene(200 + i, n)[:3] for i, n in enumerate((500, 800, 300))]
    K0 = np.array([[600.0, 0, 256], [0, 600.0, 256], [0, 0, 1]])
    R, t = _rot([0.2, -0.3, 0.1]), np.array([0.01, 0.02, 0.55])
    small = {}
    for n in (4, 5):
        P = 0.05 * rs.randn(n, 3)
        small[n] = (K0, _project(K0, P, R, t), P)
    Pc = np.tile([[0.01, 0.02, 0.03]], (20, 1))
    coincident = (K0, _project(K0, Pc, R, t), Pc)
    Pl = np.linspace(-0.05, 0.05, 30)[:, None] * np.array([[0.3, 0.5, 0.8]]) + [0.0, 0.01, 0.0]
    collinear = (K0, _project(K0, Pl, R, t) + rs.randn(30, 2) * 0.3, Pl)
    Pf = 0.05 * rs.randn(60, 3)
    Xb = -(Pf @ R.T + t)                                   # behind the camera, seen through the centre at the same pixels
    behind = (K0, _project(K0, Pf, R, t), (Xb - t) @ R)   # world points whose camera coordinates under (R, t) are Xb
    empty = (K0, np.zeros((0, 2)), np.zeros((0, 3)))
    three = (K0, small[4][1][:3], small[4][2][:3])
    frames = [big[0], empty, big[1], three, small[4], coincident, small[5], collinear, behind, big[2]]
    names = ["big0", "empty", "big1", "three", "four", "coincident", "five", "collinear", "behind", "big2"]
    out = _call(frames, 512, read_hyp=False)
    ident = np.eye(4)[:3]
    for b, name in enumerate(names):
        o0, o1 = out["off"][b], out["off"][b + 1]
        mask, pose = out["mask"][o0:o1], out["pose"][b]
        if name in ("empty", "three", "coincident", "collinear"):
            assert np.array_equal(pose, ident) and out["cnt"][b] == 0 and not mask.any(), name
        elif name in ("four", "five"):
            assert ref.pose_error(pose[:, :3], pose[:, 3], R, t) <= 1e-8, (name, pose)
            assert out["cnt"][b] == len(mask) and mask.all(), name
        elif name == "behind":
            K, uv, P = frames[b]
            z = P @ pose[:, :3].T[:, 2] + pose[2, 3]
            assert not np.any(mask.astype(bool) & (z <= 0)), z[mask.astype(bool)]
            assert out["cnt"][b] == mask.sum()
    emptied = [f if n.startswith("big") else empty for f, n in zip(frames, names)]
    again = _call(emptied, 512, read_hyp=False)
    for b, name in enumerate(names):
        if name.startswith("big"):
            assert out["pose"][b].tobytes() == again["pose"][b].tobytes() and out["cnt"][b] == again["cnt"][b], name
            m_out = out["mask"][out["off"][b]:out["off"][b + 1]]
            m_again = again["mask"][again["off"][b]:again["off"][b + 1]]
            assert np.array_equal(m_out, m_again), name
        else:
            assert again["cnt"][b] == 0


def test_more_frames_than_a_grid_row():
    """70000 frames of 4 or 5 noise-free points: frames sit on the grid's x dimension, which has no 65535 limit."""
    B = 70000
    K0 = np.array([[600.0, 0, 256], [0, 600.0, 256], [0, 0, 1]])
    rs = np.random.RandomState(8)
    R, t = _rot([0.1, 0.4, -0.2]), np.array([-0.01, 0.02, 0.6])
    P = 0.05 * rs.randn(5, 3)
    uv = _project(K0, P, R, t)
    frames = [(K0, uv[:4 + b % 2], P[:4 + b % 2]) for b in range(B)]
    out = _call(frames, 16, read_hyp=False)
    ns = np.diff(out["off"])
    assert np.array_equal(out["cnt"], ns)
    assert np.all(out["mask"] == 1)
    err_R = np.abs(out["pose"][:, :, :3] - R).max()
    err_t = np.abs(out["pose"][:, :, 3] - t).max() / np.linalg.norm(t)
    assert max(err_R, err_t) <= 1e-8, (err_R, err_t)
