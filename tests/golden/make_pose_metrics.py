"""Generate the pose-metric golden vectors by running the UNMODIFIED reference functions.

Run in the build container only (needs /root/reference and cv2, which ``src/utils/eval_utils.py`` imports):

    python tests/golden/make_pose_metrics.py

Imports ``query_pose_error`` / ``aggregate_metrics`` (reference ``src/utils/eval_utils.py:45-63``, ``:105-120``) and
``cmd_evaluator.Evaluator`` (``src/evaluators/cmd_evaluator.py``) and runs them on seeded (pose_pred, pose_gt) pairs.  The
pairs are stored with the results in ``pnp_pose_metrics.npz`` (the ``pnp_`` prefix keeps it out of the matcher cases that
``tests/golden_util.py`` collects).
"""
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, "/root/reference")


def _axis_angle(axis, deg):
    k = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    th = np.deg2rad(deg)
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx


def pose_metric_pairs(seed=17):
    """~40 seeded (pose_pred, pose_gt) pairs for the pose metric: identical poses, 3x4 / 4x4 mixes, errors just below / above
    1, 3 and 5 (never on a threshold), near-180 degree rotations (one whose trace rounds below -1), the identity pose of a
    failed solve and a non-finite pose.  Returns (tags, pred [P,4,4], gt [P,4,4], pred_rows [P], gt_rows [P]): rows = 3 or 4
    is the shape the pair is evaluated with."""
    rs = np.random.RandomState(seed)

    def rand_pose():
        R = _axis_angle(rs.randn(3), rs.uniform(0, 180))
        return np.concatenate([np.concatenate([R, (0.1 * rs.randn(3) + [0, 0, 0.6])[:, None]], 1), [[0, 0, 0, 1.0]]], 0)

    def perturbed(gt, deg, cm):
        p = gt.copy()
        p[:3, :3] = _axis_angle(rs.randn(3), deg) @ gt[:3, :3]
        d = rs.randn(3)
        p[:3, 3] = gt[:3, 3] + d / np.linalg.norm(d) * cm / 100
        return p

    pairs = []
    gt = np.eye(4)
    pairs.append(("identical_identity", gt.copy(), gt, 3, 3))
    for rows in ((3, 3), (4, 4), (3, 4), (4, 3)):
        gt = rand_pose()
        pairs.append((f"identical_{rows[0]}x4_{rows[1]}x4", gt.copy(), gt, *rows))
    for thr in (1, 3, 5):
        for side, f in (("below", 0.999), ("above", 1.001)):
            gt = rand_pose()
            pairs.append((f"rot_{side}_{thr}", perturbed(gt, thr * f, 0.2 * thr), gt, 3, 4))
            gt = rand_pose()
            pairs.append((f"trans_{side}_{thr}", perturbed(gt, 0.2 * thr, thr * f), gt, 4, 3))
            gt = rand_pose()
            pairs.append((f"both_{side}_{thr}", perturbed(gt, thr * f, thr * f), gt, 4, 4))
    for k in range(6):
        gt = rand_pose()
        pairs.append((f"random_{k}", perturbed(gt, rs.uniform(0, 10), rs.uniform(0, 10)), gt, 3, 3))
    for deg in (179.0, 179.9, 179.999):
        gt = rand_pose()
        pairs.append((f"near180_{deg}", perturbed(gt, deg, 0.5), gt, 3, 3))
    found = 0
    while found < 2:        # exactly 180 degrees: one pair whose computed trace stays >= -1, one whose trace rounds below -1 (NaN)
        gt = rand_pose()
        p = perturbed(gt, 180.0, 0.5)
        below = np.trace(np.dot(p[:3, :3], gt[:3, :3].T)) < -1
        if below == bool(found):
            pairs.append(("exact180_nan" if below else "exact180", p, gt, 4, 4))
            found += 1
    for k in range(3):
        gt = rand_pose()
        pairs.append((f"failed_solve_{k}", np.eye(4), gt, 3 if k % 2 == 0 else 4, 4))
    gt = rand_pose()
    bad = gt.copy()
    bad[:3, :] = np.nan
    pairs.append(("non_finite", bad, gt, 3, 4))
    tags, pred, gts, pr, gr = zip(*pairs)
    return np.array(tags), np.stack(pred), np.stack(gts), np.array(pr), np.array(gr)


def pose_metric_cases():
    """query_pose_error / aggregate_metrics and cmd_evaluator.Evaluator of the imported, unmodified reference on the pairs of
    pose_metric_pairs (stored with the results)."""
    from src.utils import eval_utils
    from src.evaluators.cmd_evaluator import Evaluator
    tags, pred, gt, pred_rows, gt_rows = pose_metric_pairs()
    R, t = [], []
    ev = Evaluator()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")           # arccos of the trace below -1: the reference's own NaN
        for p, g, pr, gr in zip(pred, gt, pred_rows, gt_rows):
            r_err, t_err = eval_utils.query_pose_error(p[:pr], g[:gr])
            R.append(r_err)
            t.append(t_err)
            ev.evaluate(p[:pr], g[:gr])
        agg = eval_utils.aggregate_metrics({"R_errs": R, "t_errs": t})
        summ = ev.summarize()
    out = {"tags": tags, "pose_pred": pred, "pose_gt": gt, "pred_rows": pred_rows, "gt_rows": gt_rows,
           "rot_err_deg": np.array(R, np.float64), "trans_err_cm": np.array(t, np.float64),
           "aggregate_keys": np.array(list(agg.keys())), "aggregate_vals": np.array(list(agg.values()), np.float64),
           "summarize_keys": np.array(list(summ.keys())), "summarize_vals": np.array(list(summ.values()), np.float64)}
    print("pose metrics:", len(tags), "pairs,", int(np.isnan(out["rot_err_deg"]).sum()), "NaN rotation errors,", agg, summ)
    np.savez_compressed(os.path.join(HERE, "pnp_pose_metrics.npz"), **out)


if __name__ == "__main__":
    pose_metric_cases()
