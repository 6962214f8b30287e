"""Generate the SfM post-processing golden vectors with the reference's own functions (run.py postprocess, :154-163).

    python tests/golden/make_sfm.py <path of the reference checkout>

Writes ``pnp_sfm_cases.npz`` (the ``pnp_`` prefix keeps it out of the matcher's forward cases, which tests/golden_util.py
collects by file name).  A synthetic COLMAP model is written with the reference's ``write_model``; ``get_tkl``, ``filter_3d``,
``merge`` and ``get_kpt_ann`` run on it as run.py runs them, with ``h5py`` and ``matplotlib`` stubbed (the features file is a
dict of per-image keypoints / descriptors / scores from ``sfm_reference.features``), and the annotation files they write are
read back.  The file keeps the two ``.bin`` files' bytes, the box corners, image names and feature seed, and what the
reference made of them: the threshold, the merge groups, the averages and each collected observation as an (image, feature)
pair.  The reference's collect arrays are asserted equal to those features, so they are not stored.

What the model plants: about 2000 points with sparse unsorted ids (some above 2^31), track lengths 2..40 with max_num_kp3d set
so that the kept group at the threshold overshoots it, a quarter of the points outside the box and every point at least
1e-4 |v|^2 from each box plane, clusters of 2-5 points within 0.2-0.8 mm, a chain A-B-C whose middle link makes the greedy
pass drop C without recording it, no pair distance within 1e-9 of the threshold, images without a valid observation, a point
observed twice in one image, and D = 32.
"""
import os
import sys
import tempfile
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from tests import sfm_reference as sr  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "pnp_sfm_cases.npz")
SEED, D, F, THRESHOLD = 7, 32, 24, 1e-3
EMPTY_IMAGES = (5, 17)


def _stub_modules(features):
    h5py = types.ModuleType("h5py")
    h5py.File = lambda path, mode="r": features
    sys.modules["h5py"] = h5py
    mpl = types.ModuleType("matplotlib")
    mpl.pyplot = types.ModuleType("matplotlib.pyplot")
    sys.modules["matplotlib"] = mpl
    sys.modules["matplotlib.pyplot"] = mpl.pyplot


def _plant(rng):
    o = np.array([0.05, -0.02, 0.3])
    R = np.linalg.qr(rng.normal(size=(3, 3)))[0]
    e = R * np.array([0.21, 0.17, 0.13])                      # orthogonal edges (columns)
    e1, e2, e3 = e[:, 0], e[:, 1], e[:, 2]
    corners = np.array([o + e2, o + e1 + e2, o + e1 + e2 + e3, o + e2 + e3, o, o + e1, o + e1 + e3, o + e3])   # c4 = o, c5, c0, c7
    box = lambda u: o + u[..., 0:1] * e1 + u[..., 1:2] * e2 + u[..., 2:3] * e3  # noqa: E731
    pts = []
    for _ in range(1500):                                      # inside, every box coordinate in [0.002, 0.998]
        pts.append(box(rng.uniform(0.002, 0.998, 3)))
    for _ in range(500):                                       # outside along at least one axis
        u = rng.uniform(0.002, 0.998, 3)
        a = rng.integers(0, 3)
        u[a] = rng.uniform(-0.3, -0.002) if rng.random() < 0.5 else rng.uniform(1.002, 1.3)
        pts.append(box(u))
    lens = list(rng.integers(2, 41, len(pts)))
    for _ in range(40):                                        # clusters of 2-5 points within 0.2-0.8 mm of a centre
        c = box(rng.uniform(0.05, 0.95, 3))
        for _ in range(rng.integers(2, 6)):
            d = rng.normal(size=3)
            pts.append(c + d / np.linalg.norm(d) * rng.uniform(2e-4, 8e-4))
            lens.append(40)
    c = box(np.array([0.5, 0.5, 0.5]))                         # the chain: |AB| = |BC| = 0.7 mm, |AC| = 1.4 mm
    chain = [len(pts), len(pts) + 1, len(pts) + 2]
    for t in (0.0, 7e-4, 1.4e-3):
        pts.append(c + t * e1 / np.linalg.norm(e1))
        lens.append(40)
    return np.array(pts), np.array(lens, np.int64), corners, chain


def main(reference):
    sys.path.insert(0, reference)
    rng = np.random.default_rng(20261018)
    while True:
        xyz, lens, corners, chain = _plant(rng)
        from scipy.spatial.distance import pdist
        dist = pdist(xyz.astype(np.float32))
        if not (np.abs(dist - THRESHOLD) < 1e-9).any():
            break
    P = len(xyz)
    # sparse unsorted ids, a few above 2^31; the chain's ids ascend so that A is walked first
    ids = rng.choice(np.arange(1, 40 * P), P, replace=False).astype(np.int64)
    ids[rng.choice(P, 25, replace=False)] += 2 ** 31 + 12345
    ids[chain] = np.sort(ids[chain])
    order_in_file = rng.permutation(P)

    # observations in the images: each point in 1-3 images, one point twice in one image, two images without a valid one
    obs_of = {}
    for i in range(P):
        imgs = rng.choice([f for f in range(F) if f not in EMPTY_IMAGES], rng.integers(1, 4), replace=False)
        obs_of[i] = list(imgs)
    dup = int(chain[0])
    obs_of[dup].append(obs_of[dup][0])
    feats = [[] for _ in range(F)]
    for i in order_in_file:
        for f in obs_of[i]:
            feats[f].append(int(ids[i]))
    for f in range(F):                                          # features without a 3D point in between
        ext = feats[f] + [-1] * (3 + int(rng.integers(0, 20)))
        feats[f] = [ext[j] for j in rng.permutation(len(ext))]
    cap = max(len(p) for p in feats)
    scores, desc = sr.features(SEED, F, D, cap)

    names = [f"scan/color/{f}.png" for f in range(F)]          # relative: get_kpt_ann writes beside them
    features = {names[f]: {"keypoints": np.zeros((len(feats[f]), 2), np.float32), "descriptors": desc[f, :, :len(feats[f])],
                           "scores": scores[f, :len(feats[f])]} for f in range(F)}
    _stub_modules(features)
    from src.utils.colmap import read_write_model as rwm
    from src.sfm.postprocess import feature_process, filter_points, filter_tkl

    max_num_kp3d = 1200
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        os.chdir(tmp)                                           # save_2d_anno writes next to each image's directory
        model = os.path.join(tmp, "outputs", "sfm_ws", "model")
        os.makedirs(model)
        cams = {1: rwm.Camera(id=1, model="PINHOLE", width=640, height=480, params=np.array([500.0, 500.0, 320.0, 240.0]))}
        imgs = {}
        for f in range(F):
            p = np.array(feats[f], dtype=np.int64)
            imgs[f + 1] = rwm.Image(id=f + 1, qvec=np.array([1.0, 0, 0, 0]), tvec=np.zeros(3), camera_id=1, name=names[f],
                                    xys=np.zeros((len(p), 2)), point3D_ids=p)
        pts3d = {}
        for i in order_in_file:
            L = int(lens[i])
            pts3d[int(ids[i])] = rwm.Point3D(id=int(ids[i]), xyz=xyz[i], rgb=np.zeros(3, np.uint8), error=0.5,
                                             image_ids=np.arange(L, dtype=np.int32) % F + 1, point2D_idxs=np.arange(L, dtype=np.int32))
        rwm.write_model(cams, imgs, pts3d, model, ".bin")
        box_path = os.path.join(tmp, "box3d_corners.txt")
        np.savetxt(box_path, corners)
        tl, _ = filter_tkl.get_tkl(model, thres=max_num_kp3d)
        kxyz, kidx = filter_points.filter_3d(model, tl, box_path)
        mxyz, midx = filter_points.merge(kxyz, kidx, dist_threshold=THRESHOLD)
        cfg = types.SimpleNamespace(network=types.SimpleNamespace(detection="superpoint"))
        out = os.path.join(tmp, "outputs")
        feature_process.get_kpt_ann(cfg, names, "feats.h5", out, midx, mxyz)
        avg = dict(np.load(os.path.join(out, "anno", "anno_3d_average.npz")))
        clt = dict(np.load(os.path.join(out, "anno", "anno_3d_collect.npz")))
        idxs = np.load(os.path.join(out, "anno", "idxs.npy"))
        pbin = np.frombuffer(open(os.path.join(model, "points3D.bin"), "rb").read(), np.uint8)
        ibin = np.frombuffer(open(os.path.join(model, "images.bin"), "rb").read(), np.uint8)
        os.chdir(cwd)

    # the model agrees with the reference bit for bit, and the fixture plants what it claims
    m = sr.postprocess(ids, xyz, lens, [np.array(p) for p in feats], scores, desc, corners,
                       max_num_kp3d, THRESHOLD)
    groups = [np.asarray(midx[g], np.int64) for g in range(len(midx))]
    assert m["track_length"] == tl and np.sum(lens >= tl) > max_num_kp3d
    assert len(groups) == len(m["groups"]) and all(np.array_equal(a, b) for a, b in zip(groups, m["groups"]))
    assert np.array_equal(m["keypoints3d"], mxyz) and np.array_equal(avg["keypoints3d"], mxyz)
    assert np.array_equal(idxs, m["idxs"]) and idxs.dtype == np.int64
    assert np.array_equal(clt["descriptors3d"], m["descriptors3d_collect"]) and np.array_equal(clt["scores3d"], m["scores3d_collect"])
    assert np.array_equal(avg["descriptors3d"], m["descriptors3d"]) and np.array_equal(avg["scores3d"], m["scores3d"])
    members = np.concatenate(groups)
    kept = set(np.asarray(kidx).tolist())
    assert ids[chain[2]] in kept and ids[chain[2]] not in set(members.tolist()), "the chain's last point must be dropped"
    assert any(len(g) > 1 for g in groups)
    assert (np.asarray(kidx) > 2 ** 31).any()
    np.savez_compressed(OUT, points3d_bin=pbin, images_bin=ibin, corners=corners, names=np.array(names), seed=SEED, D=D, cap=cap,
                        max_num_kp3d=max_num_kp3d, dist_threshold=THRESHOLD, track_length=tl,
                        kept_ids=np.asarray(kidx, np.int64),
                        group_offsets=np.concatenate([[0], np.cumsum([len(g) for g in groups])]).astype(np.int64), group_ids=members,
                        keypoints3d=mxyz, descriptors3d=avg["descriptors3d"], scores3d=avg["scores3d"], obs=m["obs"], idxs=idxs,
                        chain_ids=ids[chain], dup_id=ids[dup])
    print(f"{OUT}: P={P}, track_length={tl}, kept={len(kidx)}, groups={len(groups)}, observations={len(m['obs'])}, "
          f"{os.path.getsize(OUT)} bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.environ.get("ONEPOSE_REFERENCE", ""))
