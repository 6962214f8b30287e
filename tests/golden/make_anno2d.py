"""Generate the 2D annotation golden vectors with the reference's own functions (feature_process.count_features,
get_assign_matrix through save_2d_anno, src/sfm/postprocess/feature_process.py:95-135, :197-294).

    python tests/golden/make_anno2d.py <path of the reference checkout>

Writes ``pnp_anno2d_cases.npz``.  For D = 1 and D = 256, a planted model -- point ids (some above 2^31), merge groups and each
image's point ids -- and features from ``anno2d_reference.features(seed, ...)`` go through the reference with ``h5py``
stubbed (the features file is a dict of per-image arrays).  The file keeps the inputs, the assign matrices read back from
the written files, each file's SHA-256 and the bytes of ``anno_2d.json``.

What the model plants: in image 0 a point observed twice (features 0 and 3) beside a point of the same group (feature 2), so
the last index wins and the group is paired once; other images draw ids with repeats from a pool of kept and dropped ids;
image 3 has no kept point and gets no file; and features past each image's count hold unrelated ids.
"""
import hashlib
import json
import os
import sys
import tempfile
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from tests import anno2d_reference as ar  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "pnp_anno2d_cases.npz")
CASES = ((1, 11, 9, 40), (256, 12, 6, 24))        # (D, seed, F, cap)
EMPTY_IMAGE = 3


def plant(rng, F, cap):
    ids = rng.choice(np.arange(1, 5000), 60, replace=False).astype(np.int64)
    ids[rng.choice(60, 12, replace=False)] += 2 ** 31 + 777
    kept = ids[:45]
    sizes, groups, i = [], [], 0
    while i < len(kept):
        s = min(int(rng.integers(1, 4)), len(kept) - i)
        groups.append(kept[i:i + s])
        i += s
    dropped = ids[45:]
    A, B = groups[0][0], None
    for g in groups:
        if len(g) >= 2:
            A, B = g[0], g[1]
            break
    rows = []
    for f in range(F):
        n = int(rng.integers(cap // 2, cap + 1))
        if f == EMPTY_IMAGE:
            row = rng.choice(np.concatenate([dropped, [-1]]), n)
        else:
            row = rng.choice(np.concatenate([kept, dropped, [-1, -1]]), n)
        if f == 0:
            row[:4] = [A, -1, B, A]
        rows.append(row.astype(np.int64))
    return groups, rows, A, B


def main(reference):
    sys.path.insert(0, reference)
    h5py = types.ModuleType("h5py")
    sys.modules["h5py"] = h5py
    from src.sfm.postprocess import feature_process
    out = {}
    for D, seed, F, cap in CASES:
        rng = np.random.default_rng(seed)
        groups, rows, A, B = plant(rng, F, cap)
        kp, de, sc = ar.features(seed, F, D, cap)
        names = [f"seq{D}/color/{f}.png" for f in range(F)]
        feats = {names[f]: {"keypoints": kp[f, :len(rows[f])], "descriptors": de[f, :, :len(rows[f])], "scores": sc[f, :len(rows[f])]}
                 for f in range(F)}
        images = {f + 1: types.SimpleNamespace(name=names[f], point3D_ids=rows[f]) for f in range(F)}
        points_idxs = {g: [int(x) for x in groups[g]] for g in range(len(groups))}
        mapping = feature_process.id_mapping(points_idxs)
        xyzs = np.zeros((len(groups), 3))
        cwd = os.getcwd()
        with tempfile.TemporaryDirectory() as tmp:
            os.chdir(tmp)
            _, _, _, _, _, to_2d = feature_process.count_features(names, feats, images, mapping)
            cfg = types.SimpleNamespace(network=types.SimpleNamespace(detection="superpoint"))
            feature_process.save_2d_anno(cfg, names, feats, xyzs, points_idxs, to_2d, "anno_2d.json")
            index = open("anno_2d.json", "rb").read()
            written = json.loads(index)
            texts = {a["img_file"]: open(a["anno_file"], "rb").read() for a in written}
            os.chdir(cwd)
        gmap = ar.group_map(np.concatenate(groups), np.concatenate([[0], np.cumsum([len(g) for g in groups])]))
        assign, sha = [], []
        for f in range(F):
            t = texts.get(names[f])
            m = ar.assign_pairs(rows[f], gmap)
            if t is None:
                assert m.shape[1] == 0
                assign.append(m)
                sha.append("")
                continue
            a = np.array(json.loads(t)["assign_matrix"], np.int64)
            assert np.array_equal(a, m)
            assert t.decode() == ar.anno_text(kp[f, :len(rows[f])], de[f, :, :len(rows[f])], sc[f, :len(rows[f])], a)
            assign.append(a)
            sha.append(hashlib.sha256(t).hexdigest())
        assert names[EMPTY_IMAGE] not in texts and (np.concatenate(groups) > 2 ** 31).any()
        a0 = assign[0]
        g_ab = gmap[int(A)]
        assert gmap[int(B)] == g_ab and list(a0[:, 0]) == [3, g_ab] and int((a0[1] == g_ab).sum()) == 1
        pid = np.full((F, cap), -1, np.int64)
        for f in range(F):
            pid[f, :len(rows[f])] = rows[f]
            pid[f, len(rows[f]):] = rng.integers(1, 2 ** 40, cap - len(rows[f]))    # past the count: never read
        pre = f"d{D}_"
        out.update({pre + "seed": seed, pre + "pid": pid, pre + "counts": np.array([len(r) for r in rows], np.int64),
                    pre + "names": np.array(names), pre + "group_ids": np.concatenate(groups).astype(np.int64),
                    pre + "group_offsets": np.concatenate([[0], np.cumsum([len(g) for g in groups])]).astype(np.int64),
                    pre + "assign": np.concatenate(assign, axis=1), pre + "num_matches": np.array([a.shape[1] for a in assign], np.int64),
                    pre + "sha256": np.array(sha), pre + "index": np.frombuffer(index, np.uint8)})
    np.savez_compressed(OUT, **out)
    print(f"{OUT}: {os.path.getsize(OUT)} bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.environ.get("ONEPOSE_REFERENCE", ""))
