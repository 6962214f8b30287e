"""The numpy model of the SfM post-processing (tests/sfm_reference.py) against the reference's output in
tests/golden/pnp_sfm_cases.npz, the COLMAP readers on the fixture's bytes, and the reference's quirks the model pins."""
import os

import numpy as np
import pytest

from onepose_b200 import sfm
from tests import sfm_reference as sr

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pnp_sfm_cases.npz")


@pytest.fixture(scope="module")
def case(tmp_path_factory):
    z = dict(np.load(GOLDEN))
    d = tmp_path_factory.mktemp("model")
    z["points3d_bin"].tofile(d / "points3D.bin")
    z["images_bin"].tofile(d / "images.bin")
    z["dir"] = d
    z["points"] = sfm.read_points3d_bin(d / "points3D.bin")
    z["images"] = sfm.read_images_bin(d / "images.bin")
    z["scores"], z["desc"] = sr.features(int(z["seed"]), len(z["names"]), int(z["D"]), int(z["cap"]))
    return z


def _model(z, **kw):
    ids, xyz, lens = z["points"]
    pid = dict(z["images"])
    a = dict(max_num_kp3d=int(z["max_num_kp3d"]), dist_threshold=float(z["dist_threshold"]))
    a.update(kw)
    return sr.postprocess(ids, xyz, lens, [pid[n] for n in z["names"]], z["scores"], z["desc"], z["corners"], **a)


def _groups(z):
    o = z["group_offsets"]
    return [z["group_ids"][o[g]:o[g + 1]] for g in range(len(o) - 1)]


def test_model_equals_the_reference_bit_for_bit(case):
    m = _model(case)
    assert m["track_length"] == int(case["track_length"])
    assert np.array_equal(m["kept_ids"], case["kept_ids"])
    ref = _groups(case)
    assert len(m["groups"]) == len(ref) and all(np.array_equal(a, b) for a, b in zip(m["groups"], ref))
    assert np.array_equal(m["keypoints3d"], case["keypoints3d"])
    assert np.array_equal(m["idxs"], case["idxs"])
    assert np.array_equal(m["obs"], case["obs"])
    assert np.array_equal(m["descriptors3d"], case["descriptors3d"]) and np.array_equal(m["scores3d"], case["scores3d"])


def test_readers_return_the_models_arrays(case):
    ids, xyz, lens = case["points"]
    assert ids.dtype == np.int64 and xyz.dtype == np.float64 and lens.dtype == np.int64 and xyz.shape == (len(ids), 3)
    assert len(np.unique(ids)) == len(ids) and (ids > 2 ** 31).any() and not np.all(np.diff(ids) > 0)   # sparse, unsorted
    assert lens.min() == 2 and lens.max() == 40
    assert set(case["kept_ids"].tolist()) <= set(ids.tolist())
    names = [n for n, _ in case["images"]]
    assert names == list(case["names"])
    for _, p in case["images"]:
        assert p.dtype == np.int64 and p.ndim == 1
    assert any(np.all(p == -1) for _, p in case["images"])          # an image without a valid observation


@pytest.mark.parametrize("which", ["points3D.bin", "images.bin"])
def test_truncated_or_padded_files_raise_naming_the_file(case, tmp_path, which):
    data = (case["dir"] / which).read_bytes()
    read = sfm.read_points3d_bin if which == "points3D.bin" else sfm.read_images_bin
    for bad in (data[:-5], data[:3], data + b"\0"):
        p = tmp_path / which
        p.write_bytes(bad)
        with pytest.raises(ValueError, match=which.replace(".", r"\.")):
            read(p)
    p = tmp_path / which
    p.write_bytes(b"\xff" * 8)                                      # a count no file can hold
    with pytest.raises(ValueError, match=which.replace(".", r"\.")):
        read(p)


def test_threshold_group_overshoots(case):
    ids, xyz, lens = case["points"]
    tl, mx = int(case["track_length"]), int(case["max_num_kp3d"])
    assert sr.get_tkl(lens, mx) == tl
    assert np.sum(lens >= tl) > mx >= np.sum(lens > tl)
    assert sr.get_tkl(lens, len(lens)) == lens.min() and sr.get_tkl(lens, 0) == lens.max()


def test_chain_drops_an_unrecorded_neighbour(case):
    a, b, c = case["chain_ids"]
    members = set(case["group_ids"].tolist())
    assert a in members and b in members and c in set(case["kept_ids"].tolist()) and c not in members
    g = next(g for g in _groups(case) if a in g)
    assert list(g) == [a, b]


def test_group_position_is_the_fp32_mean(case):
    m = _model(case)
    kept = dict(zip(m["kept_ids"].tolist(), range(len(m["kept_ids"]))))
    ids, xyz, lens = case["points"]
    _, kx = sr.filter_3d(ids, xyz, lens, int(case["track_length"]), case["corners"])
    f64 = np.array([np.mean(kx[[kept[q] for q in g]].astype(np.float64), axis=0) for g in m["groups"]])
    assert np.array_equal(case["keypoints3d"], np.array([np.mean(kx[[kept[q] for q in g]], axis=0) for g in m["groups"]]).astype(np.float64))
    assert not np.array_equal(case["keypoints3d"], f64)


def test_observations_are_group_major_then_member_then_image(case):
    pid = dict(case["images"])
    order = [pid[n] for n in case["names"]]
    obs, groups = case["obs"], _groups(case)
    ids_of_obs = np.array([order[f][k] for f, k in obs])
    r = 0
    for g, cnt in zip(groups, case["idxs"]):
        seg = ids_of_obs[r:r + cnt]
        pos = np.array([list(g).index(q) for q in seg])
        assert np.all(np.diff(pos) >= 0)                              # by member position within the group
        for q in g:
            rows = obs[r:r + cnt][seg == q]
            assert np.all(np.diff(rows[:, 0] * 10 ** 6 + rows[:, 1]) > 0)   # then image, feature
        r += cnt
    dup = int(case["dup_id"])
    rows = obs[ids_of_obs == dup]
    assert len(rows) > len(np.unique(rows[:, 0]))                    # one image observes it twice; both kept


def test_errors(case):
    with pytest.raises(ValueError):
        _model(case, max_num_kp3d=-1)
    ids, xyz, lens = case["points"]
    pid = dict(case["images"])
    imgs = [pid[n].copy() for n in case["names"]]
    q = int(case["group_ids"][0])
    for p in imgs:
        p[p == q] = -1
    with pytest.raises(KeyError):
        sr.postprocess(ids, xyz, lens, imgs, case["scores"], case["desc"], case["corners"], int(case["max_num_kp3d"]))
    with pytest.raises(ValueError):
        sr.postprocess(ids[:0], xyz[:0], lens[:0], imgs, case["scores"], case["desc"], case["corners"])


def test_planted_defects_break_equality(case, monkeypatch):
    base = _model(case)
    # the group at the threshold dropped: filter by length > threshold
    tkl = sr.get_tkl
    monkeypatch.setattr(sr, "get_tkl", lambda lens, t: tkl(lens, t) + 1)
    assert not np.array_equal(_model(case)["kept_ids"], base["kept_ids"])
    monkeypatch.setattr(sr, "get_tkl", tkl)
    # a row whose only recorded neighbour is someone else's: not skipped
    nl = sr.neighbour_lists
    monkeypatch.setattr(sr, "neighbour_lists", lambda x, t: [r[r >= j] for j, r in enumerate(nl(x, t))])
    assert len(_model(case)["groups"]) != len(base["groups"])
    monkeypatch.setattr(sr, "neighbour_lists", nl)
    # the observations in image-major order
    g = sr.gather
    def image_major(pids, members):
        obs, idxs = g(pids, members)
        out, r = [], 0
        for c in idxs:
            seg = obs[r:r + c]
            out.append(seg[np.lexsort((seg[:, 1], seg[:, 0]))])
            r += c
        return np.concatenate(out), idxs
    monkeypatch.setattr(sr, "gather", image_major)
    assert not np.array_equal(_model(case)["obs"], base["obs"])
