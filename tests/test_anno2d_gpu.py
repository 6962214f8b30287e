"""The 2D annotation files on an H100: sfm.assign_matrices and sfm.save_anno_2d against the reference's fixture
(tests/golden/make_anno2d.py) and the model of tests/anno2d_reference.py, the device float formatter against Python's repr,
chunked text against unchunked, the C entry points' outputs against sentinels, a busy caller stream, and the refusals."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

from onepose_b200 import _lib, sfm
from tests import anno2d_reference as ar
from tests.test_anno2d_reference_cpu import case, python_repr, stratified_floats

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def device_features(kp, de, sc):
    return {"keypoints": torch.from_numpy(kp).to(DEV), "descriptors": torch.from_numpy(de).to(DEV), "scores": torch.from_numpy(sc).to(DEV)}


def fixture_inputs(D):
    c = case(D)
    F, cap = c["pid"].shape
    images = [(str(c["names"][f]), c["pid"][f, :c["counts"][f]]) for f in range(F)]
    result = {"group_ids": c["group_ids"], "group_offsets": c["group_offsets"]}
    kp, de, sc = ar.features(int(c["seed"]), F, D, cap)
    return c, images, result, (kp, de, sc)


@pytest.mark.parametrize("D", (1, 256))
def test_pairs_equal_fixture(D):
    c, images, result, feats = fixture_inputs(D)
    mats, num = sfm.assign_matrices(result, images, device_features(*feats))
    assert np.array_equal(num, c["num_matches"])
    assert np.array_equal(np.concatenate(mats, axis=1), c["assign"]) and all(m.dtype == np.int64 and m.shape[0] == 2 for m in mats)


@pytest.mark.parametrize("D", (1, 256))
@pytest.mark.parametrize("small", (False, True))
def test_files_equal_fixture(D, small, tmp_path):
    c, images, result, feats = fixture_inputs(D)
    n, k = c["counts"], c["num_matches"]
    chunk = int((27 * (3 * n + D * n + 2 * k + 1) + 128).max()) if small else 1 << 30     # small: about one image per chunk
    cwd = os.getcwd()
    os.chdir(tmp_path)
    try:
        index = sfm.save_anno_2d("anno", [n for n, _ in images], result, images, device_features(*feats), max_chunk_bytes=chunk)
        assert open(os.path.join("anno", "anno_2d.json"), "rb").read() == c["index"].tobytes()
        assert json.dumps(index).encode() == c["index"].tobytes()
        for f, (name, _) in enumerate(images):
            path = os.path.join(os.path.dirname(os.path.dirname(name)), "anno_superpoint", os.path.basename(name).replace(".png", ".json"))
            if c["sha256"][f] == "":
                assert not os.path.exists(path)
            else:
                assert hashlib.sha256(open(path, "rb").read()).hexdigest() == c["sha256"][f]
    finally:
        os.chdir(cwd)


def dense_case(seed, F, cap, pool, D=2):
    rng = np.random.default_rng(seed)
    ids = rng.permutation(np.unique(rng.integers(1, 1 << 40, 2 * pool))[:pool]).astype(np.int64)
    kept = ids[: pool * 3 // 4]
    cuts = np.sort(rng.choice(np.arange(1, kept.size), kept.size // 3, replace=False))
    offsets = np.concatenate([[0], cuts, [kept.size]]).astype(np.int64)
    images = []
    for f in range(F):
        n = int(rng.integers(cap // 2, cap + 1)) if f else cap
        images.append((f"s/color/{f}.png", rng.choice(np.concatenate([ids, [-1]]), n)))
    kp = rng.uniform(0, 640, (F, cap, 2)).astype(np.float32)
    de = rng.normal(size=(F, D, cap)).astype(np.float32)
    sc = rng.uniform(size=(F, cap)).astype(np.float32)
    return images, {"group_ids": kept, "group_offsets": offsets}, (kp, de, sc)


@pytest.mark.parametrize("F,cap,pool", [(300, 2048, 5000), (40, 8192, 200), (8, 8192, 20000), (3, 1, 4)])
def test_pairs_equal_model(F, cap, pool):
    images, result, feats = dense_case(F + cap, F, cap, pool)
    mats, num = sfm.assign_matrices(result, images, device_features(*feats))
    gmap = ar.group_map(result["group_ids"], result["group_offsets"])
    for f, (_, p) in enumerate(images):
        want = ar.assign_pairs(p, gmap)
        assert np.array_equal(mats[f], want), f
        assert num[f] == want.shape[1]


def test_text_equal_json_dumps(tmp_path):
    images, result, feats = dense_case(5, 6, 300, 400, D=256)
    index = sfm.save_anno_2d(tmp_path / "anno", [str(tmp_path / n) for n, _ in images], result, images, device_features(*feats),
                             max_chunk_bytes=3 << 20)
    gmap = ar.group_map(result["group_ids"], result["group_offsets"])
    kp, de, sc = feats
    assert len(index) == 6
    for f, (_, p) in enumerate(images):
        n = len(p)
        want = ar.anno_text(kp[f, :n], de[f, :, :n], sc[f, :n], ar.assign_pairs(p, gmap))
        assert open(index[f]["anno_file"], "rb").read() == want.encode()


def device_repr(x):
    x = torch.from_numpy(np.ascontiguousarray(x, np.float32)).to(DEV)
    out = torch.zeros(x.numel(), 24, dtype=torch.uint8, device=DEV)
    ln = torch.empty(x.numel(), dtype=torch.int32, device=DEV)
    _lib.call(DEV, "opb_json_float_repr", x, x.numel(), out, ln)
    got = out.cpu().numpy().view("S24").ravel()
    assert np.array_equal(ln.cpu().numpy(), np.char.str_len(got))
    return got


def test_float_repr_stratified_and_one_binade():
    x = stratified_floats(seed=1)
    binade = (np.arange(1 << 23, dtype=np.uint32) | np.uint32(134 << 23)).view(np.float32)     # [128, 256): every value
    specials = np.array([np.inf, -np.inf, np.nan, 0.0, -0.0], np.float32)
    for v in (x, binade, specials):
        for i in range(0, v.size, 1 << 22):
            got, want = device_repr(v[i:i + (1 << 22)]), python_repr(v[i:i + (1 << 22)])
            bad = np.nonzero(got != want)[0]
            assert bad.size == 0, [(float(v[i + j]), got[j], want[j]) for j in bad[:5]]


def test_c_entries_sentinels():
    images, result, feats = dense_case(9, 5, 256, 300)
    F, cap = 5, 256
    ids = np.asarray(result["group_ids"])
    off = np.asarray(result["group_offsets"])
    grp = np.repeat(np.arange(off.size - 1, dtype=np.int32), np.diff(off))
    o = np.argsort(ids)
    pid = np.full((F, cap), -1, np.int64)
    for f, (_, p) in enumerate(images):
        pid[f, :len(p)] = p
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)  # noqa: E731
    SENT = -7777
    pairs = torch.full((2, F * cap + 64), SENT, dtype=torch.int64, device=DEV)
    outs = torch.full((2 * F + 1 + 64,), SENT, dtype=torch.int64, device=DEV)
    ws = sfm._ws(DEV, "opb_sfm_assign_workspace_bytes", F, cap)
    counts = t(np.array([len(p) for _, p in images], np.int32))
    _lib.call(DEV, "opb_sfm_assign_pairs", t(pid), counts, F, cap, t(ids[o]), t(grp[o]), ids.size, ws, ws.numel(), pairs, outs[:F + 1],
              outs[F + 1:2 * F + 1])
    h, ho = pairs.cpu().numpy(), outs.cpu().numpy()
    total = int(ho[F])
    assert (ho[2 * F + 1:] == SENT).all()
    # pairs is [2, F * cap + 64] here, so its row stride is not F * cap: only row 0's columns past the total and row 1's tail
    # past F * cap + total are never written
    flat = pairs.reshape(-1).cpu().numpy()
    written = np.zeros(flat.size, bool)
    written[:total] = True
    written[F * cap:F * cap + total] = True
    assert (flat[~written] == SENT).all()
    gmap = ar.group_map(ids, off)
    want = np.concatenate([ar.assign_pairs(p, gmap) for _, p in images], axis=1)
    assert np.array_equal(np.stack([flat[:total], flat[F * cap:F * cap + total]]), want)
    # the text: nothing past its length
    kp, de, sc = (t(a) for a in feats)
    num = ho[F + 1:2 * F + 1]
    desc = np.stack([np.arange(F), [len(p) for _, p in images], num, ho[:F]], 1).astype(np.int64)
    items = 3 * desc[:, 1] + 2 * desc[:, 1] + 2 * num + 1
    item_off = np.concatenate([[0], np.cumsum(items)]).astype(np.int64)
    ws2 = sfm._ws(DEV, "opb_anno2d_text_workspace_bytes", F, int(item_off[-1]))
    toff = torch.full((F + 1 + 8,), SENT, dtype=torch.int64, device=DEV)
    args = (t(desc), t(item_off), F)
    _lib.call(DEV, "opb_anno2d_text_lengths", *args, int(item_off[-1]), int(items.max()), 2, cap, kp, de, sc, pairs, F * cap, ws2, ws2.numel(),
              toff)
    to = toff.cpu().numpy()
    assert (to[F + 1:] == SENT).all()
    text = torch.full((int(to[F]) + 256,), 0xAB, dtype=torch.uint8, device=DEV)
    _lib.call(DEV, "opb_anno2d_text_write", *args, int(items.max()), 2, cap, kp, de, sc, pairs, F * cap, ws2, toff, text)
    tb = text.cpu().numpy()
    assert (tb[to[F]:] == 0xAB).all()
    for f, (_, p) in enumerate(images):
        n = len(p)
        a = ar.assign_pairs(p, gmap)
        assert tb[to[f]:to[f + 1]].tobytes() == ar.anno_text(feats[0][f, :n], feats[1][f, :, :n], feats[2][f, :n], a).encode()


def test_busy_caller_stream(tmp_path):
    c, images, result, feats = fixture_inputs(256)
    s = torch.cuda.Stream(DEV)
    with torch.cuda.stream(s):
        torch.cuda._sleep(200_000_000)             # the caller's stream is still busy when the calls are made
        fd = device_features(*feats)
        mats, num = sfm.assign_matrices(result, images, fd)
        sfm.save_anno_2d(tmp_path / "anno", [str(tmp_path / n) for n, _ in images], result, images, fd)
    assert np.array_equal(np.concatenate(mats, axis=1), c["assign"])
    assert open(tmp_path / "anno" / "anno_2d.json", "rb").read().count(b"anno_id") == int((c["num_matches"] > 0).sum())


def test_refusals(tmp_path):
    images, result, feats = dense_case(2, 2, 8192, 50)
    kp, de, sc = feats
    big = {"keypoints": torch.zeros(2, 8193, 2, device=DEV), "descriptors": torch.zeros(2, 2, 8193, device=DEV),
           "scores": torch.zeros(2, 8193, device=DEV)}
    with pytest.raises(_lib.OpbError, match="cap <= OPB_SFM_ASSIGN_MAX_CAP"):
        sfm.assign_matrices(result, images, big)
    with pytest.raises(ValueError, match="max_chunk_bytes"):
        sfm.save_anno_2d(tmp_path, [n for n, _ in images], result, images, device_features(kp, de, sc), max_chunk_bytes=1000)
    with pytest.raises(ValueError, match="image paths"):
        sfm.save_anno_2d(tmp_path, ["a.png"], result, images, device_features(kp, de, sc))
    with pytest.raises(ValueError, match="group_ids"):
        sfm.assign_matrices({"group_ids": np.zeros(0, np.int64), "group_offsets": np.zeros(1, np.int64)}, images, device_features(kp, de, sc))
