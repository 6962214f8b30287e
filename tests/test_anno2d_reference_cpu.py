"""The 2D annotation files without a GPU: the pair model against the reference's fixture (tests/golden/make_anno2d.py), the
planted defects that must break it, the library's float formatter -- the code the device runs, compiled for the host --
against Python's float.__repr__, and the argument checks of the new entry points."""
import ctypes as C
import hashlib
import json
import os

import numpy as np
import pytest

from onepose_b200 import _lib
from tests import anno2d_reference as ar

FIXTURE = os.path.join(os.path.dirname(__file__), "golden", "pnp_anno2d_cases.npz")
DIMS = (1, 256)


def case(D):
    z = np.load(FIXTURE)
    return {k[len(f"d{D}_"):]: z[k] for k in z.files if k.startswith(f"d{D}_")}


def model_pairs(c, **defect):
    gmap = ar.group_map(c["group_ids"], c["group_offsets"])
    return [ar.assign_pairs(c["pid"][f, :c["counts"][f]], gmap, **defect) for f in range(len(c["counts"]))]


@pytest.mark.parametrize("D", DIMS)
def test_model_equals_fixture(D):
    c = case(D)
    pairs = model_pairs(c)
    assert np.array_equal(np.array([p.shape[1] for p in pairs]), c["num_matches"])
    assert np.array_equal(np.concatenate(pairs, axis=1), c["assign"])
    assert (c["num_matches"] == 0).any() and (c["group_ids"] > 2 ** 31).any()


@pytest.mark.parametrize("D", DIMS)
@pytest.mark.parametrize("defect", [{"first_wins": True}, {"dedup": False}])
def test_defects_break_equality(D, defect):
    c = case(D)
    assert not np.array_equal(np.concatenate(model_pairs(c, **defect), axis=1), c["assign"])


@pytest.mark.parametrize("D", DIMS)
def test_text_and_index_equal_fixture(D):
    c = case(D)
    kp, de, sc = ar.features(int(c["seed"]), len(c["counts"]), D, c["pid"].shape[1])
    index = []
    for f, p in enumerate(model_pairs(c)):
        n = int(c["counts"][f])
        if p.shape[1] == 0:
            assert c["sha256"][f] == ""
            continue
        text = ar.anno_text(kp[f, :n], de[f, :, :n], sc[f, :n], p)
        assert hashlib.sha256(text.encode()).hexdigest() == c["sha256"][f]
        name = str(c["names"][f])
        index.append({"anno_id": len(index) + 1, "anno_file": os.path.join(os.path.dirname(os.path.dirname(name)), "anno_superpoint",
                                                                           os.path.basename(name).replace(".png", ".json")),
                      "img_file": name, "pose_file": name.replace("/color/", "/poses_ba/").replace(".png", ".txt")})
    assert json.dumps(index).encode() == c["index"].tobytes()


def stratified_floats(seed=0, per_exponent=31 * 1024) -> np.ndarray:
    """2^24 fp32 values: every biased exponent 0..254 with random significands and both signs, integers up to 2^24, the
    notation edges 1e-4 and 1e16 with 64 neighbours each side, powers of two and +-0."""
    rng = np.random.default_rng(seed)
    parts = []
    for be in range(255):
        m = rng.integers(0, 1 << 23, 2 * per_exponent, dtype=np.uint32)
        s = np.repeat(np.array([0, 1], np.uint32), per_exponent)
        parts.append((s << 31) | (np.uint32(be) << 23) | m)
    ints = np.concatenate([np.arange(0, 1 << 16), rng.integers(1 << 16, (1 << 24) + 1, 1 << 17)]).astype(np.float32)
    parts.append(ints.view(np.uint32))
    for edge in (1e-4, 1e16):
        b = np.array([edge], np.float32).view(np.uint32)[0]
        parts.append(np.arange(int(b) - 64, int(b) + 65, dtype=np.uint32))
    parts.append((np.arange(1, 255, dtype=np.uint32) << 23))
    parts.append(np.array([0, 1 << 31, 1, 0x807fffff], np.uint32))
    bits = np.concatenate(parts)
    bits = np.concatenate([bits, rng.integers(0, 0x7f800000, (1 << 24) - bits.size, dtype=np.uint32)])
    return bits.view(np.float32)


def python_repr(x: np.ndarray) -> np.ndarray:
    """json.dump's text of each widened value as NUL-padded 24-byte records (the formatter's output layout)."""
    special = {float("inf"): "Infinity", float("-inf"): "-Infinity"}
    return np.array([special.get(v, "NaN" if v != v else repr(v)) for v in x.astype(np.float64).tolist()], dtype="S24")


def host_repr(x: np.ndarray) -> np.ndarray:
    x = np.ascontiguousarray(x, np.float32)
    out = np.zeros((x.size, 24), np.uint8)
    ln = np.zeros(x.size, np.int32)
    _lib.check(_lib.load().opb_json_float_repr_host(x.ctypes.data, x.size, out.ctypes.data, ln.ctypes.data))
    assert np.array_equal(ln, np.char.str_len(out.view("S24").ravel()))
    return out.view("S24").ravel()


def test_float_repr_stratified():
    x = stratified_floats()
    assert x.size == 1 << 24
    for i in range(0, x.size, 1 << 21):
        got, want = host_repr(x[i:i + (1 << 21)]), python_repr(x[i:i + (1 << 21)])
        bad = np.nonzero(got != want)[0]
        assert bad.size == 0, [(float(x[i + j]), got[j], want[j]) for j in bad[:5]]


def test_float_repr_nonfinite_and_edges():
    x = np.array([np.inf, -np.inf, np.nan, -np.nan, 0.0, -0.0, 1e-4, 1e16, 1e-5, 123.0, 0.1, 2.0 ** -149, 3.4028235e38], np.float32)
    got = host_repr(x)
    assert got[:6].tolist() == [b"Infinity", b"-Infinity", b"NaN", b"NaN", b"0.0", b"-0.0"]
    assert got[9:11].tolist() == [b"123.0", b"0.10000000149011612"]
    assert np.array_equal(got, python_repr(x))


def _refused(name, *args, text):
    lib = _lib.load()
    rc = getattr(lib, name)(*args)
    assert rc == -1
    assert text in lib.opb_last_error(None).decode()
    with pytest.raises(_lib.OpbError, match=name):
        _lib.check(rc)


P = 64


def test_assign_refusals():
    b = C.c_int64()
    _refused("opb_sfm_assign_workspace_bytes", 2, 8193, C.byref(b), text="cap <= OPB_SFM_ASSIGN_MAX_CAP")
    _refused("opb_sfm_assign_pairs", P, P, 2, 8193, P, P, 10, P, 1 << 30, P, P, P, None, text="cap <= OPB_SFM_ASSIGN_MAX_CAP")
    _refused("opb_sfm_assign_pairs", P, P, 2, 64, P, P, 0, P, 1 << 30, P, P, P, None, text="M > 0")
    _refused("opb_sfm_assign_pairs", P, P, 2, 64, P, P, 10, P, 1 << 30, P, P, P, None, text="((uintptr_t)workspace & 255) == 0")
    _refused("opb_sfm_assign_pairs", P, P, 2, 64, P, P, 10, 256, 100, P, P, P, None, text="workspace_bytes >=")
    _refused("opb_sfm_assign_pairs", P, None, 2, 64, P, P, 10, P, 1 << 30, P, P, P, None, text="point3d_ids && counts")


def test_text_refusals():
    args = dict(images=P, item_off=P, Fc=1, items=100, max_items=100, D=4, cap=8, kp=P, de=P, sc=P, pairs=P, stride=8, ws=P,
                ws_bytes=1 << 20, offsets=P, stream=None)

    def lengths(**kw):
        a = dict(args)
        a.update(kw)
        return tuple(a.values())

    _refused("opb_anno2d_text_lengths", *lengths(max_items=(1 << 24) + 1), text="max_items <= OPB_ANNO2D_MAX_IMAGE_ITEMS")
    _refused("opb_anno2d_text_lengths", *lengths(Fc=65536), text="Fc <= 65535")
    _refused("opb_anno2d_text_lengths", *lengths(ws_bytes=8), text="workspace_bytes >=")
    _refused("opb_anno2d_text_lengths", *lengths(items=50), text="items >= max_items")
    _refused("opb_anno2d_text_write", P, P, 1, 100, 4, 8, P, P, P, P, 8, P, P, None, None, text="offsets && out")
    _refused("opb_json_float_repr_host", None, 4, P, P, text="x && out && len")
