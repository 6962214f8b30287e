"""Host side of the multi-object detection (detect.boxes_from_matches_objects / detect_from_matches_objects / ObjectDetectors,
crop.crop_frames(..., frame_index)): the C entry points' refusals, the argument checks that run before the library is called,
and the pair table against a numpy model.  No GPU: the library call is replaced by a recorder."""
import numpy as np
import pytest
import torch

from onepose_b200 import _lib, crop, detect

OPB_E_INVALID = -1
P = 64                      # a non-null address; never dereferenced (the call is refused first)
CPU = torch.device("cpu")


def _refused(name, args, cond):
    lib = _lib.load()
    assert getattr(lib, name)(*args, None) == OPB_E_INVALID
    msg = lib.opb_last_error(None)
    assert msg.startswith(name.encode() + b": ") and cond.encode() in msg, msg


def _objects_args(**kw):
    a = dict(n_views=3, cap_ref=16, V_max=2, n_query=1, cap_query=16, matches_int64=1, B=1, query_h=480, query_w=640)
    a.update(kw)
    return (P, P, P, a["n_views"], a["cap_ref"], P, P, a["V_max"], P, P, a["n_query"], a["cap_query"], P, P, a["matches_int64"], a["B"],
            a["query_h"], a["query_w"], P, P, P, P, P)


@pytest.mark.parametrize("kw,cond", [(dict(n_views=0), "n_views > 0"), (dict(V_max=257), "V_max <= opb::kMaxViews"),
                                     (dict(V_max=0), "V_max > 0"), (dict(cap_ref=8193), "cap_ref <= opb::kMaxRefPoints"),
                                     (dict(n_query=0), "n_query > 0"), (dict(B=0), "B > 0"), (dict(matches_int64=2), "matches_int64 == 1"),
                                     (dict(query_w=0), "query_w > 0")])
def test_boxes_from_matches_objects_refusals(kw, cond):
    _refused("opb_boxes_from_matches_objects", _objects_args(**kw), cond)


def test_null_pointers_and_crop_refusals():
    args = list(_objects_args())
    args[5] = None                                                              # view_first
    _refused("opb_boxes_from_matches_objects", tuple(args), "view_first && view_count")
    crop_args = [P, 100, 10, 2, 10, 10, P, 3, P, P, 16, P, P, P, P]
    _refused("opb_crop_resize_indexed", tuple(crop_args[:6] + [None] + crop_args[7:]), "frame_index && box")
    _refused("opb_crop_resize_indexed", tuple(crop_args[:3] + [0] + crop_args[4:]), "n_frames > 0")
    _refused("opb_crop_resize_indexed", tuple(crop_args[:7] + [65536] + crop_args[8:]), "B <= 65535")
    _refused("opb_crop_resize_indexed", tuple(crop_args[:10] + [12] + crop_args[11:]), "crop_size % 8 == 0")


def pair_table_numpy(pairs, views):
    """The model: per pair its frame, and its object's first view and view count."""
    arr = np.asarray(pairs, np.int64).reshape(-1, 2)
    first = np.array([views[o][0] for o in arr[:, 1]])
    count = np.array([views[o][1] for o in arr[:, 1]])
    return arr[:, 0], first, count


def test_pair_table_against_numpy():
    rng = np.random.default_rng(0)
    for _ in range(20):
        ids = rng.choice(1000, int(rng.integers(1, 12)), replace=False)
        counts = rng.integers(1, 40, len(ids))
        first = np.cumsum(np.concatenate([[0], counts[:-1]]))
        views = {int(i): (int(f), int(c)) for i, f, c in zip(ids, first, counts)}
        F = int(rng.integers(1, 9))
        pairs = [(int(rng.integers(0, F)), int(rng.choice(ids))) for _ in range(int(rng.integers(1, 30)))]
        got = detect.pair_table(pairs, F, views)
        for g, w in zip(got, pair_table_numpy(pairs, views)):
            assert g.dtype == np.int32 and np.array_equal(g, w)
    views = {3: (0, 2), 7: (2, 5)}
    for bad in ([], [(0, 4)], [(2, 3)], [(-1, 3)]):
        with pytest.raises(ValueError):
            detect.pair_table(bad, 2, views)


class _Stub:
    """A table of two objects' views, as ObjectDetectors.table builds it, without a device."""

    def __init__(self):
        self.ref = {"keypoints": torch.zeros(2, 5, 2), "counts": torch.tensor([5, 3], dtype=torch.int32), "sizes": torch.full((2, 2), 64, dtype=torch.int32)}
        self.views = [{}, {}]


def test_object_registry():
    det = detect.ObjectDetectors(extractor=None, matcher=None, device="cpu")
    with pytest.raises(ValueError, match="no object registered"):
        det.table()
    with pytest.raises(ValueError, match="unknown object id"):
        det.remove_object(0)
    det._objects = {0: _Stub(), 4: _Stub(), 2: _Stub()}
    refs, views = det.table()
    assert views == {0: (0, 2), 2: (2, 2), 4: (4, 2)} and tuple(refs["keypoints"].shape) == (6, 5, 2)
    assert refs["counts"].tolist() == [5, 3] * 3
    det.remove_object(2)
    assert det.table()[1] == {0: (0, 2), 4: (2, 2)}


@pytest.fixture
def recorder(monkeypatch):
    calls = []
    monkeypatch.setattr(_lib, "cuda_device", lambda t: CPU)
    monkeypatch.setattr(_lib, "call", lambda dev, name, *args: calls.append((name, args)))
    return calls


def _inputs(B=3, V_max=4, cap=16, n_views=9, F=2):
    refs = {"keypoints": torch.zeros(n_views, cap, 2), "counts": torch.full((n_views,), cap), "sizes": torch.full((n_views, 2), 64)}
    query = {"keypoints": torch.zeros(F, 20, 2), "counts": torch.full((F,), 20)}
    return dict(refs=refs, view_first=[0, 4, 4][:B], view_count=[4, 2, 2][:B], query=query, query_index=[1, 0, 1][:B],
                matches0=torch.zeros(B, V_max, cap, dtype=torch.int64), query_size=(480, 640))


def test_checks_before_the_library_call(recorder):
    detect.boxes_from_matches_objects(**_inputs())
    name, args = recorder.pop()
    assert name == "opb_boxes_from_matches_objects"
    assert [args[k] for k in (3, 4, 7, 10, 11, 14, 15, 16, 17)] == [9, 16, 4, 2, 20, 1, 3, 480, 640]
    assert args[5].dtype == args[6].dtype == args[12].dtype == torch.int32 and args[12].tolist() == [1, 0, 1]
    big = detect.boxes_from_matches_objects(**{**_inputs(), "query_index": torch.tensor([1, 5, -9], dtype=torch.int64),
                                               "view_first": torch.tensor([0, 1 << 40, 4])})
    assert big is not None
    _, args = recorder.pop()
    assert args[12].tolist() == [1, 2, -1] and args[5].tolist() == [0, 9, 4]         # clamped, never wrapped into range
    bad = [dict(matches0=torch.zeros(3, 4, 15, dtype=torch.int64)), dict(matches0=torch.zeros(3, 257, 16, dtype=torch.int64)),
           dict(matches0=torch.zeros(3, 4, 16)), dict(matches0=torch.zeros(0, 4, 16, dtype=torch.int64)), dict(view_first=[0, 1]),
           dict(view_count=[1.0, 2.0, 3.0]), dict(query_index=torch.zeros(3, 1, dtype=torch.int32)), dict(query_size=(480, 0)),
           dict(query={"keypoints": torch.zeros(2, 20, 2), "counts": torch.zeros(3)})]
    for kw in bad:
        with pytest.raises(ValueError):
            detect.boxes_from_matches_objects(**{**_inputs(), **kw})
    assert not recorder


def test_affine_budgets_reach_the_library_as_int32_or_are_refused(recorder):
    """maxIters and refineIters cross into the library as int32: 2**31 - 1 passes unchanged, anything above is refused rather than
    wrapped (2**32 + 5 would otherwise run 5 iterations, and 2**31 arrive negative)."""
    f, offs = torch.zeros(4, 2), torch.tensor([0, 4], dtype=torch.int32)
    detect.affine_partial_batch(f, f, offs, max_iters=2**31 - 1, refine_iters=2**31 - 1)
    name, args = recorder.pop()
    assert name == "opb_estimate_affine_partial" and args[5] == args[7] == 2**31 - 1
    for kw in (dict(max_iters=2**31), dict(max_iters=2**32 + 5), dict(refine_iters=2**31), dict(refine_iters=2**32 + 1), dict(max_iters=-1)):
        with pytest.raises(ValueError, match="2\\*\\*31 - 1"):
            detect.affine_partial_batch(f, f, offs, **kw)
    assert not recorder


def test_crop_and_detect_checks_before_the_library_call(recorder):
    frames = torch.zeros(2, 48, 64, dtype=torch.uint8)
    K = torch.eye(3, dtype=torch.float64)
    boxes = torch.zeros(3, 4, dtype=torch.int32)
    crop.crop_frames(frames, boxes, K, 16, frame_index=[1, 0, 1])
    name, args = recorder.pop()
    assert name == "opb_crop_resize_indexed" and args[3:6] == (2, 48, 64) and args[6].tolist() == [1, 0, 1] and args[7] == 3
    crop.crop_frames(frames, boxes[:2], K, 16)
    assert recorder.pop()[0] == "opb_crop_resize"
    for kw in (dict(frame_index=[0, 1]), dict(frame_index=[[0, 1, 1]]), dict(frame_index=[True, False, True]), dict(frame_index=[])):
        with pytest.raises(ValueError):
            crop.crop_frames(frames, boxes, K, 16, **kw)
    inp = _inputs()
    for kw in (dict(crop_size=12), dict(K=torch.eye(3, dtype=torch.float64)[None].expand(2, 3, 3))):
        a = dict(frames_u8=frames, frame_index=[1, 0, 1], K=K, refs=inp["refs"], view_first=inp["view_first"], view_count=inp["view_count"],
                 query=inp["query"], matches0=inp["matches0"])
        with pytest.raises(ValueError):
            detect.detect_from_matches_objects(**{**a, **kw})
    with pytest.raises(ValueError):
        detect.detect_from_matches_objects(frames[:1], [0, 0, 0], K, inp["refs"], inp["view_first"], inp["view_count"], inp["query"], inp["matches0"])
    assert not recorder
    detect.detect_from_matches_objects(frames, [1, 0, 1], K, inp["refs"], inp["view_first"], inp["view_count"], inp["query"], inp["matches0"], 16)
    assert [c[0] for c in recorder] == ["opb_boxes_from_matches_objects", "opb_crop_resize_indexed"]
