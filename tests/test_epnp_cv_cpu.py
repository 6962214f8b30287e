"""CPU checks of the confidence mode of EPnP-RANSAC (opb_ransac_epnp_cv): the symbol and its test hooks declared, bound and
exported, argument checks that fail before any CUDA call, and the Python option's validation."""
import ctypes as C
import inspect
import os

import pytest

from onepose_b200 import _lib, pnp

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "onepose_b200.h")
NEW_SYMBOLS = ("opb_ransac_epnp_cv", "opb_debug_set_cv_wave", "opb_debug_set_cv_trace", "opb_debug_cv_subsets")


def test_new_symbols_declared_bound_and_exported():
    header = open(HEADER).read()
    lib = _lib.load()
    for name in NEW_SYMBOLS:
        assert f"int {name}(" in header and name in _lib.SYMBOLS, name
        assert getattr(lib, name).restype is C.c_int


def test_entry_point_rejects_bad_arguments():
    lib = _lib.load()
    buf = C.c_void_p(16)     # never dereferenced: every call below fails its argument check first

    def call(K=buf, p2=buf, p3=buf, off=buf, B=2, H=64, thr=5.0, conf=0.99, ws=buf, pose=buf, mask=buf, cnt=buf, its=buf):
        return lib.opb_ransac_epnp_cv(K, p2, p3, off, B, H, thr, conf, ws, pose, mask, cnt, its, None)

    for kw in (dict(K=None), dict(p2=None), dict(p3=None), dict(off=None), dict(ws=None), dict(pose=None), dict(mask=None),
               dict(cnt=None), dict(its=None), dict(B=0), dict(H=0), dict(H=65535 * 128 + 1), dict(thr=0.0), dict(thr=float("nan")),
               dict(thr=-5.0), dict(thr=-float("inf")),
               dict(conf=-0.01), dict(conf=1.01), dict(conf=float("nan"))):
        assert call(**kw) == -1, kw
    assert lib.opb_debug_set_cv_wave(-1) == -1
    assert lib.opb_debug_set_cv_trace(buf, None, None, 0) == -1
    assert lib.opb_debug_set_cv_trace(None, None, None, 0) == 0
    assert lib.opb_debug_cv_subsets(4, 10, 10, buf, None) == -1
    assert lib.opb_debug_cv_subsets(6, 0, 10, buf, None) == -1
    assert lib.opb_debug_cv_subsets(6, 10, 0, buf, None) == -1


def test_confidence_option_is_checked_and_defaults_kept():
    for fn in (pnp.ransac_pnp_batch, pnp.poses_from_matches, pnp.poses_from_matches_objects, pnp.ransac_PnP):
        params = inspect.signature(fn).parameters
        assert params["confidence"].default is None and params["method"].default == "p3p", fn.__name__
    assert pnp._hypotheses("epnp", None, 0.99) == pnp.EPNP_HYPOTHESES
    for method, conf in (("p3p", 0.99), ("epnp", 1.5), ("epnp", -0.1), ("epnp", float("nan"))):
        with pytest.raises(ValueError):
            pnp._hypotheses(method, None, conf)
    with pytest.raises(ValueError):
        pnp.ransac_PnP([[600, 0, 256], [0, 600, 256], [0, 0, 1]], [[0, 0]] * 6, [[0, 0, 1]] * 6, confidence=0.99)
