"""CPU checks of the several-objects-per-call interface: the new C entry points are declared in the header, bound in _lib and
exported by the library; the argument checks of opb_gather_matches_objects that fail before any device work; and the numpy
restatement of the mixed gather (used by the GPU tests) against the reference's masking expression frame by frame."""
import ctypes as C
import os
import re

import numpy as np

from onepose_b200 import _lib
from tests.test_multi_object_gpu import gather_objects_numpy

NEW_SYMBOLS = ("opb_add_object", "opb_remove_object", "opb_forward_objects", "opb_gather_matches_objects")
HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "onepose_b200.h")


def test_new_symbols_declared_bound_and_exported():
    with open(HEADER) as f:
        header = f.read()
    lib = _lib.load()
    for name in NEW_SYMBOLS:
        assert re.search(r"\bint " + name + r"\(", header), name
        assert name in _lib.SYMBOLS, name
        assert getattr(lib, name) is not None


def test_gather_matches_objects_rejects_bad_arguments():
    lib = _lib.load()
    buf = C.c_void_p(16)     # never dereferenced: every call below fails its argument check first

    def call(m0=buf, sc=None, kp2=buf, kp3=buf, first=buf, count=buf, B=2, N=4, p2=buf, p3=buf, mconf=None, qi=None, off=buf):
        return lib.opb_gather_matches_objects(m0, sc, kp2, kp3, first, count, B, N, p2, p3, mconf, qi, off, None)

    for kw in (dict(B=0), dict(B=-1), dict(N=-1), dict(off=None), dict(kp3=None), dict(first=None), dict(count=None), dict(m0=None),
               dict(kp2=None), dict(p2=None), dict(p3=None), dict(mconf=buf), dict(B=1 << 16, N=1 << 16)):
        assert call(**kw) == -1, kw


def test_mixed_gather_restatement_matches_reference_masking():
    """Per frame: valid = matches > -1; kpts2d[valid]; kpts3d_of_its_object[matches[valid]]; conf[valid]."""
    rs = np.random.RandomState(5)
    kp3 = {7: rs.randn(50, 3).astype(np.float32), 2: rs.randn(7000, 3).astype(np.float32), 9: rs.randn(1, 3).astype(np.float32)}
    for ids, N in (([7], 1), ([2, 7, 9, 7, 2], 37), ([9, 2, 2], 500), ([7, 9], 0)):
        B = len(ids)
        m0 = np.stack([np.where(rs.rand(N) < 0.4, rs.randint(0, len(kp3[i]), size=N), -1) for i in ids]).astype(np.int64).reshape(B, N)
        kp2 = rs.randn(B, N, 2).astype(np.float32)
        sc = rs.rand(B, N).astype(np.float32)
        g = gather_objects_numpy(m0, kp2, kp3, ids, sc)
        for b, oid in enumerate(ids):
            matches, kpts2d, confidence, kpts3d = m0[b], kp2[b], sc[b], kp3[oid]
            valid = matches > -1
            o0, o1 = g["offsets"][b], g["offsets"][b + 1]
            assert np.array_equal(g["pts2d"][o0:o1], kpts2d[valid].astype(np.float64))
            assert np.array_equal(g["pts3d"][o0:o1], kpts3d[matches[valid]].astype(np.float64))
            assert np.array_equal(g["mconf"][o0:o1], confidence[valid])
            assert np.array_equal(g["query_index"][o0:o1], np.nonzero(valid)[0])
        assert g["offsets"][0] == 0 and g["offsets"][-1] == len(g["pts2d"])
