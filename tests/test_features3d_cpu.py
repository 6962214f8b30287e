"""The rule the segmented means follow (no GPU): numpy's summation order for np.mean(x[s:e], axis=0), pinned on the numpy
installed here, and a Python twin of the kernel's np_pairwise_sum (onepose_b200/csrc/kernels_aux.cuh) that equals np.mean bit
for bit.  Planted defects in the twin -- no eight-way accumulators, the wrong split point, no identity add -- break that
equality, so the lengths and values below can tell a correct restatement from a subtly wrong one.

numpy's reduction loop runs along the axis with the smaller stride.  When that is the reduced axis (F-ordered [len, D], a
strided view of one, or D = 1) the loop is numpy's pairwise sum; otherwise each channel's running sum takes the rows in order.
Both start from the identity +0.0.  tests/test_features3d_gpu.py holds the device to numpy itself."""
from __future__ import annotations

import numpy as np
import pytest
import torch

from onepose_b200 import features3d

LENGTHS = list(range(1, 18)) + [63, 64, 65, 127, 128, 129, 135, 136, 137, 255, 256, 257, 1023, 1024, 1025, 8191, 8192, 8193, 20000]


def pairwise(a, n=None, blocks=8, split=lambda n: n // 2 - (n // 2) % 8):
    """numpy's pairwise sum of a 1-D run (the kernel's np_pairwise_sum); `blocks` / `split` plant defects."""
    n = len(a) if n is None else n
    if n < 8:
        res = 0.0
        for i in range(n):
            res += a[i]
        return res
    if n <= 128:
        r = [float(a[j]) for j in range(blocks)] + [0.0] * (8 - blocks)
        i = blocks
        while i < n - n % blocks:
            for j in range(blocks):
                r[j] += a[i + j]
            i += blocks
        res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
        while i < n:
            res += a[i]
            i += 1
        return res
    n2 = split(n)
    return pairwise(a[:n2], None, blocks, split) + pairwise(a[n2:], None, blocks, split)


def kernel_mean(a, identity=True, **defect):
    """The kernel's mean of one channel's contiguous track: (0.0 + pairwise) / n."""
    s = pairwise([float(v) for v in a], None, **defect)
    return (0.0 + s if identity else s) / len(a)


def sequential_mean(a):
    acc = 0.0
    for v in a:
        acc += float(v)
    return acc / len(a)


def wide(rs, *shape):
    """Values over ~40 binary orders of magnitude, both signs (make_track_scores' spread, signed): the order matters."""
    return rs.randn(*shape) * np.exp(3.0 * rs.randn(*shape))


def same(a, b):
    return np.asarray(a, np.float64).tobytes() == np.asarray(b, np.float64).tobytes()


# ------------------------------------------------------------------------------------------------ numpy's rule
LAYOUTS = {
    # name: (view of a base array -> [n, D], pairwise?)
    "C": (lambda rs, n, D: wide(rs, n, D), False),
    "F": (lambda rs, n, D: wide(rs, D, n).T, True),
    "row_strided": (lambda rs, n, D: wide(rs, 2 * n, D)[::2], False),
    "column_sliced": (lambda rs, n, D: wide(rs, n, D + 2)[:, 1:D + 1], False),
    "F_row_strided": (lambda rs, n, D: wide(rs, D, 2 * n).T[::2], True),
    "D1": (lambda rs, n, D: wide(rs, n, 1), True),
}


@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_numpy_sums_pairwise_exactly_along_a_contiguous_reduced_axis(layout):
    """np.mean(x, axis=0) equals the pairwise twin per channel where the reduced axis has the smaller stride, the rows-in-order
    sum otherwise -- and not the other one, at lengths where the two differ."""
    make, is_pairwise = LAYOUTS[layout]
    rs = np.random.RandomState(1)
    differ = 0
    for n in (9, 40, 130, 400, 9000):
        x = make(rs, n, 5)
        got = x.mean(axis=0)
        pw = [kernel_mean(x[:, c]) for c in range(x.shape[1])]
        sq = [sequential_mean(x[:, c]) for c in range(x.shape[1])]
        assert same(got, pw if is_pairwise else sq), (layout, n)
        differ += not same(pw, sq)
    assert differ >= 3, "the lengths do not tell the two orders apart"


@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_numpy_starts_from_positive_zero(layout):
    """An all -0.0 track averages to +0.0 in every layout and at every length: numpy adds its sum to the identity 0.0."""
    for n in (1, 7, 8, 9, 130):
        x = -np.abs(LAYOUTS[layout][0](np.random.RandomState(2), n, 3) * 0.0)
        assert np.signbit(x).all()
        assert not np.signbit(x.mean(axis=0)).any(), (layout, n)


def test_numpy_mean_of_fp32_stays_fp32():
    """np.mean of fp32 accumulates and returns fp32: why the device refuses fp32 instead of widening it."""
    assert np.ones((9, 3), np.float32).mean(axis=0).dtype == np.float32


# ------------------------------------------------------------------------------------------------ the twin
@pytest.mark.parametrize("n", LENGTHS)
def test_pairwise_twin_equals_numpy(n):
    rs = np.random.RandomState(n)
    for a in (wide(rs, n), rs.rand(n) * np.exp(3.0 * rs.randn(n))):
        assert same(kernel_mean(a), np.mean(a)), n


DEFECTS = {
    "no eight-way accumulators": dict(blocks=1),
    "four-way accumulators": dict(blocks=4),
    "split at n / 2": dict(split=lambda n: n // 2),
    "split one block late": dict(split=lambda n: n // 2 - (n // 2) % 8 + 8),
}


@pytest.mark.parametrize("defect", list(DEFECTS))
def test_planted_order_defect_breaks_equality(defect):
    """Each defect changes the result at some of the lengths above (and leaves short runs alone, where it has no effect)."""
    broken = []
    for n in LENGTHS:
        a = wide(np.random.RandomState(n), n)
        if not same(kernel_mean(a, **DEFECTS[defect]), np.mean(a)):
            broken.append(n)
    print(f"{defect}: differs from numpy at {len(broken)} of {len(LENGTHS)} lengths")
    assert broken and min(broken) >= 8


def test_planted_missing_identity_add_breaks_equality():
    """Without the 0.0 + the twin keeps -0.0 on all -0.0 tracks of 8 or more; numpy gives +0.0."""
    for n in (8, 9, 64, 130):
        z = -np.zeros(n)
        assert same(kernel_mean(z), np.mean(z)), n
        assert not same(kernel_mean(z, identity=False), np.mean(z)), n


# ------------------------------------------------------------------------------------------------ the wrapper's refusals
@pytest.mark.parametrize("fn", [features3d.mean_descriptors, features3d.mean_scores])
@pytest.mark.parametrize("make", [lambda: np.ones((9, 3), np.float32), lambda: torch.ones(9, 3), lambda: np.ones((9, 3), np.int64)])
def test_means_refuse_what_is_not_fp64(fn, make):
    """No silent widening: anything but fp64 is refused before the device is touched."""
    with pytest.raises(ValueError, match="fp64"):
        fn(make(), np.array([4, 5]))
