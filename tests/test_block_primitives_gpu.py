"""The block-wide primitives of csrc/block.cuh on their own (opb_debug_block): block_reduce, block_scan forward and reverse and
block_rank, for every operator and element type the library uses, at every block size the header accepts (each multiple of
32 from 32 to 1024), against numpy integer arithmetic exactly.  One block walks one or three tiles with the same shared
scratch, as the library's tile loops do, and every thread's value and total is checked, not only thread 0's.

The patterns are the ones a warp- or block-level mistake shows on: random values, all-identity tiles, one non-identity value
at lanes 0 and 31 of the first, a middle and the last warp, INT32_MIN / INT32_MAX under Max and Min, negative and past-2^32
values under the signed 64-bit sum, and Sum64's wrap modulo 2^64.  Signed 32-bit overflow is undefined, so the Sum32 values
stay far below it."""
import numpy as np
import pytest
import torch

from onepose_b200 import _lib

OPB_E_INVALID = -1
P = 64                      # a non-null address; never dereferenced (the call is refused first)
I32_MIN, I32_MAX = int(np.iinfo(np.int32).min), int(np.iinfo(np.int32).max)
THREADS = list(range(32, 1025, 32))
REDUCE, SCAN, RANK = 0, 1, 2
# op -> (name, numpy dtype, numpy ufunc, identity)
OPS = {0: ("Sum32", np.int32, np.add, 0), 1: ("Max", np.int32, np.maximum, I32_MIN), 2: ("Min", np.int32, np.minimum, I32_MAX),
       3: ("Sum64", np.uint64, np.add, 0), 4: ("SumS64", np.int64, np.add, 0)}


def _positions(n):
    """Lanes 0 and 31 of the first, a middle and the last warp of an n-thread block."""
    mid = (n // 32) // 2
    return sorted({0, 31, 32 * mid, 32 * mid + 31, n - 32, n - 1})


def _patterns(op, n, rs):
    """The tiles every operator goes through: random, all-identity, and one non-identity value at each of _positions(n)."""
    _, dt, _, ident = OPS[op]
    if op == 0:
        rand, single = [rs.randint(-(1 << 20), 1 << 20, n)], [-123457]
    elif op in (1, 2):
        x = rs.randint(I32_MIN, I32_MAX, n, dtype=np.int64)
        u = rs.rand(n)
        x[u < 0.1], x[u > 0.9] = I32_MIN, I32_MAX
        lone = [I32_MAX if op == 1 else I32_MIN]                 # the extreme alone among identities
        rand, single = [x, np.full(n, lone[0]), np.where(np.arange(n) % 2, I32_MIN, I32_MAX)], [-5 if op == 1 else 5, lone[0]]
    elif op == 3:
        big = rs.randint(0, 1 << 62, n, dtype=np.int64).astype(np.uint64) * np.uint64(4) + rs.randint(0, 4, n).astype(np.uint64)
        rand, single = [big, np.full(n, np.iinfo(np.uint64).max, np.uint64)], [(1 << 63) + 3]    # every sum wraps
    else:
        rand = [rs.randint(-(1 << 52), 1 << 52, n, dtype=np.int64),
                (1 << 32) + rs.randint(-(1 << 31), 1 << 31, n, dtype=np.int64)]              # carries past bit 31
        single = [-((1 << 40) + 5)]
    out = [np.asarray(x).astype(dt) for x in rand] + [np.full(n, ident, dt)]
    for v in single:
        for p in _positions(n):
            x = np.full(n, ident, dt)
            x[p] = dt(v)
            out.append(x)
    return out


def _groups(pats, tiles):
    """Each pattern alone (tiles = 1), or every pattern once in consecutive stacks of three (tiles = 3)."""
    if tiles == 1:
        return [p[None] for p in pats]
    return [np.stack([pats[(i + k) % len(pats)] for k in range(3)]) for i in range(0, len(pats), 3)]


def _run(prim, op, x, reverse=0):
    """opb_debug_block on x [tiles, threads] -> (value, total) [tiles, threads] in x's dtype; the outputs start as a sentinel."""
    tiles, n = x.shape
    wide = x.dtype.itemsize == 8
    inp = torch.from_numpy(np.ascontiguousarray(x).view(np.int64 if wide else np.int32)).cuda()
    value = torch.full_like(inp, 0x5A5A5A5A)
    total = torch.full_like(inp, 0x5A5A5A5A)
    _lib.call(torch.device("cuda"), "opb_debug_block", prim, op, reverse, n, tiles, inp, value, total)
    return value.cpu().numpy().view(x.dtype), total.cpu().numpy().view(x.dtype)


def _exclusive(ufunc, ident, x, reverse):
    """numpy's exclusive scan of each row of x in x's dtype, from the last entry when reverse."""
    y = x[:, ::-1] if reverse else x
    inc = ufunc.accumulate(y, axis=1, dtype=x.dtype)
    exc = np.concatenate([np.full((x.shape[0], 1), ident, x.dtype), inc[:, :-1]], axis=1)
    return exc[:, ::-1] if reverse else exc


@pytest.mark.gpu
@pytest.mark.parametrize("tiles", [1, 3])
@pytest.mark.parametrize("threads", THREADS)
def test_reduce_and_both_scans_equal_numpy(threads, tiles):
    rs = np.random.RandomState(threads * 10 + tiles)
    for op, (name, dt, uf, ident) in OPS.items():
        for x in _groups(_patterns(op, threads, rs), tiles):
            whole = np.broadcast_to(uf.reduce(x, axis=1, dtype=dt)[:, None], x.shape)
            value, total = _run(REDUCE, op, x)
            assert np.array_equal(value, whole) and np.array_equal(total, whole), (name, "reduce", x[:, :4])
            for reverse in (0, 1):
                value, total = _run(SCAN, op, x, reverse)
                assert np.array_equal(value, _exclusive(uf, ident, x, reverse)), (name, "scan", reverse, x[:, :4])
                assert np.array_equal(total, whole), (name, "scan total", reverse)


def _keep_patterns(n, rs):
    """none, all, alternating, the first thread only, the last thread only, one warp full (the first, a middle, the last) with
    the rest empty, and random flags whose kept entries are any nonzero value."""
    ar = np.arange(n)
    mid = (n // 32) // 2
    pats = [np.zeros(n), np.ones(n), ar % 2, (ar + 1) % 2, ar == 0, ar == n - 1]
    pats += [(ar >= 32 * w) & (ar < 32 * w + 32) for w in sorted({0, mid, n // 32 - 1})]
    pats.append(np.where(rs.rand(n) < 0.3, rs.randint(-5, 6, n) | 1, 0))
    return [np.asarray(p).astype(np.int32) for p in pats]


@pytest.mark.gpu
@pytest.mark.parametrize("tiles", [1, 3])
@pytest.mark.parametrize("threads", THREADS)
def test_rank_equals_numpy(threads, tiles):
    rs = np.random.RandomState(threads * 10 + tiles)
    for x in _groups(_keep_patterns(threads, rs), tiles):
        kept = (x != 0).astype(np.int32)
        value, total = _run(RANK, 0, x)
        assert np.array_equal(value, np.cumsum(kept, axis=1, dtype=np.int32) - kept), x
        assert np.array_equal(total, np.broadcast_to(kept.sum(1, dtype=np.int32)[:, None], x.shape)), x


# (prim, op, reverse, threads, tiles, in, value, total) of a refused call, and the text of the refused condition
REFUSALS = [
    ((SCAN, 0, 0, 256, 1, None, P, P), "in && value && total"),
    ((SCAN, 0, 0, 256, 1, P, None, P), "in && value && total"),
    ((SCAN, 0, 0, 256, 1, P, P, None), "in && value && total"),
    ((SCAN, 0, 0, 0, 1, P, P, P), "threads >= 32"),
    ((SCAN, 0, 0, 16, 1, P, P, P), "threads >= 32"),
    ((SCAN, 0, 0, 33, 1, P, P, P), "threads % 32 == 0"),
    ((SCAN, 0, 0, 1000, 1, P, P, P), "threads % 32 == 0"),
    ((SCAN, 0, 0, 1056, 1, P, P, P), "threads <= 1024"),
    ((SCAN, 0, 0, 256, 0, P, P, P), "tiles > 0"),
    ((3, 0, 0, 256, 1, P, P, P), "prim <= 2"),
    ((-1, 0, 0, 256, 1, P, P, P), "prim >= 0"),
    ((SCAN, 5, 0, 256, 1, P, P, P), "op <= 4"),
    ((REDUCE, -1, 0, 256, 1, P, P, P), "op >= 0"),
    ((RANK, 1, 0, 256, 1, P, P, P), "prim != 2 || op == 0"),
    ((REDUCE, 0, 1, 256, 1, P, P, P), "reverse == 0 || (prim == 1 && reverse == 1)"),
    ((RANK, 0, 1, 256, 1, P, P, P), "reverse == 0 || (prim == 1 && reverse == 1)"),
    ((SCAN, 0, 2, 256, 1, P, P, P), "reverse == 0 || (prim == 1 && reverse == 1)"),
]


@pytest.mark.parametrize("args,cond", REFUSALS, ids=[f"{i}:{c[1]}" for i, c in enumerate(REFUSALS)])
def test_a_refused_call_names_the_hook_and_its_condition(args, cond):
    """The argument checks run before any CUDA call: these need no GPU, and no kernel is launched."""
    lib = _lib.load()
    assert lib.opb_debug_block(*args, None) == OPB_E_INVALID
    for msg in (lib.opb_last_error(None), lib.opb_sp_last_error(None)):
        assert msg.startswith(b"opb_debug_block: ") and cond.encode() in msg, (cond, msg)
