"""next_idx and peer_committed are stored on the device as 32-bit offsets from the cell's matched, with an escape to
the exact u64 value (k_common.cuh).  Column IO must stay lossless at the edges of the offset range and across writes
of matched, in whichever order the columns are written."""
import numpy as np
import pytest

from helpers import B

pytestmark = pytest.mark.gpu

I32_MIN, I32_MAX = -(2 ** 31), 2 ** 31 - 1
U64 = 2 ** 64


def edge_values(matched):
    """Values around the representable window [matched + INT32_MIN + 1, matched + INT32_MAX] (mod 2^64)."""
    out = []
    for m in matched:
        m = int(m)
        ds = [0, 1, -1, I32_MAX, I32_MAX + 1, I32_MIN + 1, I32_MIN, I32_MIN - 1, 2 ** 40, -(2 ** 40)]
        out.append([(m + d) % U64 for d in ds])
    return np.array(out, dtype=np.uint64)


def test_offset_columns_round_trip_at_the_edges_and_across_matched_writes():
    rng = np.random.default_rng(7)
    base = np.array([0, 1, 2 ** 31, 2 ** 32 - 1, 2 ** 48, U64 - 1, U64 - 2 ** 31], dtype=np.uint64)
    vals = edge_values(base)                      # [len(base), 10]
    n = vals.size
    matched = np.repeat(base, vals.shape[1])
    nxt = vals.reshape(-1)
    pc = nxt[rng.permutation(n)]
    arena = B.Arena(n)
    try:
        assert arena.group_alloc_range(n) == 0
        for s in range(B.SLOTS):
            arena.column_write(B.COL_MATCHED, s, 0, matched)
            arena.column_write(B.COL_NEXT_IDX, s, 0, nxt)
            arena.column_write(B.COL_PEER_COMMITTED, s, 0, pc)
        for s in range(B.SLOTS):
            assert np.array_equal(arena.column_read(B.COL_NEXT_IDX, s, 0, n, np.uint64), nxt)
            assert np.array_equal(arena.column_read(B.COL_PEER_COMMITTED, s, 0, n, np.uint64), pc)
        # a new matched keeps both values, whether they were escaped before, after, or both
        new_m = rng.integers(0, 2 ** 63, n, dtype=np.uint64)
        new_m[::3] = nxt[::3]                     # offset 0 after the write
        new_m[1::5] = 0
        arena.column_write(B.COL_MATCHED, 3, 0, new_m)
        assert np.array_equal(arena.column_read(B.COL_MATCHED, 3, 0, n, np.uint64), new_m)
        assert np.array_equal(arena.column_read(B.COL_NEXT_IDX, 3, 0, n, np.uint64), nxt)
        assert np.array_equal(arena.column_read(B.COL_PEER_COMMITTED, 3, 0, n, np.uint64), pc)
        # a partial range leaves its neighbours alone
        arena.column_write(B.COL_NEXT_IDX, 3, 5, nxt[:7][::-1].copy())
        want = nxt.copy()
        want[5:12] = nxt[:7][::-1]
        assert np.array_equal(arena.column_read(B.COL_NEXT_IDX, 3, 0, n, np.uint64), want)
        assert np.array_equal(arena.column_read(B.COL_PEER_COMMITTED, 3, 0, n, np.uint64), pc)
    finally:
        arena.close()
