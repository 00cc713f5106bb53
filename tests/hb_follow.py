"""Helpers for the follower heartbeat tests: frame headers read and rewritten in place (the transport's part: a leader's
(group << 4 | slot) becomes the follower's (group << 4 | x) and back), selection bitmaps, and the columns the pass may
write."""
import numpy as np

from helpers import B

GROUP_STATE = ("committed", "last_index", "term", "term_start", "meta")


def headers(blob, offsets) -> np.ndarray:
    """The u32 LE header of every frame."""
    o = np.asarray(offsets[:-1], dtype=np.int64)
    b = np.asarray(blob, dtype=np.uint32)
    return b[o] | (b[o + 1] << 8) | (b[o + 2] << 16) | (b[o + 3] << 24)


def with_headers(blob, offsets, hdrs) -> np.ndarray:
    """A copy of blob with every frame's header replaced by hdrs."""
    out = np.array(blob, dtype=np.uint8, copy=True)
    o = np.asarray(offsets[:-1], dtype=np.int64)
    h = np.asarray(hdrs, dtype=np.uint32)
    for k in range(4):
        out[o + k] = (h >> (8 * k)) & 0xFF
    return out


def bitmap(bits) -> np.ndarray:
    """u32 words from group 0 of a bool per group slot (padded to whole words)."""
    bits = np.asarray(bits, dtype=bool)
    pad = np.zeros((-len(bits)) % 32, dtype=bool)
    return np.packbits(np.concatenate([bits, pad]), bitorder="little").view(np.uint32).copy()


def frames_of(blob, offsets):
    """[(header, body bytes)] of a blob."""
    return [(int.from_bytes(bytes(blob[lo:lo + 4]), "little"), bytes(blob[lo + 4:hi]))
            for lo, hi in zip(np.asarray(offsets[:-1]).tolist(), np.asarray(offsets[1:]).tolist())]


def state(c, n):
    """The group columns of groups [0, n) (what the pass may write), copied."""
    return {k: getattr(c, k)[:n].copy() for k in GROUP_STATE}


def same_state(x, y) -> bool:
    return all(np.array_equal(x[k], y[k]) for k in GROUP_STATE)


def self_ids(rng, n):
    """Random Raft ids for n followers, a few of them 0, 128 and 2^64 - 1."""
    ids = rng.integers(1, 1 << 63, n, dtype=np.uint64)
    k = rng.random(n)
    ids[k < 0.03] = 0
    ids[(k > 0.03) & (k < 0.06)] = (1 << 64) - 1
    ids[(k > 0.06) & (k < 0.09)] = 128
    return ids


def group_state(a, n):
    """The group columns the follower passes write (and meta, which they leave alone) of groups [0, n)."""
    c = a.read_columns(n)
    return {"committed": c.committed, "last_index": c.last_index, "term_start": c.term_start,
            "term": a.column_read(B.COL_TERM, 0, 0, n, np.uint64), "meta": c.meta}
