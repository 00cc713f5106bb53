"""Arenas for the MsgAppend-frame tests (raftgpu_append_frames, oracle/app_frames_oracle.c): random leaders whose peers
fall on every branch of maybe_send_append -- paused in each state, a requested snapshot, entries to send, next_idx - 1
below term_start, and caught up at or above last_index + 1 -- with next_idx near and far from matched, so that the
offset codec's escapes occur; and the frames of a blob decoded back."""
import numpy as np

from helpers import B, O
from oracle import hb_wire_oracle as H
import read_cases as R

U64 = (1 << 64) - 1
TERMS = np.array([1, 127, 128, 1 << 32, 1 << 40, 1 << 63, U64], np.uint64)


def random_columns(rng, n, n_wide, cap=None, base=None):
    """Host columns of n group slots: narrow groups [0, n - 2 n_wide), then n_wide wide pairs; c.term set.  base: the
    leaders' term_start values (default: small and large)."""
    c = O.new_columns(cap or n + 64, n)
    shape = (O.SLOTS, n)
    inc = rng.integers(1, 256, n)
    inc[rng.random(n) < 0.4] = 0x1F
    out = np.where(rng.random(n) < 0.2, rng.integers(0, 256, n), 0)
    learn = np.where(rng.random(n) < 0.3, rng.integers(0, 256, n), 0) & ~(inc | out)
    self_slot = rng.integers(0, 8, n)
    has_self = rng.random(n) < 0.9
    meta = inc | out << 8 | learn << 16 | np.where(has_self, self_slot << 24 | B.META_HAS_SELF, 0)
    lo = np.arange(n - 2 * n_wide, n, 2)
    meta[lo] |= R.META_WIDE_LO
    meta[lo + 1] = (meta[lo + 1] & ~(0xF << 24) & ~B.META_HAS_SELF) | R.META_WIDE_HI
    c.meta[:n] = meta.astype(np.uint32)
    if base is None:
        base = np.where(rng.random(n) < 0.8, rng.integers(1, 1000, n), rng.integers(1, 1 << 62, n, dtype=np.int64))
    ts = np.asarray(base, np.uint64)
    last = ts + rng.choice(np.array([0, 1, 3, 40], np.uint64), n)
    below = rng.random(n) < 0.05                                     # a state no real leader has: last_index < term_start
    last[below] = ts[below] - np.minimum(ts[below], 1)
    c.term_start[:n] = np.where(rng.random(n) < 0.85, ts, np.uint64(U64))
    c.last_index[:n] = last
    c.committed[:n] = last - rng.integers(0, 3, n).astype(np.uint64) * (last > 3)
    c.term[:n] = np.where(rng.random(n) < 0.06, 0, TERMS[rng.integers(0, len(TERMS), n)])
    # next_idx around last_index + 1 (caught up), below it (entries), below term_start (the log's term), and 0
    lastp = np.broadcast_to(last, shape).astype(np.uint64)
    d = rng.choice(np.array([1, 1, 1, 2, 7, 0, -1, -5], np.int64), shape)
    nx = np.maximum(lastp.astype(np.int64) + d, 0).astype(np.uint64)
    deep = rng.random(shape) < 0.05
    nx[deep] = rng.integers(0, 2, deep.sum()).astype(np.uint64)
    c.next_idx[:, :n] = nx
    gap = rng.choice(np.array([1, 1, 2, 100, 40_000, 1 << 20], np.uint64), shape)
    c.matched[:, :n] = np.where(nx > gap, nx - gap, 0)
    zero = rng.random(shape) < 0.03                                  # Raft::reset's matched 0: next_idx escapes
    c.matched[:, :n][zero] = 0
    c.peer_committed[:, :n] = c.matched[:, :n]
    state = rng.choice(np.array([0, 1, 2], np.uint8), shape, p=[0.45, 0.45, 0.1])
    c.pflags[:, :n] = state | np.where(rng.random(shape) < 0.2, B.PF_PAUSED, 0).astype(np.uint8) \
        | np.where(rng.random(shape) < 0.15, B.PF_INS_FULL, 0).astype(np.uint8)
    c.pending_request_snapshot[:, :n] = np.where(rng.random(shape) < 0.05, rng.integers(1, 1 << 40, shape), 0)
    return c


def ids_for(rng, n):
    ids = rng.integers(1, 1 << 63, (9, n), dtype=np.uint64)
    k = rng.random((9, n))
    ids[k < 0.05] = 0
    ids[(k > 0.05) & (k < 0.1)] = U64
    ids[(k > 0.1) & (k < 0.15)] = 128
    return ids


def select_bits(rng, cap, density):
    bits = rng.random((cap + 31) // 32 * 32) < density
    return np.packbits(bits, bitorder="little").view(np.uint32).copy()


def frames_of(blob, offsets):
    """[(group, slot, decoded message)] of a frame blob."""
    out = []
    for lo, hi in zip(offsets[:-1].tolist(), offsets[1:].tolist()):
        hdr = int.from_bytes(bytes(blob[lo:lo + 4]), "little")
        m = H.decode_message(bytes(blob[lo + 4:hi]))
        assert m is not None
        out.append((hdr >> 4, hdr & 15, m))
    return out


def frame_cells(blob, offsets):
    """{(group, slot)} of the frames' headers."""
    return [(int.from_bytes(bytes(blob[lo:lo + 4]), "little") >> 4, int.from_bytes(bytes(blob[lo:lo + 4]), "little") & 15)
            for lo in offsets[:-1].tolist()]


def sending_groups(c, n, first=0):
    """bool [n]: group slots [first, first + n) whose leader (the low half's) sends: a leader with a term."""
    g = np.arange(first, first + n)
    lo = np.where(c.meta[g] & R.META_WIDE_HI, g - 1, g)
    return (c.term_start[lo] != np.uint64(U64)) & (c.term[lo] != 0)


def send_list_of_senders(c, first, n, select):
    """The oracle's send list for the selection, restricted to the groups that send (the send list itself does not
    look at roles or terms)."""
    sl = O.arena_send_list(c, select, first, n)
    ok = sending_groups(c, n, first)
    return sl[ok[sl["group"].astype(np.int64) - first]] if len(sl) else sl
