"""ctypes front-end of the vote-response oracle (oracle/vote_wire_oracle.c).

TEST INFRASTRUCTURE ONLY, like oracle.py.  vote_wire_oracle.c is part of libraft_oracle.so; lib() declares its functions
on oracle.lib().
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import oracle as O

WIRE_ROLE, WIRE_COMMIT_VOTE = 7, 9
FOLLOWER, PRE_CANDIDATE, CANDIDATE, LEADER = range(4)
OUTCOME_DTYPE = np.dtype([("group", "<u4"), ("result", "<u4")])
NONE = 0xFFFFFFFF


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        L = O.lib()
        vp, sz = C.c_void_p, C.c_size_t
        L.vwo_batch.argtypes = [C.POINTER(O.ArenaView), vp, vp, vp, sz, C.c_uint64, vp, vp, vp, vp, C.POINTER(C.c_uint64),
                                C.POINTER(C.c_uint64)]
        L.vwo_batch.restype = None
        L.vwo_literal.argtypes, L.vwo_literal.restype = [C.POINTER(O.ArenaView), vp, vp, vp, vp, sz, C.c_uint64,
                                                             vp], None
        _lib = L
    return _lib


def _frames(blob, offsets):
    return np.ascontiguousarray(blob, dtype=np.uint8), np.ascontiguousarray(offsets, dtype=np.uint32)


def batch(c, votes, blob, offsets, select, pre=None, n_bytes=None):
    """vwo_batch over columns c (c.term = Raft::term; groups [0, c.n_groups) are the arena's) and votes ([SLOTS][cap] u8,
    changed in place) -> (status u8[n], outcomes OUTCOME_DTYPE[k], touched groups); n_bytes as in O.wire_decode_batch."""
    assert votes.dtype == np.uint8 and votes.shape == (O.SLOTS, c.cap) and votes.flags.c_contiguous
    blob, offsets = _frames(blob, offsets)
    sel = np.ascontiguousarray(select, dtype=np.uint32)
    pr = None if pre is None else np.ascontiguousarray(pre, dtype=np.uint32)
    assert len(sel) * 32 >= c.n_groups and (pr is None or len(pr) * 32 >= c.n_groups)
    n = len(offsets) - 1
    status, out = np.zeros(n, np.uint8), np.zeros(max(1, min(n, c.n_groups)), OUTCOME_DTYPE)
    k, t = C.c_uint64(), C.c_uint64()
    v = O.view(c)
    lib().vwo_batch(C.byref(v), votes.ctypes.data, blob.ctypes.data, offsets.ctypes.data, n,
                    O.wire_n_bytes(blob, n_bytes), sel.ctypes.data,
                    None if pr is None else pr.ctypes.data, status.ctypes.data, out.ctypes.data, C.byref(k), C.byref(t))
    return status, out[: k.value].copy(), t.value


def literal(c, votes, role, blob, offsets, n_bytes=None):
    """vwo_literal: the frames one at a time through step / step_candidate / poll and its transitions.  c, votes and
    role (u8 per group slot, FOLLOWER..LEADER; a pair's is its low half's) change in place -> first u32[n_groups]: the
    first Won or Lost word of each group, NONE where there was none.  n_bytes as in O.wire_decode_batch."""
    assert role.dtype == np.uint8 and len(role) >= c.n_groups and role.flags.c_contiguous
    blob, offsets = _frames(blob, offsets)
    first = np.full(max(1, c.n_groups), NONE, np.uint32)
    v = O.view(c)
    lib().vwo_literal(C.byref(v), votes.ctypes.data, role.ctypes.data, blob.ctypes.data, offsets.ctypes.data,
                      len(offsets) - 1, O.wire_n_bytes(blob, n_bytes), first.ctypes.data)
    return first[: c.n_groups]


def outcomes_of(first):
    """literal()'s first decided words as an outcome list in ascending group order."""
    g = np.flatnonzero(first != NONE).astype(np.uint32)
    out = np.zeros(len(g), OUTCOME_DTYPE)
    out["group"], out["result"] = g, first[g]
    return out
