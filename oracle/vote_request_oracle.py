"""ctypes front-end of the vote-request oracle (oracle/vote_request_oracle.c).

TEST INFRASTRUCTURE ONLY, like oracle.py.  vote_request_oracle.c is part of libraft_oracle.so; lib() declares its
functions on oracle.lib().
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import oracle as O
from oracle import read_oracle as RO

FRAME_MAX = 64  # 4-byte header + at most 59 bytes of Message
WIRE_ROLE, WIRE_COMMIT_VOTE, WIRE_IGNORED = 7, 9, 10
SELECT, LEADER, LEASE, CHECK_QUORUM = 0x1, 0x2, 0x4, 0x100
GRANTED, VOTED, BUMPED = 0x1, 0x2, 0x4
FOLLOWER, PRE_CANDIDATE, CANDIDATE, LEADER_ROLE = range(4)
VOTER_DTYPE = np.dtype([("id", "<u8"), ("vote", "<u8"), ("last_term", "<u8"), ("commit_term", "<u8"),
                        ("persisted", "<u8"), ("priority", "<u8"), ("flags", "<u4"), ("reserved", "<u4"),
                        ("reserved2", "<u8")])


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        L = O.lib()
        u32, u64, vp, sz = C.c_uint32, C.c_uint64, C.c_void_p, C.c_size_t
        L.vro_encode_response.argtypes, L.vro_encode_response.restype = [u32, u64, u64, u64, u64, C.c_int, u64, vp], sz
        args = [C.POINTER(O.ArenaView), C.POINTER(RO.Queues), vp, vp, vp, sz, u64, vp, vp, vp, vp, vp, vp]
        L.vro_batch.argtypes, L.vro_batch.restype = args, None
        L.vro_bench.argtypes, L.vro_bench.restype = args, C.c_double
        L.vro_literal.argtypes = [C.POINTER(O.ArenaView), C.POINTER(RO.Queues), vp, vp, vp, vp, vp, sz, u64, vp, vp,
                                 vp]
        L.vro_literal.restype = None
        _lib = L
    return _lib


def encode_response(msg_type, to, frm, term, commit=0, reject=False, commit_term=0) -> bytes:
    """vro_encode_response: a vote response's serialized Message (no header)."""
    buf = (C.c_uint8 * 64)()
    k = lib().vro_encode_response(msg_type, to, frm, term, commit, int(reject), commit_term, buf)
    return bytes(buf[:k])


def _common(c, q, votes, blob, offsets, n_bytes):
    assert votes.dtype == np.uint8 and votes.shape == (O.SLOTS, c.cap) and votes.flags.c_contiguous
    blob = np.ascontiguousarray(blob, dtype=np.uint8)
    offsets = np.ascontiguousarray(offsets, dtype=np.uint32)
    n = len(offsets) - 1
    resp, roff, totals = np.zeros(max(16, n * FRAME_MAX), np.uint8), np.zeros(n + 1, np.uint32), np.zeros(2, np.uint64)
    v = O.view(c)
    qq = q._q() if q is not None else None
    return blob, offsets, n, O.wire_n_bytes(blob, n_bytes), resp, roff, totals, v, qq


def batch(c, q, votes, blob, offsets, voters, bench: bool = False, n_bytes=None):
    """vro_batch over columns c (c.term = Raft::term; changed in place, as the arena is), read queues q (RO.ReadQueues
    or None) and votes ([SLOTS][cap] u8) with the caller's table voters (VOTER_DTYPE per group slot) -> (status u8[n],
    out u64[n][2], response blob, response offsets u32[responses + 1], totals u64[2]); with bench=True also seconds.
    n_bytes as in O.wire_decode_batch."""
    blob, offsets, n, nb, resp, roff, totals, v, qq = _common(c, q, votes, blob, offsets, n_bytes)
    vt = np.ascontiguousarray(voters, dtype=VOTER_DTYPE)
    assert len(vt) >= c.n_groups
    status, out = np.zeros(n, np.uint8), np.zeros((n, 2), np.uint64)
    f = lib().vro_bench if bench else lib().vro_batch
    secs = f(C.byref(v), C.byref(qq) if qq is not None else None, votes.ctypes.data, blob.ctypes.data, offsets.ctypes.data,
             n, nb, vt.ctypes.data, status.ctypes.data, out.ctypes.data, resp.ctypes.data, roff.ctypes.data, totals.ctypes.data)
    res = (status, out, resp[: int(totals[1])].copy(), roff[: int(totals[0]) + 1].copy(), totals)
    return res + (secs,) if bench else res


def literal(c, q, votes, role, voters, blob, offsets, n_bytes=None):
    """vro_literal: the frames one at a time as the reference steps them.  c, q, votes, role (u8 per group slot) and
    voters (VOTER_DTYPE, a contiguous array: its vote and flags change) change in place -> (response blob, response
    offsets u32[responses + 1], totals u64[2]).  n_bytes as in O.wire_decode_batch."""
    blob, offsets, n, nb, resp, roff, totals, v, qq = _common(c, q, votes, blob, offsets, n_bytes)
    assert voters.dtype == VOTER_DTYPE and voters.flags.c_contiguous and len(voters) >= c.n_groups
    assert role.dtype == np.uint8 and role.flags.c_contiguous and len(role) >= c.n_groups
    lib().vro_literal(C.byref(v), C.byref(qq) if qq is not None else None, votes.ctypes.data, role.ctypes.data,
                      voters.ctypes.data, blob.ctypes.data, offsets.ctypes.data, n, nb, resp.ctypes.data, roff.ctypes.data,
                      totals.ctypes.data)
    return resp[: int(totals[1])].copy(), roff[: int(totals[0]) + 1].copy(), totals
