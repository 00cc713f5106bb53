"""ctypes front-end of the leader term-prefix oracle (oracle/leader_term_oracle.c).

TEST INFRASTRUCTURE ONLY, like oracle.py.  leader_term_oracle.c is part of libraft_oracle.so; lib() declares its
functions on oracle.lib().
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import follow_term_oracle as FT
from oracle import oracle as O
from oracle import read_oracle as RO
from oracle import vote_request_oracle as VR

WIRE_IGNORED = 10
IGNORED = 4  # the literal form's outcome beyond FT.NONE, FT.PASS, FT.ANSWERED, FT.DROPPED

_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        L = O.lib()
        FT.lib()
        vp, sz, u64 = C.c_void_p, C.c_size_t, C.c_uint64
        args = [C.POINTER(O.ArenaView), C.POINTER(RO.Queues), vp, vp, vp, sz, u64, vp, vp, vp, vp, vp, vp]
        L.lto_batch.argtypes, L.lto_batch.restype = args, None
        L.lto_bench.argtypes, L.lto_bench.restype = args, C.c_double
        L.lto_literal.argtypes = [C.POINTER(O.ArenaView), C.POINTER(RO.Queues), vp, vp, vp, vp, vp, vp, sz, u64, vp, vp,
                                  vp, vp]
        L.lto_literal.restype = None
        _lib = L
    return _lib


def _common(c, q, votes, blob, offsets, n_bytes):
    assert votes.dtype == np.uint8 and votes.shape == (O.SLOTS, c.cap) and votes.flags.c_contiguous
    blob = np.ascontiguousarray(blob, dtype=np.uint8)
    offsets = np.ascontiguousarray(offsets, dtype=np.uint32)
    n = len(offsets) - 1
    resp, roff, totals = np.zeros(max(16, n * FT.FRAME_MAX), np.uint8), np.zeros(n + 1, np.uint32), np.zeros(2, np.uint64)
    qq = q._q() if q is not None else None
    return blob, offsets, n, O.wire_n_bytes(blob, n_bytes), resp, roff, totals, O.view(c), qq


def batch(c, q, votes, blob, offsets, voters, bench: bool = False, n_bytes=None):
    """lto_batch over columns c (changed in place, as the arena is), read queues q (RO.ReadQueues or None) and votes
    ([SLOTS][cap] u8) with the caller's table voters (VR.VOTER_DTYPE per group slot) -> (status u8[n], out u64[n][2],
    response blob, response offsets u32[responses + 1], totals u64[2]); with bench=True also seconds."""
    blob, offsets, n, nb, resp, roff, totals, v, qq = _common(c, q, votes, blob, offsets, n_bytes)
    vt = np.ascontiguousarray(voters, dtype=VR.VOTER_DTYPE)
    assert len(vt) >= c.n_groups
    status, out = np.zeros(n, np.uint8), np.zeros((n, 2), np.uint64)
    f = lib().lto_bench if bench else lib().lto_batch
    secs = f(C.byref(v), C.byref(qq) if qq is not None else None, votes.ctypes.data, blob.ctypes.data, offsets.ctypes.data,
             n, nb, vt.ctypes.data, status.ctypes.data, out.ctypes.data, resp.ctypes.data, roff.ctypes.data,
             totals.ctypes.data)
    res = (status, out, resp[: int(totals[1])].copy(), roff[: int(totals[0]) + 1].copy(), totals)
    return res + (secs,) if bench else res


def literal(c, q, votes, role, leader, voters, blob, offsets, n_bytes=None):
    """lto_literal: the frames one at a time as the reference steps them at a Leader or the Follower it became.  c, q,
    votes, role (u8 per group slot), leader (u64 per group slot) and voters (VR.VOTER_DTYPE, contiguous) change in place
    -> (outcome u8[n], response blob, response offsets u32[responses + 1], totals u64[2])."""
    blob, offsets, n, nb, resp, roff, totals, v, qq = _common(c, q, votes, blob, offsets, n_bytes)
    assert voters.dtype == VR.VOTER_DTYPE and voters.flags.c_contiguous and len(voters) >= c.n_groups
    assert role.dtype == np.uint8 and role.flags.c_contiguous and len(role) >= c.n_groups
    assert leader.dtype == np.uint64 and leader.flags.c_contiguous and len(leader) >= c.n_groups
    outcome = np.zeros(n, np.uint8)
    lib().lto_literal(C.byref(v), C.byref(qq) if qq is not None else None, votes.ctypes.data, role.ctypes.data,
                      leader.ctypes.data, voters.ctypes.data, blob.ctypes.data, offsets.ctypes.data, n, nb,
                      outcome.ctypes.data, resp.ctypes.data, roff.ctypes.data, totals.ctypes.data)
    return outcome, resp[: int(totals[1])].copy(), roff[: int(totals[0]) + 1].copy(), totals
