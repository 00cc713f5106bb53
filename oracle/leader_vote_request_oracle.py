"""ctypes front-end of the leader vote-request oracle (oracle/leader_vote_request_oracle.c).

TEST INFRASTRUCTURE ONLY, like oracle.py.  leader_vote_request_oracle.c is part of libraft_oracle.so; lib() declares
its functions on oracle.lib().  The literal form it is checked against is vote_request_oracle.literal.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import oracle as O
from oracle import read_oracle as RO
from oracle import vote_request_oracle as VR

_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        L = VR.lib()
        vp, sz, u64 = C.c_void_p, C.c_size_t, C.c_uint64
        args = [C.POINTER(O.ArenaView), C.POINTER(RO.Queues), vp, vp, vp, sz, u64, vp, vp, vp, vp, vp, vp]
        L.lvro_batch.argtypes, L.lvro_batch.restype = args, None
        L.lvro_bench.argtypes, L.lvro_bench.restype = args, C.c_double
        _lib = L
    return _lib


def batch(c, q, votes, blob, offsets, voters, bench: bool = False, n_bytes=None):
    """lvro_batch over columns c (changed in place, as the arena is), read queues q (RO.ReadQueues or None) and votes
    ([SLOTS][cap] u8) with the caller's table voters (VR.VOTER_DTYPE per group slot) -> (status u8[n], out u64[n][2],
    response blob, response offsets u32[responses + 1], totals u64[2]); with bench=True also seconds.  n_bytes as in
    O.wire_decode_batch."""
    blob, offsets, n, nb, resp, roff, totals, v, qq = VR._common(c, q, votes, blob, offsets, n_bytes)
    vt = np.ascontiguousarray(voters, dtype=VR.VOTER_DTYPE)
    assert len(vt) >= c.n_groups
    status, out = np.zeros(n, np.uint8), np.zeros((n, 2), np.uint64)
    f = lib().lvro_bench if bench else lib().lvro_batch
    secs = f(C.byref(v), C.byref(qq) if qq is not None else None, votes.ctypes.data, blob.ctypes.data, offsets.ctypes.data,
             n, nb, vt.ctypes.data, status.ctypes.data, out.ctypes.data, resp.ctypes.data, roff.ctypes.data,
             totals.ctypes.data)
    res = (status, out, resp[: int(totals[1])].copy(), roff[: int(totals[0]) + 1].copy(), totals)
    return res + (secs,) if bench else res
