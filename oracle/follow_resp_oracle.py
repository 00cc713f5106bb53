"""ctypes front-end of the oracle of the responses that reach a follower or a candidate (oracle/follow_resp_oracle.c).

TEST INFRASTRUCTURE ONLY, like oracle.py.  follow_resp_oracle.c is part of libraft_oracle.so; lib() declares its
functions on oracle.lib().
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import follow_term_oracle as FT
from oracle import leader_term_oracle as LT
from oracle import oracle as O
from oracle import read_oracle as RO
from oracle import vote_request_oracle as VR

CANDIDATE, PRE_CANDIDATE = 0x10, 0x20  # the table's flags (RAFTGPU_VOTER_CANDIDATE, RAFTGPU_VOTER_PRE_CANDIDATE)
STEPPED = 0x8                          # raftgpu_follower_term_wire's step-down nibble (RAFTGPU_FTERM_STEPPED)

_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        L = O.lib()
        LT.lib()
        vp, sz, u64 = C.c_void_p, C.c_size_t, C.c_uint64
        args = [C.POINTER(O.ArenaView), C.POINTER(RO.Queues), vp, vp, vp, sz, u64, vp, vp, vp]
        L.frp_batch.argtypes, L.frp_batch.restype = args, None
        L.frp_bench.argtypes, L.frp_bench.restype = args, C.c_double
        L.frp_literal.argtypes = [C.POINTER(O.ArenaView), C.POINTER(RO.Queues), vp, vp, vp, vp, vp, vp, sz, u64, vp, vp,
                                  vp, vp]
        L.frp_literal.restype = None
        L.frp_term_batch.argtypes = [C.POINTER(O.ArenaView), C.POINTER(RO.Queues), vp, vp, vp, sz, u64, vp, vp, vp, vp, vp,
                                     vp]
        L.frp_term_batch.restype = None
        _lib = L
    return _lib


def _common(c, q, votes, blob, offsets, n_bytes):
    assert votes.dtype == np.uint8 and votes.shape == (O.SLOTS, c.cap) and votes.flags.c_contiguous
    blob = np.ascontiguousarray(blob, dtype=np.uint8)
    offsets = np.ascontiguousarray(offsets, dtype=np.uint32)
    qq = q._q() if q is not None else None
    return blob, offsets, len(offsets) - 1, O.wire_n_bytes(blob, n_bytes), O.view(c), qq


def batch(c, q, votes, blob, offsets, voters, bench: bool = False, n_bytes=None):
    """frp_batch over columns c (changed in place, as the arena is), read queues q (RO.ReadQueues or None) and votes
    ([SLOTS][cap] u8) with the caller's table voters (VR.VOTER_DTYPE per group slot) -> (status u8[n], out u64[n]);
    with bench=True also seconds."""
    blob, offsets, n, nb, v, qq = _common(c, q, votes, blob, offsets, n_bytes)
    vt = np.ascontiguousarray(voters, dtype=VR.VOTER_DTYPE)
    assert len(vt) >= c.n_groups
    status, out = np.zeros(n, np.uint8), np.zeros(n, np.uint64)
    f = lib().frp_bench if bench else lib().frp_batch
    secs = f(C.byref(v), C.byref(qq) if qq is not None else None, votes.ctypes.data, blob.ctypes.data, offsets.ctypes.data,
             n, nb, vt.ctypes.data, status.ctypes.data, out.ctypes.data)
    return (status, out, secs) if bench else (status, out)


def literal(c, q, votes, role, leader, voters, blob, offsets, n_bytes=None):
    """frp_literal: the frames one at a time as the reference steps them at a Follower, PreCandidate or Candidate.  c,
    q, votes, role (u8 per group slot), leader (u64 per group slot) and voters (VR.VOTER_DTYPE, contiguous) change in
    place -> (outcome u8[n], response blob, response offsets u32[responses + 1], totals u64[2])."""
    blob, offsets, n, nb, v, qq = _common(c, q, votes, blob, offsets, n_bytes)
    assert voters.dtype == VR.VOTER_DTYPE and voters.flags.c_contiguous and len(voters) >= c.n_groups
    assert role.dtype == np.uint8 and role.flags.c_contiguous and len(role) >= c.n_groups
    assert leader.dtype == np.uint64 and leader.flags.c_contiguous and len(leader) >= c.n_groups
    outcome = np.zeros(n, np.uint8)
    resp, roff, totals = np.zeros(max(16, n * FT.FRAME_MAX), np.uint8), np.zeros(n + 1, np.uint32), np.zeros(2, np.uint64)
    lib().frp_literal(C.byref(v), C.byref(qq) if qq is not None else None, votes.ctypes.data, role.ctypes.data,
                      leader.ctypes.data, voters.ctypes.data, blob.ctypes.data, offsets.ctypes.data, n, nb,
                      outcome.ctypes.data, resp.ctypes.data, roff.ctypes.data, totals.ctypes.data)
    return outcome, resp[: int(totals[1])].copy(), roff[: int(totals[0]) + 1].copy(), totals


def term_batch(c, q, votes, blob, offsets, voters, n_bytes=None):
    """frp_term_batch: raftgpu_follower_term_wire's batch form with the candidate's step-down, over columns c (changed in
    place), read queues q and votes with the caller's table voters -> (status u8[n], out u64[n][2], response blob,
    response offsets u32[responses + 1], totals u64[2]), as FT.batch."""
    blob, offsets, n, nb, v, qq = _common(c, q, votes, blob, offsets, n_bytes)
    vt = np.ascontiguousarray(voters, dtype=VR.VOTER_DTYPE)
    assert len(vt) >= c.n_groups
    status, out = np.zeros(n, np.uint8), np.zeros((n, 2), np.uint64)
    resp, roff, totals = np.zeros(max(16, n * FT.FRAME_MAX), np.uint8), np.zeros(n + 1, np.uint32), np.zeros(2, np.uint64)
    lib().frp_term_batch(C.byref(v), C.byref(qq) if qq is not None else None, votes.ctypes.data, blob.ctypes.data,
                         offsets.ctypes.data, n, nb, vt.ctypes.data, status.ctypes.data, out.ctypes.data, resp.ctypes.data,
                         roff.ctypes.data, totals.ctypes.data)
    return status, out, resp[: int(totals[1])].copy(), roff[: int(totals[0]) + 1].copy(), totals
