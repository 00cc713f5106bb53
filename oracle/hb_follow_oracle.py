"""ctypes front-end of the follower heartbeat oracle (oracle/hb_follow_oracle.c).

TEST INFRASTRUCTURE ONLY, like oracle.py.  hb_follow_oracle.c is part of libraft_oracle.so; lib() declares its functions
on oracle.lib().
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import oracle as O
from oracle import read_oracle as RO

FRAME_MAX = 60  # 4-byte header + at most 56 bytes of Message
WIRE_ROLE, WIRE_COMMIT_RANGE = 7, 8


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        L = O.lib()
        u64, vp, sz = C.c_uint64, C.c_void_p, C.c_size_t
        L.hfl_encode_response.argtypes, L.hfl_encode_response.restype = [u64, u64, u64, u64, vp, vp], sz
        args = [C.POINTER(O.ArenaView), C.POINTER(RO.Queues), vp, vp, sz, u64, vp, vp, vp, vp, vp, vp, vp]
        L.hfl_follower_heartbeats.argtypes, L.hfl_follower_heartbeats.restype = args, None
        L.hfl_bench.argtypes, L.hfl_bench.restype = args, C.c_double
        _lib = L
    return _lib


def encode_response(to: int, frm: int, term: int, commit: int, context: bytes | None = None) -> bytes:
    """hfl_encode_response: the serialized MsgHeartbeatResponse; context None or 8 bytes."""
    assert context is None or len(context) == 8
    buf = (C.c_uint8 * 64)()
    ctx = None if context is None else (C.c_uint8 * 8).from_buffer_copy(context)
    k = lib().hfl_encode_response(to, frm, term, commit, ctx, buf)
    return bytes(buf[:k])


def follower_heartbeats(c, q, blob, offsets, select, self_ids, bench: bool = False, n_bytes=None):
    """hfl_follower_heartbeats over columns c (c.term = Raft::term of each group; changed in place, as the arena is)
    and read queues q (RO.ReadQueues, or None for an arena without them) -> (status u8[n], from u64[n], response blob,
    response offsets u32[responses + 1], totals u64[2]); with bench=True also the pass's seconds.
    n_bytes as in O.wire_decode_batch."""
    blob = np.ascontiguousarray(blob, dtype=np.uint8)
    offsets = np.ascontiguousarray(offsets, dtype=np.uint32)
    sel = np.ascontiguousarray(select, dtype=np.uint32)
    ids = np.ascontiguousarray(self_ids, dtype=np.uint64)
    assert len(sel) * 32 >= c.n_groups and len(ids) >= c.n_groups
    n = len(offsets) - 1
    status, frm = np.zeros(n, np.uint8), np.zeros(n, np.uint64)
    resp, roff, totals = np.zeros(max(16, n * FRAME_MAX), np.uint8), np.zeros(n + 1, np.uint32), np.zeros(2, np.uint64)
    v = O.view(c)
    qq = q._q() if q is not None else None
    f = lib().hfl_bench if bench else lib().hfl_follower_heartbeats
    secs = f(C.byref(v), C.byref(qq) if qq is not None else None, blob.ctypes.data, offsets.ctypes.data, n,
             O.wire_n_bytes(blob, n_bytes), sel.ctypes.data, ids.ctypes.data, status.ctypes.data, frm.ctypes.data,
             resp.ctypes.data, roff.ctypes.data, totals.ctypes.data)
    out = (status, frm, resp[: int(totals[1])].copy(), roff[: int(totals[0]) + 1].copy(), totals)
    return out + (secs,) if bench else out
