"""ctypes front-end of the heartbeat-frame oracle (oracle/hb_frames_oracle.c).

TEST INFRASTRUCTURE ONLY, like oracle.py.  hb_frames_oracle.c is part of libraft_oracle.so; lib() declares its functions
on oracle.lib().
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import oracle as O
from oracle import read_oracle as RO

FRAME_MAX = 60  # 4-byte header + at most 56 bytes of Message


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        L = O.lib()
        u64, vp = C.c_uint64, C.c_void_p
        L.hfo_encode_heartbeat.argtypes, L.hfo_encode_heartbeat.restype = [u64, u64, u64, u64, u64, vp], C.c_size_t
        L.hfo_bcast_heartbeats.argtypes = [C.POINTER(O.ArenaView), C.POINTER(RO.Queues), C.c_uint32, C.c_uint32, vp, vp,
                                           vp, vp, vp]
        L.hfo_bcast_heartbeats.restype = None
        _lib = L
    return _lib


def encode_heartbeat(to: int, frm: int, term: int, commit: int, ctx: int = 0) -> bytes:
    """hfo_encode_heartbeat: the serialized MsgHeartbeat; ctx 0 = no context."""
    buf = (C.c_uint8 * 64)()
    k = lib().hfo_encode_heartbeat(to, frm, term, commit, ctx, buf)
    return bytes(buf[:k])


def bcast_heartbeats(c, q, first: int, n: int, ids: np.ndarray, select: np.ndarray | None = None):
    """hfo_bcast_heartbeats over columns c (c.term = Raft::term of each group) and read queues q (RO.ReadQueues, or None
    for an arena without them); ids u64 [9][n] -> (blob u8[], offsets u32[frames + 1], totals u64[3])."""
    ids = np.ascontiguousarray(ids, dtype=np.uint64)
    assert ids.shape == (O.SLOTS + 1, n)
    sel = None if select is None else np.ascontiguousarray(select, dtype=np.uint32)
    blob = np.zeros(max(16, n * O.SLOTS * FRAME_MAX), np.uint8)
    offsets = np.zeros(n * O.SLOTS + 1, np.uint32)
    totals = np.zeros(3, np.uint64)
    v = O.view(c)
    qq = q._q() if q is not None else None
    lib().hfo_bcast_heartbeats(C.byref(v), C.byref(qq) if qq is not None else None, first, n,
                               None if sel is None else sel.ctypes.data, ids.ctypes.data, blob.ctypes.data,
                               offsets.ctypes.data, totals.ctypes.data)
    return blob[: int(totals[1])].copy(), offsets[: int(totals[0]) + 1].copy(), totals
