"""ctypes front-end of the MsgAppend-frame oracle (oracle/app_frames_oracle.c).

TEST INFRASTRUCTURE ONLY, like oracle.py.  app_frames_oracle.c is part of libraft_oracle.so; lib() declares its functions
on oracle.lib().
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import oracle as O
from oracle import read_oracle as RO

FRAME_MAX = 72  # 4-byte header + at most 68 bytes of Message


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        L = O.lib()
        u64, vp = C.c_uint64, C.c_void_p
        L.afo_encode_append.argtypes, L.afo_encode_append.restype = [u64, u64, u64, u64, u64, u64, vp], C.c_size_t
        L.afo_bcast_append.argtypes = [C.POINTER(O.ArenaView), C.POINTER(RO.Queues), C.c_uint32, C.c_uint32, vp, vp, vp,
                                       vp, vp, vp]
        L.afo_bcast_append.restype = None
        _lib = L
    return _lib


def encode_append(to: int, frm: int, term: int, log_term: int, index: int, commit: int) -> bytes:
    """afo_encode_append: the serialized entry-less MsgAppend."""
    buf = (C.c_uint8 * 80)()
    k = lib().afo_encode_append(to, frm, term, log_term, index, commit, buf)
    return bytes(buf[:k])


def bcast_append(c, q, first: int, n: int, ids: np.ndarray, select: np.ndarray | None = None):
    """afo_bcast_append over columns c (c.term = Raft::term of each group) and read queues q (RO.ReadQueues, or None for
    an arena without them); ids u64 [9][n] -> (blob u8[], offsets u32[frames + 1], rest O.SEND_ENTRY_DTYPE[],
    totals u64[4])."""
    ids = np.ascontiguousarray(ids, dtype=np.uint64)
    assert ids.shape == (O.SLOTS + 1, n)
    sel = None if select is None else np.ascontiguousarray(select, dtype=np.uint32)
    blob = np.zeros(max(16, n * O.SLOTS * FRAME_MAX), np.uint8)
    offsets = np.zeros(n * O.SLOTS + 1, np.uint32)
    rest = np.zeros(max(1, n * O.SLOTS), O.SEND_ENTRY_DTYPE)
    totals = np.zeros(4, np.uint64)
    v = O.view(c)
    qq = q._q() if q is not None else None
    lib().afo_bcast_append(C.byref(v), C.byref(qq) if qq is not None else None, first, n,
                           None if sel is None else sel.ctypes.data, ids.ctypes.data, blob.ctypes.data,
                           offsets.ctypes.data, rest.ctypes.data, totals.ctypes.data)
    return blob[: int(totals[1])].copy(), offsets[: int(totals[0]) + 1].copy(), rest[: int(totals[2])].copy(), totals
