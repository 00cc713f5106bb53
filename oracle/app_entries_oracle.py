"""ctypes front-end of the follower MsgAppend-with-entries oracle (oracle/app_entries_oracle.c).

TEST INFRASTRUCTURE ONLY, like oracle.py.  app_entries_oracle.c is part of libraft_oracle.so; lib() declares its
functions on oracle.lib().
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import app_follow_oracle as AF
from oracle import oracle as O

APPENDED = 0x8
APPENDED_DTYPE = np.dtype([("first_index", "<u8"), ("last_index", "<u8"), ("run_start", "<u8"), ("run_term", "<u8"),
                           ("span_off", "<u4"), ("span_len", "<u4")])
assert APPENDED_DTYPE.itemsize == 40
ENTRY_DTYPE = np.dtype([("term", "<u8"), ("index", "<u8"), ("off", "<u4"), ("end", "<u4"), ("ld", "<u4"),
                        ("reserved", "<u4")])


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        L = AF.lib()
        u64, vp, sz = C.c_uint64, C.c_void_p, C.c_size_t
        L.aeo_decode.argtypes = [vp, sz, C.POINTER(O.WireMessage), vp, sz, C.POINTER(sz)]
        L.aeo_decode.restype = C.c_int
        from oracle import read_oracle as RO
        args = [C.POINTER(O.ArenaView), C.POINTER(RO.Queues), vp, vp, vp, sz, u64, vp, vp, vp, vp, vp, vp]
        L.aeo_batch.argtypes, L.aeo_batch.restype = args, None
        L.aeo_bench.argtypes, L.aeo_bench.restype = args, C.c_double
        _lib = L
    return _lib


def decode(raw: bytes):
    """aeo_decode: None when raw (or one of its Entries) is not a well-formed message, else (WireMessage, [entries as
    ENTRY_DTYPE rows: term, index, off, end (from the Message's start), ld])."""
    m, n = O.WireMessage(), C.c_size_t()
    cap = 4096
    ents = np.zeros(cap, ENTRY_DTYPE)
    buf = (C.c_uint8 * max(1, len(raw))).from_buffer_copy(raw or b"\0")
    if not lib().aeo_decode(buf, len(raw), C.byref(m), ents.ctypes.data, cap, C.byref(n)):
        return None
    assert n.value <= cap
    return m, ents[: n.value].copy()


def batch(c, q, logs, blob, offsets, bench: bool = False, n_bytes=None):
    """aeo_batch over columns c (changed in place, as the arena is), read queues q (RO.ReadQueues or None) and the
    caller's table logs (AF.LOG_DTYPE per group slot; its runs change in place) -> (status u8[n], from u64[n], appended
    APPENDED_DTYPE[n], response blob, response offsets u32[responses + 1], totals u64[2]); with bench=True also
    seconds."""
    blob = np.ascontiguousarray(blob, dtype=np.uint8)
    offsets = np.ascontiguousarray(offsets, dtype=np.uint32)
    assert logs.dtype == AF.LOG_DTYPE and logs.flags.c_contiguous and len(logs) >= c.n_groups
    n = len(offsets) - 1
    status, frm, app = np.zeros(n, np.uint8), np.zeros(n, np.uint64), np.zeros(n, APPENDED_DTYPE)
    resp, roff, totals = np.zeros(max(16, n * AF.FRAME_MAX), np.uint8), np.zeros(n + 1, np.uint32), np.zeros(2, np.uint64)
    v = O.view(c)
    qq = q._q() if q is not None else None
    f = lib().aeo_bench if bench else lib().aeo_batch
    secs = f(C.byref(v), C.byref(qq) if qq is not None else None, logs.ctypes.data, blob.ctypes.data, offsets.ctypes.data,
             n, O.wire_n_bytes(blob, n_bytes), status.ctypes.data, frm.ctypes.data, app.ctypes.data, resp.ctypes.data,
             roff.ctypes.data, totals.ctypes.data)
    res = (status, frm, app, resp[: int(totals[1])].copy(), roff[: int(totals[0]) + 1].copy(), totals)
    return res + (secs,) if bench else res
