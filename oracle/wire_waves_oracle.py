"""ctypes front-end of the wave oracle (oracle/wire_waves_oracle.c): the wire step and the follower's append passes at
raftgpu_arena_set_wire_waves > 1, as the existing batch forms repeated over the frames each run left DUP.

TEST INFRASTRUCTURE ONLY, like oracle.py.  wire_waves_oracle.c is part of libraft_oracle.so; lib() declares its
functions on oracle.lib().
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import oracle as O
from oracle import read_oracle as RO
from oracle import app_entries_oracle as AE
from oracle import app_follow_oracle as AF
from oracle import leader_runs_oracle as LR

_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        L = O.lib()
        u64, u32, vp, sz = C.c_uint64, C.c_uint32, C.c_void_p, C.c_size_t
        args = [C.POINTER(O.ArenaView), vp, vp, vp, sz, u64, u32, vp]
        L.wwo_leader.argtypes, L.wwo_leader.restype = args, None
        L.wwo_leader_bench.argtypes, L.wwo_leader_bench.restype = args, C.c_double
        L.wwo_follower.argtypes = [C.POINTER(O.ArenaView), C.POINTER(RO.Queues), vp, C.c_int, vp, vp, sz, u64, u32, vp, vp,
                                   vp, vp, vp, vp]
        L.wwo_follower.restype = None
        _lib = L
    return _lib


def leader(c, rows, blob, offsets, waves: int, n_bytes=None, bench: bool = False):
    """wwo_leader over columns c (changed in place; run O.arena_recompute after, as the step does) and the rows
    (LR.ROW_DTYPE per group slot, or None for an arena without runs) -> status u8[n]; with bench=True (status, seconds)."""
    blob = np.ascontiguousarray(blob, dtype=np.uint8)
    offsets = np.ascontiguousarray(offsets, dtype=np.uint32)
    if rows is not None:
        assert rows.dtype == LR.ROW_DTYPE and rows.flags.c_contiguous and len(rows) >= c.n_groups
    n = len(offsets) - 1
    status = np.zeros(n, np.uint8)
    v = O.view(c)
    f = lib().wwo_leader_bench if bench else lib().wwo_leader
    secs = f(C.byref(v), None if rows is None else rows.ctypes.data, blob.ctypes.data, offsets.ctypes.data, n,
             O.wire_n_bytes(blob, n_bytes), waves, status.ctypes.data)
    return (status, secs) if bench else status


def follower(c, q, logs, blob, offsets, waves: int, entries: bool, n_bytes=None):
    """wwo_follower over columns c (changed in place), read queues q (RO.ReadQueues or None) and the caller's table logs
    (AF.LOG_DTYPE per group slot; with entries its runs change in place) -> (status u8[n], from u64[n], appended
    AE.APPENDED_DTYPE[n], response blob, response offsets u32[responses + 1], totals u64[2]), as AE.batch returns them
    (appended all zero without entries)."""
    blob = np.ascontiguousarray(blob, dtype=np.uint8)
    offsets = np.ascontiguousarray(offsets, dtype=np.uint32)
    assert logs.dtype == AF.LOG_DTYPE and logs.flags.c_contiguous and len(logs) >= c.n_groups
    n = len(offsets) - 1
    status, frm, app = np.zeros(n, np.uint8), np.zeros(n, np.uint64), np.zeros(n, AE.APPENDED_DTYPE)
    resp, roff, totals = np.zeros(max(16, n * AF.FRAME_MAX), np.uint8), np.zeros(n + 1, np.uint32), np.zeros(2, np.uint64)
    v = O.view(c)
    qq = q._q() if q is not None else None
    lib().wwo_follower(C.byref(v), C.byref(qq) if qq is not None else None, logs.ctypes.data, int(entries),
                       blob.ctypes.data, offsets.ctypes.data, n, O.wire_n_bytes(blob, n_bytes), waves, status.ctypes.data,
                       frm.ctypes.data, app.ctypes.data, resp.ctypes.data, roff.ctypes.data, totals.ctypes.data)
    return status, frm, app, resp[: int(totals[1])].copy(), roff[: int(totals[0]) + 1].copy(), totals
