"""ctypes front-end of the follower MsgAppend oracle (oracle/app_follow_oracle.c).

TEST INFRASTRUCTURE ONLY, like oracle.py.  app_follow_oracle.c is part of libraft_oracle.so; lib() declares its
functions on oracle.lib().
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import oracle as O
from oracle import read_oracle as RO

FRAME_MAX = 85  # 4-byte header + at most 81 bytes of Message
WIRE_ROLE, WIRE_COMMIT_RANGE = 7, 8
SELECT = 0x1
RES_OK, REJECT, STALE = 0x1, 0x2, 0x4
LOG_DTYPE = np.dtype([("id", "<u8"), ("run_start", "<u8"), ("run_term", "<u8"), ("flags", "<u4"), ("reserved", "<u4")])
# the literal form's groups, flags and outcomes
FOLLOWER, LOWER_REPLY = 0x1, 0x2
NONE, ANSWERED, DROPPED, FATAL = range(4)
GROUP_DTYPE = np.dtype([("id", "<u8"), ("term", "<u8"), ("committed", "<u8"), ("last_index", "<u8"), ("flags", "<u4"),
                        ("reserved", "<u4")])


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        L = O.lib()
        u64, vp, sz = C.c_uint64, C.c_void_p, C.c_size_t
        L.afl_encode_response.argtypes = [u64, u64, u64, u64, u64, u64, C.c_int, u64, vp]
        L.afl_encode_response.restype = sz
        L.afl_decode.argtypes, L.afl_decode.restype = [vp, sz, C.POINTER(O.WireMessage), C.POINTER(sz), vp, vp, sz], C.c_int
        args = [C.POINTER(O.ArenaView), C.POINTER(RO.Queues), vp, vp, vp, sz, u64, vp, vp, vp, vp, vp]
        L.afl_batch.argtypes, L.afl_batch.restype = args, None
        L.afl_bench.argtypes, L.afl_bench.restype = args, C.c_double
        L.afl_literal.argtypes = [vp, vp, u64, sz, vp, vp, sz, u64, vp, vp, vp, vp]
        L.afl_literal.restype = None
        _lib = L
    return _lib


def encode_response(to, frm, term, log_term=0, index=0, commit=0, reject=False, reject_hint=0) -> bytes:
    """afl_encode_response: a MsgAppendResponse's serialized Message (no header)."""
    buf = (C.c_uint8 * 96)()
    k = lib().afl_encode_response(to, frm, term, log_term, index, commit, int(reject), reject_hint, buf)
    return bytes(buf[:k])


def fields7(raw: bytes):
    """afl_decode: None when raw is not a well-formed message, else the field-7 count and [(term, index)] of the
    entries."""
    m, n7 = O.WireMessage(), C.c_size_t()
    et, ei = np.zeros(64, np.uint64), np.zeros(64, np.uint64)
    buf = (C.c_uint8 * max(1, len(raw))).from_buffer_copy(raw or b"\0")
    if not lib().afl_decode(buf, len(raw), C.byref(m), C.byref(n7), et.ctypes.data, ei.ctypes.data, 64):
        return None
    k = min(n7.value, 64)
    return n7.value, list(zip(et[:k].tolist(), ei[:k].tolist()))


def _out(n):
    return np.zeros(max(16, n * FRAME_MAX), np.uint8), np.zeros(n + 1, np.uint32), np.zeros(2, np.uint64)


def batch(c, q, logs, blob, offsets, bench: bool = False, n_bytes=None):
    """afl_batch over columns c (c.term = Raft::term; changed in place, as the arena is), read queues q (RO.ReadQueues or
    None) and the caller's table logs (LOG_DTYPE per group slot) -> (status u8[n], from u64[n], response blob, response
    offsets u32[responses + 1], totals u64[2]); with bench=True also seconds.  n_bytes as in O.wire_decode_batch."""
    blob = np.ascontiguousarray(blob, dtype=np.uint8)
    offsets = np.ascontiguousarray(offsets, dtype=np.uint32)
    lt = np.ascontiguousarray(logs, dtype=LOG_DTYPE)
    assert len(lt) >= c.n_groups
    n = len(offsets) - 1
    status, frm = np.zeros(n, np.uint8), np.zeros(n, np.uint64)
    resp, roff, totals = _out(n)
    v = O.view(c)
    qq = q._q() if q is not None else None
    f = lib().afl_bench if bench else lib().afl_batch
    secs = f(C.byref(v), C.byref(qq) if qq is not None else None, lt.ctypes.data, blob.ctypes.data, offsets.ctypes.data, n,
             O.wire_n_bytes(blob, n_bytes), status.ctypes.data, frm.ctypes.data, resp.ctypes.data, roff.ctypes.data,
             totals.ctypes.data)
    res = (status, frm, resp[: int(totals[1])].copy(), roff[: int(totals[0]) + 1].copy(), totals)
    return res + (secs,) if bench else res


def literal(groups, terms, blob, offsets, n_bytes=None):
    """afl_literal: the frames one at a time as the reference steps them.  groups (GROUP_DTYPE) and terms (u64
    [groups][log_cap], terms[g][i] = the term of index i of group g's log, [0] the dummy's) change in place ->
    (outcome u8[n], response blob, response offsets u32[responses + 1], totals u64[2])."""
    assert groups.dtype == GROUP_DTYPE and groups.flags.c_contiguous
    assert terms.dtype == np.uint64 and terms.flags.c_contiguous and terms.shape[0] >= len(groups)
    blob = np.ascontiguousarray(blob, dtype=np.uint8)
    offsets = np.ascontiguousarray(offsets, dtype=np.uint32)
    n = len(offsets) - 1
    outcome = np.zeros(n, np.uint8)
    resp, roff, totals = _out(n)
    lib().afl_literal(groups.ctypes.data, terms.ctypes.data, terms.shape[1], len(groups), blob.ctypes.data,
                      offsets.ctypes.data, n, O.wire_n_bytes(blob, n_bytes), outcome.ctypes.data, resp.ctypes.data,
                      roff.ctypes.data, totals.ctypes.data)
    return outcome, resp[: int(totals[1])].copy(), roff[: int(totals[0]) + 1].copy(), totals
