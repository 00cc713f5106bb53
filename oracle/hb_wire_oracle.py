"""ctypes front-end of the heartbeat-response wire oracle (oracle/hb_wire_oracle.c).

TEST INFRASTRUCTURE ONLY, like oracle.py.  hb_wire_oracle.c is part of libraft_oracle.so; lib() declares its functions
on oracle.lib().
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import oracle as O
from oracle import read_oracle as RO

WIRE_CONTEXT = 6


class Message(C.Structure):
    _fields_ = [("m", O.WireMessage), ("ctx_off", C.c_uint32), ("ctx_len", C.c_uint32)]


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        L = O.lib()
        vp, sz = C.c_void_p, C.c_size_t
        L.hwo_decode_message.argtypes, L.hwo_decode_message.restype = [vp, sz, C.POINTER(Message)], C.c_int
        L.hwo_decode_batch.argtypes = [vp, vp, sz, C.c_uint64, vp, C.c_uint32, C.c_int, vp, vp]
        L.hwo_decode_batch.restype = None
        L.hwo_apply.argtypes = [C.POINTER(O.ArenaView), C.POINTER(RO.Queues), vp, vp, sz, C.c_uint64, vp, vp, vp,
                                C.POINTER(C.c_uint64)]
        L.hwo_apply.restype = None
        _lib = L
    return _lib


def decode_message(raw: bytes):
    """hwo_decode_message: None when the bytes are not a protobuf message, else the scalar fields of
    O.wire_decode_message plus "context" (bytes)."""
    h = Message()
    buf = (C.c_uint8 * max(1, len(raw))).from_buffer_copy(raw or b"\0")
    if not lib().hwo_decode_message(buf, len(raw), C.byref(h)):
        return None
    m = h.m
    return {"msg_type": m.msg_type, "reject": m.reject, "to": m.to, "from": m.from_, "term": m.term,
            "log_term": m.log_term, "index": m.index, "commit": m.commit, "commit_term": m.commit_term,
            "request_snapshot": m.request_snapshot, "reject_hint": m.reject_hint, "priority": m.priority,
            "context": bytes(raw[h.ctx_off:h.ctx_off + h.ctx_len])}


def _arrays(blob, offsets, terms):
    blob = np.ascontiguousarray(blob, dtype=np.uint8)
    offsets = np.ascontiguousarray(offsets, dtype=np.uint32)
    gt = None if terms is None else np.ascontiguousarray(terms, dtype=np.uint64)
    return blob, offsets, gt


def decode_batch(blob, offsets, n_groups: int, terms=None, read_queues: bool = True, n_bytes=None):
    """hwo_decode_batch -> (status u8[n] as WIRE_*, records (APPEND_RESP_DTYPE)[n]); n_bytes as in
    O.wire_decode_batch."""
    blob, offsets, gt = _arrays(blob, offsets, terms)
    n = len(offsets) - 1
    status = np.zeros(n, np.uint8)
    recs = np.zeros(n, O.APPEND_RESP_DTYPE)
    lib().hwo_decode_batch(blob.ctypes.data, offsets.ctypes.data, n, O.wire_n_bytes(blob, n_bytes),
                           None if gt is None else gt.ctypes.data, n_groups, int(read_queues), status.ctypes.data,
                           recs.ctypes.data)
    return status, recs


def apply(c, q, blob, offsets, terms=None, n_bytes=None):
    """hwo_apply over columns c (groups [0, c.n_groups) are the arena's) and read queues q (RO.ReadQueues, or None for
    an arena without them) -> (status bytes WIRE_* << 4 | RES_*, released reads); n_bytes as in O.wire_decode_batch."""
    blob, offsets, gt = _arrays(blob, offsets, terms)
    n = len(offsets) - 1
    status = np.zeros(n, np.uint8)
    out = np.zeros(max(1, n * (q.max_pending if q is not None else 1)), RO.READ_STATE_DTYPE)
    cnt = C.c_uint64()
    v = O.view(c)
    qq = q._q() if q is not None else None
    lib().hwo_apply(C.byref(v), C.byref(qq) if qq is not None else None, blob.ctypes.data, offsets.ctypes.data, n,
                    O.wire_n_bytes(blob, n_bytes), None if gt is None else gt.ctypes.data, status.ctypes.data, out.ctypes.data,
                    C.byref(cnt))
    return status, out[: cnt.value]
