"""ctypes front-end of the heartbeat-response wire oracle (oracle/hb_wire_oracle.c).

TEST INFRASTRUCTURE ONLY, like oracle.py.  hb_wire_oracle.c is compiled together with wire_oracle.c, read_oracle.c,
control_oracle.c and raft_oracle.c into its own library, libhb_wire_oracle.so: next to the sources when that directory
is writable, else in a per-user temporary directory.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from oracle import oracle as O
from oracle import control_oracle as CO
from oracle import read_oracle as RO

_HERE = os.path.dirname(os.path.abspath(__file__))
_SOURCES = ("hb_wire_oracle.c", "wire_oracle.c", "read_oracle.c", "control_oracle.c", "raft_oracle.c")
_HEADERS = ("hb_wire_oracle.h", "wire_oracle.h", "read_oracle.h", "control_oracle.h", "raft_oracle.h")
WIRE_CONTEXT = 6


def build(force: bool = False) -> str:
    """Compile libhb_wire_oracle.so when it is missing or older than its sources; returns its path."""
    out_dir = _HERE if os.access(_HERE, os.W_OK) else os.path.join(tempfile.gettempdir(), f"hb_wire_oracle_{os.getuid()}")
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, "libhb_wire_oracle.so")
    newest = max(os.path.getmtime(os.path.join(_HERE, f)) for f in _SOURCES + _HEADERS)
    if force or not os.path.exists(path) or os.path.getmtime(path) < newest:
        tmp = f"{path}.{os.getpid()}"
        subprocess.run([os.environ.get("CC", "gcc"), *CO.CFLAGS, "-shared", "-o", tmp,
                        *[os.path.join(_HERE, f) for f in _SOURCES]], check=True)
        os.replace(tmp, path)
    return path


class Message(C.Structure):
    _fields_ = [("m", O.WireMessage), ("ctx_off", C.c_uint32), ("ctx_len", C.c_uint32)]


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        L = C.CDLL(build())
        vp, sz = C.c_void_p, C.c_size_t
        L.hwo_decode_message.argtypes, L.hwo_decode_message.restype = [vp, sz, C.POINTER(Message)], C.c_int
        L.hwo_decode_batch.argtypes, L.hwo_decode_batch.restype = [vp, vp, sz, vp, C.c_uint32, C.c_int, vp, vp], None
        L.hwo_apply.argtypes = [C.POINTER(O.ArenaView), C.POINTER(RO.Queues), vp, vp, sz, vp, vp, vp, C.POINTER(C.c_uint64)]
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


def decode_batch(blob, offsets, n_groups: int, terms=None, read_queues: bool = True):
    """hwo_decode_batch -> (status u8[n] as WIRE_*, records (APPEND_RESP_DTYPE)[n])."""
    blob, offsets, gt = _arrays(blob, offsets, terms)
    n = len(offsets) - 1
    status = np.zeros(n, np.uint8)
    recs = np.zeros(n, O.APPEND_RESP_DTYPE)
    lib().hwo_decode_batch(blob.ctypes.data, offsets.ctypes.data, n, None if gt is None else gt.ctypes.data, n_groups,
                           int(read_queues), status.ctypes.data, recs.ctypes.data)
    return status, recs


def apply(c, q, blob, offsets, terms=None):
    """hwo_apply over columns c (groups [0, c.n_groups) are the arena's) and read queues q (RO.ReadQueues, or None for
    an arena without them) -> (status bytes WIRE_* << 4 | RES_*, released reads)."""
    blob, offsets, gt = _arrays(blob, offsets, terms)
    n = len(offsets) - 1
    status = np.zeros(n, np.uint8)
    out = np.zeros(max(1, n * (q.max_pending if q is not None else 1)), RO.READ_STATE_DTYPE)
    cnt = C.c_uint64()
    v = O.view(c)
    qq = q._q() if q is not None else None
    lib().hwo_apply(C.byref(v), C.byref(qq) if qq is not None else None, blob.ctypes.data, offsets.ctypes.data, n,
                    None if gt is None else gt.ctypes.data, status.ctypes.data, out.ctypes.data, C.byref(cnt))
    return status, out[: cnt.value]
