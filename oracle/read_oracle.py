"""ctypes front-end of the ReadIndex oracle (oracle/read_oracle.c).

TEST INFRASTRUCTURE ONLY, like oracle.py.  read_oracle.c is part of libraft_oracle.so; lib() declares its functions
on oracle.lib().
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import oracle as O
from oracle import control_oracle as CO


READ_REQ_DTYPE = np.dtype([("group", "<u4"), ("reserved", "<u4"), ("ctx", "<u8")])
READ_STATE_DTYPE = np.dtype([("group", "<u4"), ("reserved", "<u4"), ("ctx", "<u8"), ("index", "<u8")])
REC_HEARTBEAT, REC_READ_CTX = 0x04, 0x08
QUEUED, READY, DUP, DROPPED, FULL, NO_GROUP, NO_CTX = range(1, 8)


class Queues(C.Structure):
    _fields_ = [("cap", C.c_uint32), ("max_pending", C.c_uint32), ("count", C.c_void_p), ("ctx", C.c_void_p),
                ("index", C.c_void_p), ("acks", C.c_void_p), ("allocated", C.c_void_p)]


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        L = O.lib()
        V, vp, sz = C.POINTER(O.ArenaView), C.c_void_p, C.c_size_t
        Q = C.POINTER(Queues)
        for name in ("ro_read_request",):
            getattr(L, name).argtypes = [V, Q, vp, sz, vp, vp, C.POINTER(C.c_uint64)]
        for name in ("ro_read_ack_seq", "ro_read_ack_batch", "ro_read_recheck"):
            getattr(L, name).argtypes = [V, Q, vp, sz, vp, C.POINTER(C.c_uint64)]
        L.ro_read_control.argtypes = [V, Q, vp, vp, sz, vp]
        L.ro_read_last_ctx.argtypes, L.ro_read_last_ctx.restype = [Q, C.c_uint32], C.c_uint64
        for name in ("ro_read_request", "ro_read_ack_seq", "ro_read_ack_batch", "ro_read_recheck", "ro_read_control"):
            getattr(L, name).restype = None
        _lib = L
    return _lib


class ReadQueues:
    """Every group slot's ReadOnly: count [cap], ctx / index / acks [cap][max_pending] (front first), allocated [cap]."""

    def __init__(self, cap: int, max_pending: int = 8):
        self.cap, self.max_pending = int(cap), int(max_pending)
        self.count = np.zeros(cap, np.uint32)
        self.ctx = np.zeros((cap, max_pending), np.uint64)
        self.index = np.zeros((cap, max_pending), np.uint64)
        self.acks = np.zeros((cap, max_pending), np.uint16)
        self.allocated = np.zeros(cap, np.uint8)

    def _q(self) -> Queues:
        return Queues(self.cap, self.max_pending, self.count.ctypes.data, self.ctx.ctypes.data, self.index.ctypes.data,
                      self.acks.ctypes.data, self.allocated.ctypes.data)

    def copy(self) -> "ReadQueues":
        d = ReadQueues(self.cap, self.max_pending)
        for n in ("count", "ctx", "index", "acks", "allocated"):
            getattr(d, n)[...] = getattr(self, n)
        return d

    def pending(self, g):
        """(ctx, index, acks) of group g's pending reads, front first."""
        k = int(self.count[g])
        return self.ctx[g, :k], self.index[g, :k], self.acks[g, :k]

    def request(self, c, reqs: np.ndarray):
        """MsgReadIndex for each request in order -> (result bytes, released reads)."""
        reqs = np.ascontiguousarray(reqs, dtype=READ_REQ_DTYPE)
        res = np.zeros(len(reqs), np.uint8)
        out = np.zeros(max(1, len(reqs)), READ_STATE_DTYPE)
        n = C.c_uint64()
        v, q = O.view(c), self._q()
        lib().ro_read_request(C.byref(v), C.byref(q), reqs.ctypes.data, len(reqs), res.ctypes.data, out.ctypes.data, C.byref(n))
        return res, out[: n.value]

    def _acks(self, fn, c, recs):
        recs = np.ascontiguousarray(recs, dtype=O.APPEND_RESP_DTYPE)
        out = np.zeros(max(1, len(recs) * self.max_pending), READ_STATE_DTYPE)
        n = C.c_uint64()
        v, q = O.view(c), self._q()
        fn(C.byref(v), C.byref(q), recs.ctypes.data, len(recs), out.ctypes.data, C.byref(n))
        return out[: n.value]

    def ack_seq(self, c, recs):
        """handle_heartbeat_response's read tail for each record in order -> released reads."""
        return self._acks(lib().ro_read_ack_seq, c, recs)

    def ack_batch(self, c, recs):
        """The same batch as OR-every-ack-then-advance (the device's formulation) -> released reads."""
        return self._acks(lib().ro_read_ack_batch, c, recs)

    def recheck(self, c, groups):
        g = np.ascontiguousarray(groups, dtype=np.uint32)
        out = np.zeros(max(1, len(g) * self.max_pending), READ_STATE_DTYPE)
        n = C.c_uint64()
        v, q = O.view(c), self._q()
        lib().ro_read_recheck(C.byref(v), C.byref(q), g.ctypes.data, len(g), out.ctypes.data, C.byref(n))
        return out[: n.value]

    def last_ctx(self, g) -> int:
        q = self._q()
        return int(lib().ro_read_last_ctx(C.byref(q), g))

    def control(self, c, votes: np.ndarray, cmds: np.ndarray) -> np.ndarray:
        """ro_arena_control with the read hooks (RESET empties, SET_CONF clears removed peers' acks)."""
        assert votes.dtype == np.uint8 and votes.shape == (O.SLOTS, c.cap) and votes.flags.c_contiguous
        assert cmds.dtype.itemsize == CO.CTL_CMD_DTYPE.itemsize and cmds.flags.c_contiguous
        res = np.zeros(len(cmds), dtype=CO.CTL_RESULT_DTYPE)
        v, q = O.view(c), self._q()
        lib().ro_read_control(C.byref(v), C.byref(q), votes.ctypes.data, cmds.ctypes.data, len(cmds), res.ctypes.data)
        return res


def per_group(released: np.ndarray) -> dict:
    """Released reads -> {group: [(ctx, index), ...] in release order}."""
    d = {}
    for r in released:
        d.setdefault(int(r["group"]), []).append((int(r["ctx"]), int(r["index"])))
    return d
