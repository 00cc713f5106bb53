"""ctypes front-end of the leader-runs oracle (oracle/leader_runs_oracle.c): the wire step's decision of rejected
MsgAppendResponse frames, in a literal form (the leader's whole term array) and the batch form the device restates.

TEST INFRASTRUCTURE ONLY, like oracle.py.  leader_runs_oracle.c is part of libraft_oracle.so; lib() declares its
functions on oracle.lib().
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import oracle as O

ROW_DTYPE = np.dtype([("group", "<u4"), ("reserved", "<u4"), ("term", "<u8"), ("term_start", "<u8"),
                      ("run_start", "<u8", (2,)), ("run_term", "<u8", (2,))])
assert ROW_DTYPE.itemsize == 56
REC_DTYPE = np.dtype([("group", "<u4"), ("peer_slot", "u1"), ("flags", "u1"), ("reserved", "<u2"), ("index", "<u8"),
                      ("commit", "<u8")])
NO_TERM_START = (1 << 64) - 1

_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        L = O.lib()
        u64, vp, sz, i32 = C.c_uint64, C.c_void_p, C.c_size_t, C.c_int32
        L.lro_row_status.argtypes, L.lro_row_status.restype = [vp, C.c_int, C.c_int], i32
        L.lro_find_conflict_by_term.argtypes = [vp, u64, u64, u64, u64]
        L.lro_find_conflict_by_term.restype = u64
        L.lro_probe_by_runs.argtypes = [u64, u64, u64, vp, u64, u64, C.POINTER(u64)]
        L.lro_probe_by_runs.restype = C.c_int
        L.lro_decode_batch.argtypes = [C.POINTER(O.ArenaView), vp, vp, vp, sz, u64, vp, vp, vp, vp]
        L.lro_decode_batch.restype = None
        L.lro_literal_batch.argtypes = [vp, vp, vp, vp, C.c_uint32, vp, vp, sz, u64, vp, vp, vp, vp]
        L.lro_literal_batch.restype = None
        L.lro_bench.argtypes = [C.POINTER(O.ArenaView), vp, vp, vp, sz, u64, vp, vp, vp, vp, C.c_int]
        L.lro_bench.restype = C.c_double
        _lib = L
    return _lib


def row(group=0, term=0, term_start=0, runs=()):
    """One ROW_DTYPE row; runs = [(run_start, run_term), ...] from the top, at most two."""
    r = np.zeros(1, ROW_DTYPE)
    r["group"], r["term"], r["term_start"] = group, term, term_start
    for k, (s, t) in enumerate(runs):
        r["run_start"][0, k], r["run_term"][0, k] = s, t
    return r[0]


def row_status(r, allocated: bool = True, wide_hi: bool = False) -> int:
    a = np.array([r], ROW_DTYPE)
    return int(lib().lro_row_status(a.ctypes.data, int(allocated), int(wide_hi)))


def find_conflict_by_term(terms, first_index: int, h: int, lt: int) -> int:
    """The literal walk: terms[i] = term of entry i (entry 0 included), last index len(terms) - 1."""
    t = np.ascontiguousarray(terms, dtype=np.uint64)
    return int(lib().lro_find_conflict_by_term(t.ctypes.data, first_index, len(t) - 1, h, lt))


def probe_by_runs(term, term_start, last_index, r, h, lt):
    """The device rule for one group: the conflict index, or None where the frame stays NEEDS_LOG.  r: a row or None."""
    out = C.c_uint64()
    a = None if r is None else np.array([r], ROW_DTYPE)
    ok = lib().lro_probe_by_runs(term, term_start, last_index, None if a is None else a.ctypes.data, h, lt, C.byref(out))
    return int(out.value) if ok else None


def _outs(n):
    return np.zeros(n, np.uint8), np.zeros(n, REC_DTYPE), np.zeros(n, np.uint64), np.zeros(n, np.uint64)


def decode_batch(c, rows, blob, offsets, n_bytes=None):
    """lro_decode_batch over columns c (read only) and the rows (ROW_DTYPE per group slot, or None for an arena without
    runs) -> (status u8[n], records[n], hint u64[n], request_snapshot u64[n])."""
    blob = np.ascontiguousarray(blob, dtype=np.uint8)
    offsets = np.ascontiguousarray(offsets, dtype=np.uint32)
    if rows is not None:
        assert rows.dtype == ROW_DTYPE and rows.flags.c_contiguous and len(rows) >= c.n_groups
    n = len(offsets) - 1
    st, recs, hint, snap = _outs(n)
    v = O.view(c)
    lib().lro_decode_batch(C.byref(v), None if rows is None else rows.ctypes.data, blob.ctypes.data, offsets.ctypes.data,
                           n, O.wire_n_bytes(blob, n_bytes), st.ctypes.data, recs.ctypes.data, hint.ctypes.data,
                           snap.ctypes.data)
    return st, recs, hint, snap


def bench(c, rows, blob, offsets, iters=3):
    """Seconds per lro_decode_batch on one core."""
    blob = np.ascontiguousarray(blob, dtype=np.uint8)
    offsets = np.ascontiguousarray(offsets, dtype=np.uint32)
    n = len(offsets) - 1
    st, recs, hint, snap = _outs(n)
    v = O.view(c)
    return lib().lro_bench(C.byref(v), None if rows is None else rows.ctypes.data, blob.ctypes.data, offsets.ctypes.data,
                           n, len(blob), st.ctypes.data, recs.ctypes.data, hint.ctypes.data, snap.ctypes.data, iters)


def literal_batch(logs, first_index, group_term, blob, offsets, n_bytes=None):
    """lro_literal_batch: logs = one term array per group (entry 0 first), first_index u64 per group, group_term u64
    per group or None -> (status, records, hint, request_snapshot)."""
    blob = np.ascontiguousarray(blob, dtype=np.uint8)
    offsets = np.ascontiguousarray(offsets, dtype=np.uint32)
    off = np.zeros(len(logs) + 1, np.uint64)
    off[1:] = np.cumsum([len(t) for t in logs])
    terms = np.ascontiguousarray(np.concatenate([np.asarray(t, np.uint64) for t in logs]) if logs else np.zeros(1, np.uint64))
    fi = np.ascontiguousarray(first_index, dtype=np.uint64)
    gt = None if group_term is None else np.ascontiguousarray(group_term, dtype=np.uint64)
    n = len(offsets) - 1
    st, recs, hint, snap = _outs(n)
    lib().lro_literal_batch(off.ctypes.data, terms.ctypes.data, fi.ctypes.data, None if gt is None else gt.ctypes.data,
                            len(logs), blob.ctypes.data, offsets.ctypes.data, n, O.wire_n_bytes(blob, n_bytes),
                            st.ctypes.data, recs.ctypes.data, hint.ctypes.data, snap.ctypes.data)
    return st, recs, hint, snap


def runs_of_log(terms, first_index, n_runs):
    """The row a leader states for its log (terms[i] of entry i, the leader's own term the last run): (term,
    term_start, [(run_start, run_term), ...]) with at most n_runs runs below term_start, each at or above
    first_index - 1 (a run cut by compaction starts at first_index - 1)."""
    t = [int(x) for x in terms]
    last = len(t) - 1
    term = t[last]
    ts = last
    while ts - 1 >= max(first_index - 1, 1) and t[ts - 1] == term:
        ts -= 1
    runs = []
    top = ts - 1
    while len(runs) < n_runs and top >= max(first_index - 1, 1) and t[top] > 0:
        s = top
        while s - 1 >= max(first_index - 1, 1) and t[s - 1] == t[top]:
            s -= 1
        runs.append((s, t[top]))
        top = s - 1
    return term, ts, runs
