"""ctypes front-end of the follower-runs oracle (oracle/follower_runs_oracle.c): raftgpu_follower_append and
raftgpu_follower_append_entries on an arena with follower runs, one wave in C and the waves (DESIGN 3.19) here.

TEST INFRASTRUCTURE ONLY, like oracle.py.  follower_runs_oracle.c is part of libraft_oracle.so; lib() declares its
functions on oracle.lib().
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import app_entries_oracle as AE
from oracle import app_follow_oracle as AF
from oracle import leader_runs_oracle as LR
from oracle import oracle as O

# == raftgpu_follower_runs
ROW_DTYPE = np.dtype([("group", "<u4"), ("reserved", "<u4"), ("anchor_start", "<u8"), ("anchor_term", "<u8"),
                      ("run_start", "<u8", (2,)), ("run_term", "<u8", (2,))])
assert ROW_DTYPE.itemsize == 56

_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        L = AE.lib()
        LR.lib()
        u64, vp, sz = C.c_uint64, C.c_void_p, C.c_size_t
        from oracle import read_oracle as RO
        args = [C.POINTER(O.ArenaView), C.POINTER(RO.Queues), vp, vp, C.c_int, vp, vp, sz, u64, vp, vp, vp, vp, vp, vp]
        L.fro_batch.argtypes, L.fro_batch.restype = args, None
        L.fro_bench.argtypes, L.fro_bench.restype = args, C.c_double
        _lib = L
    return _lib


def row(group=0, anchor_start=0, anchor_term=0, runs=()):
    """One ROW_DTYPE row; runs = [(run_start, run_term), ...] from the top, at most two."""
    r = np.zeros(1, ROW_DTYPE)
    r["group"], r["anchor_start"], r["anchor_term"] = group, anchor_start, anchor_term
    for k, (s, t) in enumerate(runs):
        r["run_start"][0, k], r["run_term"][0, k] = s, t
    return r[0]


def rows_for(n):
    """n empty rows, group = the slot (as raftgpu_follower_runs_get reports them)."""
    rows = np.zeros(n, ROW_DTYPE)
    rows["group"] = np.arange(n)
    return rows


def row_status(r, allocated: bool = True, wide_hi: bool = False) -> int:
    """raftgpu_follower_runs_set's verdict on one row: the leader setter's check with the anchor's term and start in
    place of term and term_start."""
    lr = LR.row(int(r["group"]), int(r["anchor_term"]), int(r["anchor_start"]),
                [(int(r["run_start"][k]), int(r["run_term"][k])) for k in range(2)])
    return LR.row_status(lr, allocated, wide_hi)


def segments(terms, first_index=1):
    """The term runs of a literal log (terms[i] of entry i, entry 0 the dummy) from the top: [(start, term), ...], each
    at or above first_index - 1 and at least 1 (a run cut by compaction starts at first_index - 1)."""
    t = [int(x) for x in terms]
    out = []
    top = len(t) - 1
    lo = max(first_index - 1, 1)
    while top >= lo:
        s = top
        while s - 1 >= lo and t[s - 1] == t[top]:
            s -= 1
        out.append((s, t[top]))
        top = s - 1
    return out


def stated_ok(terms, log, r, last):
    """Every segment the table row log and the follower row r state -- the table's run, and run 1 and run 2 when r is
    anchored there -- has its stated term at every index of the literal log terms."""
    rs, rt = int(log["run_start"]), int(log["run_term"])
    if rs > last:
        return True
    segs = [(rs, last, rt)]
    if r is not None and int(r["anchor_term"]) and (int(r["anchor_start"]), int(r["anchor_term"])) == (rs, rt):
        top = rs - 1
        for k in range(2):
            s = int(r["run_start"][k])
            if not s:
                break
            segs.append((s, top, int(r["run_term"][k])))
            top = s - 1
    return all(int(terms[i]) == t for s, e, t in segs for i in range(s, e + 1))


def batch(c, q, logs, rows, blob, offsets, entries: bool, bench: bool = False, n_bytes=None):
    """fro_batch over columns c (changed in place, as the arena is), read queues q (RO.ReadQueues or None), the caller's
    table logs (AF.LOG_DTYPE per group slot) and rows (ROW_DTYPE per group slot, or None: no follower runs); logs and
    rows change in place as the device's do -> (status u8[n], from u64[n], appended AE.APPENDED_DTYPE[n] (zero without
    entries), response blob, response offsets u32[responses + 1], totals u64[2]); with bench=True also seconds."""
    blob = np.ascontiguousarray(blob, dtype=np.uint8)
    offsets = np.ascontiguousarray(offsets, dtype=np.uint32)
    assert logs.dtype == AF.LOG_DTYPE and logs.flags.c_contiguous and len(logs) >= c.n_groups
    if rows is not None:
        assert rows.dtype == ROW_DTYPE and rows.flags.c_contiguous and len(rows) >= c.n_groups
    n = len(offsets) - 1
    status, frm, app = np.zeros(n, np.uint8), np.zeros(n, np.uint64), np.zeros(n, AE.APPENDED_DTYPE)
    resp, roff, totals = np.zeros(max(16, n * AF.FRAME_MAX), np.uint8), np.zeros(n + 1, np.uint32), np.zeros(2, np.uint64)
    v = O.view(c)
    qq = q._q() if q is not None else None
    f = lib().fro_bench if bench else lib().fro_batch
    secs = f(C.byref(v), C.byref(qq) if qq is not None else None, logs.ctypes.data,
             None if rows is None else rows.ctypes.data, int(entries), blob.ctypes.data, offsets.ctypes.data, n,
             O.wire_n_bytes(blob, n_bytes), status.ctypes.data, frm.ctypes.data, app.ctypes.data, resp.ctypes.data,
             roff.ctypes.data, totals.ctypes.data)
    res = (status, frm, app, resp[: int(totals[1])].copy(), roff[: int(totals[0]) + 1].copy(), totals)
    return res + (secs,) if bench else res


def waves(c, q, logs, rows, blob, offsets, entries: bool, waves: int):
    """batch() repeated as raftgpu_arena_set_wire_waves runs it: wave j + 1 takes the frames wave j left DUP, in batch
    order, but for the groups whose claimant was NEEDS_LOG or COMMIT_RANGE.  A frame's status, from and appended record
    are those of the last wave that saw it; the responses of every wave go out in frame order.  Returns what batch()
    returns."""
    blob = np.ascontiguousarray(blob, dtype=np.uint8)
    offsets = np.ascontiguousarray(offsets, dtype=np.uint32)
    n = len(offsets) - 1
    status, frm, app = np.zeros(n, np.uint8), np.zeros(n, np.uint64), np.zeros(n, AE.APPENDED_DTYPE)
    own = [b""] * n
    stopped = set()
    frames = list(range(n))
    for j in range(waves):
        if not frames:
            break
        parts = [blob[offsets[i]:offsets[i + 1]].tobytes() for i in frames]
        sub_off = np.zeros(len(frames) + 1, np.uint32)
        sub_off[1:] = np.cumsum([len(p) for p in parts])
        sub = np.frombuffer(b"".join(parts) or b"\0", np.uint8)
        st, fr, ap, rb, ro, _ = batch(c, q, logs, rows, sub, sub_off, entries, n_bytes=int(sub_off[-1]))
        answered = 0
        nxt = []
        for k, i in enumerate(frames):
            status[i], frm[i], app[i] = st[k], fr[k], ap[k]
            if ap[k]["span_len"]:
                app[i]["span_off"] += int(offsets[i]) - int(sub_off[k])
            s = st[k] >> 4
            if s == O.WIRE_OK and st[k] & AF.RES_OK:
                own[i] = rb[ro[answered]:ro[answered + 1]].tobytes()
                answered += 1
            if s in (O.WIRE_NEEDS_LOG, AF.WIRE_COMMIT_RANGE):
                stopped.add(int.from_bytes(parts[k][:4], "little") >> 4)
        for k, i in enumerate(frames):
            if st[k] >> 4 == O.WIRE_DUP and (int.from_bytes(parts[k][:4], "little") >> 4) not in stopped:
                nxt.append(i)
        frames = nxt
    roff = np.zeros(1, np.uint32)
    ends = np.cumsum([len(x) for x in own if x]).astype(np.uint32)
    roff = np.concatenate([roff, ends])
    rb = np.frombuffer(b"".join(own), np.uint8).copy()
    return status, frm, app, rb, roff, np.array([len(roff) - 1, len(rb)], np.uint64)
