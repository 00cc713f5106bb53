"""The overlapped tick on the GPU: the schedules of tests/overlap_schedule.py replayed on an arena, every call made with
0, 1 or 2 steps in flight or right after a wait that left one in flight, each compared with the sequential model at
the call: statuses and outputs of every call, every step's result at its wait, and after each wait every column, the
votes, the terms, the read queues, the Inflights windows' meta and the counter deltas.  Then the refusals inside the
window: ERR_FULL and a short heartbeat_frames capacity with two steps in flight, a third begin right after a host
form, and raftgpu_control with records enqueued for the next step.  Run with -m gpu."""
import ctypes as C
import importlib

import numpy as np
import pytest

from oracle import hb_frames_oracle as HF
from helpers import B, assert_columns_equal
from control_cmds import cmds
import hb_frames as F
import read_cases as R
import overlap_schedule as S

pytestmark = pytest.mark.gpu

W = importlib.import_module("raft-rs_b200.wire")
PK_EXT = 1 << 37           # packed record: EXT payload or padding
JUNK = 0xAB


def _released_equal(got, want, what):
    g, w = R.by_group(got), R.by_group(want)
    assert len(g) == len(w) and np.array_equal(g, w), (what, len(g), len(w))


def _entries_sorted(e):
    return e[np.lexsort((e["peer_slot"], e["group"]))]


class Runner:
    """An arena built from a World's recipe, the pinned buffers of every step form (two of each: a step's buffer stays
    untouched until its wait), and the replay of events against the model's expectations."""

    def __init__(self, w: S.World, max_recs: int):
        self.w, n = w, w.n
        a = self.a = B.Arena(n + 64)
        if w.inflights:
            a.enable_inflights(S.INS_CAP)
        a.enable_read_index(S.P)
        assert a.group_alloc_range(w.n_narrow) == 0
        for k in range(w.n_wide):
            assert a.group_alloc_wide() == w.n_narrow + 2 * k
        if w.setup is not None:
            assert np.array_equal(a.control(w.setup), w.setup_want)
        else:
            a.load_columns(w.init)
            a.column_write(B.COL_TERM, 0, 0, w.init.term[:n].copy())
        assert a.cap <= S.side_len(n)
        self.base = a.counters()
        self.max_recs = max_recs
        self.pinned = [a.host_alloc_bytes(24 * max_recs).view(B.APPEND_RESP_DTYPE) for _ in range(2)]
        self.pk = [a.host_alloc_packed(4 * max_recs) for _ in range(2)]
        self.blob = [a.host_alloc_bytes(B.compact_bound(max_recs)) for _ in range(2)]
        self.wb = [W.WireBuffers(a, max_recs) for _ in range(2)]
        self.turn = 0
        self.pending = []          # (outcome, n_records expected or None, slot-result map or None), oldest first
        self.last = None

    def close(self):
        for wb in self.wb:
            wb.free()
        self.a.close()

    # ------------------------------------------------------------------ steps
    def begin(self, e, between=None):
        a, recs, flags, form = self.a, e.args["recs"], e.args["flags"], e.name
        assert len(recs) <= self.max_recs
        i, self.turn = self.turn, self.turn ^ 1
        main = (recs["flags"] & B.REC_EXT) == 0
        n_rec = slot_map = None
        if form in ("records_sorted", "records_shuffled"):
            a.step_begin_records(recs, flags)
        elif form in ("raw", "hybrid"):
            buf = self.pinned[i][: len(recs)]
            buf[:] = recs
            a.step_begin_records(buf, flags | (B.STEP_RAW if form == "raw" else B.STEP_HYBRID))
            n_rec = len(recs) if form == "raw" else None
        elif form == "packed":
            k = a.pack_records(recs, self.pk[i])
            slot_map = ((self.pk[i][:k, 0] & np.uint64(PK_EXT)) == 0, main)
            a.step_begin_packed(self.pk[i], k, flags)
            n_rec = k
        elif form == "compact":
            nb, units = B.pack_compact(recs, self.blob[i], want_units=True)
            n_rec = int(self.blob[i][: B.COMPACT_HDR_DTYPE.itemsize].view(B.COMPACT_HDR_DTYPE)[0]["n_records"])
            slot_map = (units[main], main)
            a.step_begin_compact(self.blob[i], nb, flags)
        elif form == "wire":
            wb = self.wb[i].encode(recs, e.args["term"])
            a.step_begin_wire(wb, flags)
            n_rec = wb.n + wb.n_records
        else:
            a.enqueue(recs)
            if between is not None:
                between()
            a.step_begin(flags)
            n_rec = len(recs)
        self.pending.append((e.want, n_rec, slot_map))

    def wait(self, e):
        o, n_rec, slot_map = self.pending.pop(0)
        assert o is e.want
        r = self.a.step_wait()
        what = f"wait of {o.form}"
        assert (r.n_advanced, r.n_duplicates) == (o.n_advanced, 0), (what, r.n_advanced, o.n_advanced, r.n_duplicates)
        if n_rec is not None:
            assert r.n_records == n_rec, (what, r.n_records, n_rec)
        self.last = (o, slot_map)
        self.check_results(o, what)
        self.check_state(e.args["totals"], what)

    def check_results(self, o, what):
        """raftgpu_step_results / _slot_results against the outcome o (None: no completed step is held)."""
        L, h = self.a._L, self.a._h
        pa, pc = C.c_void_p(), C.c_void_p()
        rc = L.raftgpu_step_results(h, C.byref(pa), C.byref(pc))
        ps, ns = C.c_void_p(), C.c_uint64()
        rs = L.raftgpu_step_slot_results(h, C.byref(ps), C.byref(ns))
        if o is None:
            assert (rc, rs) == (B.ERR_INVALID, B.ERR_INVALID), (what, rc, rs)
            return
        assert rc == B.OK, (what, rc)
        n, words = self.w.n, len(o.bitmap)
        bm = np.ctypeslib.as_array(C.cast(pa, C.POINTER(C.c_uint32)), shape=(words,))
        assert np.array_equal(bm, o.bitmap), (what, "bitmap")
        com = np.ctypeslib.as_array(C.cast(pc, C.POINTER(C.c_uint64)), shape=(n,))
        assert np.array_equal(com[o.advanced], o.committed[o.advanced]), (what, "committed")
        assert self.last[0] is o
        if not o.flags & S.RR:
            assert rs == B.ERR_INVALID, (what, rs)
            return
        assert rs == B.OK, (what, rs)
        res = np.ctypeslib.as_array(C.cast(ps, C.POINTER(C.c_uint8)), shape=(ns.value,))
        at, main = self.last[1]
        assert np.array_equal(res[at], o.results[main]), (what, "slot results")

    def check_state(self, totals, what):
        a, w, n = self.a, self.w, self.w.n
        assert_columns_equal(a.read_columns(n), w.c, n, what)
        for s in range(B.SLOTS):
            assert np.array_equal(a.column_read(B.COL_VOTES, s, 0, n, np.uint8), w.votes[s, :n]), (what, "votes", s)
            if w.inflights:
                assert np.array_equal(a.column_read(B.COL_INS_META, s, 0, n, np.uint32), w.c.ins_meta[s, :n]), (what, s)
        assert np.array_equal(a.column_read(B.COL_TERM, 0, 0, n, np.uint64), w.c.term[:n]), (what, "term")
        for name, x, y in zip(("count", "ctx", "index", "acks"), a.read_index_read(0, n), S.queue_view(w.q, 0, n)):
            assert np.array_equal(x, y), (what, "read queue", name, np.argwhere(x != y)[:3].tolist())
        self.check_counters(totals, what)

    def check_counters(self, totals, what):
        now = self.a.counters()
        got = {k: now[k] - self.base[k] for k in totals}
        assert got == totals, (what, got, totals)

    # ------------------------------------------------------------------ calls
    def call(self, e):
        a, L, h, want, x = self.a, self.a._L, self.a._h, e.want, e.args
        what = f"{e.name} with {e.point} in flight"
        if e.name == "commit_to":
            got = [a.group_commit_to(g, t) for g, t in zip(x["groups"], x["to"])]
            assert got == want, (what, got, want)
        elif e.name == "set_conf":
            got = [L.raftgpu_group_set_conf(h, g, a4[0], a4[1], a4[2], -1 if s == B.CTL_NO_SELF else s, a4[3])
                   for _, g, s, _, a4 in x["rows"]]
            assert got == want, (what, got, want)
        elif e.name == "control":
            assert np.array_equal(a.control(x["cmds"]), want), what
        elif e.name == "heartbeat_resp":
            assert np.array_equal(a.heartbeat_resp(x["recs"]), want), what
        elif e.name == "update_state":
            assert np.array_equal(a.update_state(x["entries"]), want), what
        elif e.name == "read_index_request":
            res, rel = a.read_index_request(x["reqs"])
            assert np.array_equal(res, want[0]), what
            _released_equal(rel, want[1], what)
        elif e.name == "read_index_ack":
            _released_equal(a.read_index_ack(x["recs"]), want, what)
        elif e.name == "read_index_recheck":
            _released_equal(a.read_index_recheck(x["groups"]), want, what)
        elif e.name == "heartbeat_wire":
            st, rel = a.heartbeat_wire(F.Frames(x["frames"]))
            assert np.array_equal(st, want[0]), what
            _released_equal(rel, want[1], what)
        elif e.name == "heartbeat_frames":
            rc, blob, off, tot = a.heartbeat_frames(x["first"], x["n"], x["ids"], x["select"])
            assert rc == B.OK and np.array_equal(tot, want[2]), (what, tot, want[2])
            assert np.array_equal(blob, want[0]) and np.array_equal(off, want[1]), what
        elif e.name == "follower_heartbeat":
            got = a.follower_heartbeat(F.Frames(x["frames"]), x["ids"], x["select"])
            for k, (g, wv) in enumerate(zip(got, want)):
                assert np.array_equal(g, wv), (what, k)
        elif e.name == "vote_wire":
            st, out = a.vote_wire(F.Frames(x["frames"]), x["select"])
            assert np.array_equal(st, want[0]) and np.array_equal(out, want[1]), what
        elif e.name == "vote_request_wire":
            got = a.vote_request_wire(F.Frames(x["frames"]), x["table"])
            for k, (g, wv) in enumerate(zip(got, want)):
                assert np.array_equal(g, wv), (what, k)
        elif e.name == "step_send_list":
            cap = 8 * self.w.n
            out, k = np.zeros(cap, B.SEND_ENTRY_DTYPE), C.c_uint64()
            rc = L.raftgpu_step_send_list(h, out.ctypes.data, cap, C.byref(k))
            if want is None:
                assert rc == B.ERR_INVALID, (what, rc)
            else:
                assert rc == B.OK, (what, rc)
                assert np.array_equal(_entries_sorted(out[: k.value]), want.astype(B.SEND_ENTRY_DTYPE)), what
        elif e.name in ("step_results", "slot_results"):
            self.check_results(want, what)
        elif e.name == "column_read":
            n = self.w.n
            assert np.array_equal(a.column_read(B.COL_COMMITTED, 0, 0, n, np.uint64), want[0]), what
            assert np.array_equal(a.column_read(B.COL_MATCHED, 1, 0, n, np.uint64), want[1]), what
        elif e.name == "counters_read":
            self.check_counters(want, what)
        elif e.name == "read_index_get":
            for g, wv in zip(x["groups"], want):
                for u, v in zip(a.read_index_get(g), wv):
                    assert np.array_equal(u, v), (what, g)
        elif e.name == "read_index_read":
            for u, v in zip(a.read_index_read(x["first"], x["n"]), want):
                assert np.array_equal(u, v), what
        else:
            raise AssertionError(e.name)

    def run(self, e):
        if e.op == "begin":
            self.begin(e)
        elif e.op == "wait":
            self.wait(e)
        else:
            self.call(e)


def _max_recs(n, frac):
    """Room for any batch random_batch draws from a fraction frac of n groups (5 cells, 2 records each, EXTs)."""
    return int(frac * n * 5 * 2 * 2) + 4096


@pytest.mark.parametrize("name,shape,n,seed,rounds,frac,window", S.SCHEDULES, ids=[s[0] for s in S.SCHEDULES])
def test_schedule_matches_the_sequential_model(name, shape, n, seed, rounds, frac, window):
    w = S.World(shape, n, seed)
    m = S.Model(w, frac, window)
    r = Runner(w, _max_recs(window, frac))
    seen = set()
    try:
        for e in S.schedule(m, rounds):
            r.run(e)
            seen.add((e.op, e.name, e.point))
        assert not r.pending
        r.check_state(m.totals, f"{name}: end")
    finally:
        r.close()
    assert {("call", k, p) for k in S.CALLS for p in S.POINTS} <= seen


# --------------------------------------------------------------------------- refusals inside the window

def _small():
    w = S.World("random", 4096, 0x0E9)
    m = S.Model(w, 0.5)
    return w, m, Runner(w, _max_recs(4096, 0.5))


def test_refusals_with_two_steps_in_flight():
    """With two steps in flight: a host form past the staging buffer is refused with ERR_FULL and writes nothing, a
    heartbeat_frames one byte short of what it needs is refused with ERR_FULL and reports the totals, a host form that
    is admitted does not let a third begin through (ERR_BUSY).  Both steps then complete exactly as the model says."""
    w, m, r = _small()
    a, L, h = r.a, r.a._L, r.a._h
    try:
        r.run(m.begin("records_sorted"))
        r.run(m.begin("packed"))
        big = np.zeros(1 << 20, B.APPEND_RESP_DTYPE)
        big["group"], big["peer_slot"], big["flags"] = np.arange(len(big)) % w.n_narrow, 1, B.REC_HEARTBEAT
        res = np.full(len(big), JUNK, np.uint8)
        assert L.raftgpu_heartbeat_resp(h, big.ctypes.data, len(big), res.ctypes.data) == B.ERR_FULL
        assert np.all(res == JUNK)
        k = 1024
        ids = w.rng.integers(1, 1 << 62, (B.SLOTS + 1, k), dtype=np.uint64)
        blob, off, tot = HF.bcast_heartbeats(w.c, w.q, 0, k, ids)
        assert int(tot[1]) > 0
        rc, _, _, got = a.heartbeat_frames(0, k, ids, bytes_capacity=int(tot[1]) - 1)
        assert rc == B.ERR_FULL and got[:2].tolist() == tot[:2].tolist(), (got, tot)
        r.run(m.call("update_state"))
        with pytest.raises(B.RaftGpuError) as ei:
            a.step_begin_records(S.random_batch(w.c, w.rng, 1), S.RC)
        assert ei.value.status == B.ERR_BUSY
        r.run(m.wait())
        r.run(m.wait())
        r.check_state(m.totals, "after the refusals")
    finally:
        r.close()


def test_control_is_busy_with_records_enqueued_for_the_next_step():
    """One step in flight and records enqueued for the next: raftgpu_control is refused with ERR_BUSY and changes
    nothing, its results stay as they were; the enqueued step then runs whole, and both complete as the model says."""
    w, m, r = _small()
    a, L, h = r.a, r.a._L, r.a._h
    try:
        r.run(m.begin("records_sorted"))
        g = int(m.hot(1)[0])
        lst = cmds((B.CTL_COMMIT_TO, g, 0, 0, (int(w.c.last_index[g]),)), (B.CTL_RESET_VOTES, g))
        out = np.full(len(lst), -7, B.CTL_RESULT_DTYPE)
        refused = []

        def control():
            refused.append(L.raftgpu_control(h, lst.ctypes.data, len(lst), out.ctypes.data))

        r.begin(m.begin("ring"), between=control)
        assert refused == [B.ERR_BUSY] and np.all(out["status"] == -7)
        r.run(m.wait())
        r.run(m.wait())
        r.check_state(m.totals, "after the refused control list")
    finally:
        r.close()


def test_records_api_several_records_per_cell_in_a_sparse_batch():
    """Regression: a group-sorted batch too sparse for the fused kernels' tiles (a unit block spans more than 4095
    groups), with two records on some cells, through raftgpu_step_begin_records.  It used to go to the scatter kernel,
    which applies one record per cell: the second records were counted as duplicates, the step failed and applied only
    part of the batch.  It now takes the general staging path.  With RAFTGPU_STEP_ASYNC the path is chosen after the
    call has returned, so the batch is refused at its wait with ERR_FULL, unapplied, and goes through without it."""
    n = 1 << 18
    rng = np.random.default_rng(0x0EA)
    init = S.random_state(n, S.Shape(((0x1F, 0, 0xE0),)), rng)
    a = B.Arena(n)
    try:
        assert a.group_alloc_range(n) == 0
        a.load_columns(init)
        ref = S.O.copy_columns(init)
        # every 32nd group, none with indexes near 2^48 (those leave the stream untileable whatever its density)
        recs = S.random_batch(ref, rng, 2, keep=(np.arange(n) % 32 == 0) & (init.last_index < (1 << 40)))
        main = recs[(recs["flags"] & B.REC_EXT) == 0]
        cells = main["group"].astype(np.int64) * 8 + main["peer_slot"]
        assert len(np.unique(cells)) < len(cells), "no cell holds two records"
        blob = np.zeros(B.compact_bound(len(recs) + 64), np.uint8)
        B.pack_compact(recs, blob)
        assert not blob[: B.COMPACT_HDR_DTYPE.itemsize].view(B.COMPACT_HDR_DTYPE)[0]["flags"] & B.COMPACT_TILEABLE
        assert len(recs) >= 16384          # several staging threads: the asynchronous submission is taken
        a.step_begin_records(recs, S.RC | B.STEP_ASYNC)
        assert a.step_wait(check=False).status == B.ERR_FULL
        assert_columns_equal(a.read_columns(n), init, n, "refused asynchronous batch")
        a.step_begin_records(recs, S.RC)
        r = a.step_wait()
        S.O.arena_apply(ref, recs, mode=0)
        adv, bm, _, _ = S.O.arena_recompute(ref)
        assert (r.n_advanced, r.n_duplicates) == (adv, 0) and adv > 0
        got_bm, com = a.step_results(n)
        assert np.array_equal(got_bm, bm[: len(got_bm)])
        on = S.bitmap_to_bool(got_bm, n)
        assert np.array_equal(com[on], ref.committed[:n][on])
        assert_columns_equal(a.read_columns(n), ref, n, "sparse batch, several records per cell")
    finally:
        a.close()
