"""MsgHeartbeatResponse frames on the GPU (raftgpu_heartbeat_wire[_device]), bit-exact against the oracle
(oracle/hb_wire_oracle.c): the golden vectors, a 100K-group differential test of mixed batches that go through
raftgpu_wire_apply_device and then the heartbeat pass over one device buffer, the frame form against the record form
at 1M groups, the AppendResponse step leaving heartbeat frames alone, and the refusals.  Run with -m gpu."""
import ctypes as C
import importlib
import json
import os

import numpy as np
import pytest

from oracle import control_oracle as CO
from oracle import hb_wire_oracle as H
from helpers import B, O, assert_columns_equal, checksum, oracle_wire_apply
from control_cmds import NO_TERM_START, cmds
import hb_frames as F
import read_cases as R

pytestmark = pytest.mark.gpu

W = importlib.import_module("raft-rs_b200.wire")
HERE = os.path.dirname(os.path.abspath(__file__))
P = 8


def _released_equal(got, want, what):
    g, w = R.by_group(got), R.by_group(want)
    assert len(g) == len(w), (what, len(g), len(w))
    assert np.array_equal(g, w), what


# --------------------------------------------------------------------------- 1. golden vectors

@pytest.mark.parametrize("reads", [True, False], ids=["read_queues", "no_read_queues"])
def test_golden_vectors_through_the_gpu(reads):
    with open(os.path.join(HERE, "golden", "wire", "heartbeat_responses.json")) as f:
        vs = json.load(f)["vectors"]
    n = 512
    s = B.Synth(n, 0x4EA2, k_peers=5)
    a = B.Arena(n)
    if reads:
        a.enable_read_index(P)
    assert a.group_alloc_range(n) == 0
    a.load_columns(s.initial)
    ref = O.copy_columns(s.initial)
    q = None
    if reads:
        q = R.RO.ReadQueues(ref.cap, P)
        q.allocated[:n] = 1
        reqs = R.reqs(*[(g, 1000 + g) for g in range(n)])
        res, rel = a.read_index_request(reqs)
        want_res, want_rel = q.request(ref, reqs)
        assert np.array_equal(res, want_res) and (res == B.READ_QUEUED).sum() > n // 10
        _released_equal(rel, want_rel, "requests")
    terms = np.zeros(a.cap, dtype=np.uint64)
    terms[:n:2] = 7
    a.column_write(B.COL_TERM, 0, 0, terms[:n].copy())
    frames, prev = [], (0, 1)
    for i, v in enumerate(vs):
        g, slot = (i * 7) % n, 1 + i % 7            # slots 5..7 have no Progress: RES_NO_PROGRESS
        if i % 11 == 0:
            g, slot = prev
        prev = (g, slot)
        frames.append(F.frame(g, slot, bytes.fromhex(v["hex"])))
    # responses that name pending reads, some from two peers (a quorum of 5 voters is 3 with the leader's own ack)
    for g in range(1, n, 3):
        for slot in (1, 2) if g % 2 else (3,):
            frames.append(F.frame(g, slot, F.message(9, term=int(terms[g]), commit=3, context=F.ctx_bytes(1000 + g))))
    for g in range(0, 64, 2):          # a second response of a cell in the batch
        frames += [F.frame(g, 4, F.message(9, term=7, commit=2))] * 2
    frames.append(b"\x01\x02")
    frames.append(F.frame(n, 1, F.message(9)))
    fb = F.Frames(frames)
    status, rel = a.heartbeat_wire(fb)
    want, want_rel = H.apply(ref, q, fb.bytes[: fb.n_bytes], fb.offsets, terms)
    bad = np.nonzero(status != want)[0]
    assert len(bad) == 0, [(int(i), hex(status[i]), hex(want[i])) for i in bad[:5]]
    kinds = set(int(x) >> 4 for x in status)
    assert kinds == {B.WIRE_OK, B.WIRE_SKIP_TYPE, B.WIRE_TERM, B.WIRE_MALFORMED, B.WIRE_DUP, B.WIRE_CONTEXT}, kinds
    assert_columns_equal(a.read_columns(n), ref, n, "golden frames")
    if reads:
        assert len(want_rel) > 20
        _released_equal(rel, want_rel, "golden frames")
        R.queues_equal(a, q, n, "golden frames")
    else:
        assert len(rel) == 0
    a.close()


# --------------------------------------------------------------------------- 2. the 100K-group differential test

N_NARROW, N_WIDE = 99_000, 500


def _setup(rng, reads, inflights):
    n = N_NARROW + 2 * N_WIDE
    a = B.Arena(n + 64)
    if inflights:
        a.enable_inflights(2)
    if reads:
        a.enable_read_index(P)
    assert a.group_alloc_range(N_NARROW) == 0
    for k in range(N_WIDE):
        assert a.group_alloc_wide() == N_NARROW + 2 * k
    d = R.OracleDriver(n, max_pending=P)
    if inflights:
        O.enable_inflights(d.c, 2)
    for k in range(N_WIDE):
        lo = N_NARROW + 2 * k
        d.c.meta[lo], d.c.meta[lo + 1] = R.META_WIDE_LO, R.META_WIDE_HI
    setup = R.random_setup(rng, N_NARROW, N_WIDE)
    gc = rng.choice(N_NARROW, N_NARROW // 20, replace=False)          # group commit on 5 % of the narrow groups
    setup = np.concatenate([setup, cmds(*[(B.CTL_SET_GROUP_COMMIT, int(g), 0, 1) for g in gc])])
    _control(a, d, reads, setup, "setup")
    terms = np.zeros(a.cap, np.uint64)
    terms[:n] = rng.integers(1, 4, n)
    terms[N_NARROW + 1:n:2] = terms[N_NARROW:n:2]                      # the halves of a wide group share the term
    terms[rng.random(a.cap) < 0.1] = 0                                 # the caller filters these groups' terms
    a.column_write(B.COL_TERM, 0, 0, terms[:n].copy())
    return a, d, n, terms


def _control(a, d, reads, lst, what):
    want = d.q.control(d.c, d.votes, lst) if reads else CO.arena_control(d.c, d.votes, lst)
    assert np.array_equal(a.control(lst), want), what


@pytest.mark.parametrize("inflights", [False, True], ids=["host_inflights", "device_inflights"])
@pytest.mark.parametrize("reads", [True, False], ids=["read_queues", "no_read_queues"])
def test_mixed_batches_vs_oracle(reads, inflights):
    rng = np.random.default_rng(0x4B + 2 * reads + inflights)
    a, d, n, terms = _setup(rng, reads, inflights)
    k = 120_000
    nb_max = 64 * 2 * k
    d_bytes, d_off = a.device_alloc(nb_max), a.device_alloc(4 * (2 * k + 2))
    d_st1, d_st2 = a.device_alloc(2 * k), a.device_alloc(2 * k)
    cap = min(2 * k, n) * P
    d_rel, d_cnt = a.device_alloc(24 * cap), a.device_alloc(8)
    seen = np.zeros(8, np.int64)
    n_rel = 0
    for rnd in range(3):
        if reads:
            reqs = R.random_requests(rng, n, 0.5 if rnd else 3.0, 12)
            res, rel = a.read_index_request(reqs)
            want_res, want_rel = d.q.request(d.c, reqs)
            assert np.array_equal(res, want_res), rnd
            _released_equal(rel, want_rel, f"round {rnd}: requests")
        blob, offsets = R.mixed_batch(rng, d, n, terms, reads, k)
        m = len(offsets) - 1
        a.h2d(d_bytes, blob)
        a.h2d(d_off, offsets)
        a.wire_apply_device(d_bytes, len(blob), d_off, m, d_st1)
        if reads:
            a.heartbeat_wire_device(d_bytes, len(blob), d_off, m, d_st2, d_rel, cap, d_cnt)
        else:
            a.heartbeat_wire_device(d_bytes, len(blob), d_off, m, d_st2)
        a.synchronize()
        st1, st2 = np.zeros(m, np.uint8), np.zeros(m, np.uint8)
        a.d2h(st1, d_st1), a.d2h(st2, d_st2)
        want1 = oracle_wire_apply(d.c, blob, offsets, n, terms)
        want2, want_rel = H.apply(d.c, d.q if reads else None, blob, offsets, terms)
        assert np.array_equal(st1, want1), f"round {rnd}: append statuses"
        bad = np.nonzero(st2 != want2)[0]
        assert len(bad) == 0, (rnd, [(int(i), hex(st2[i]), hex(want2[i])) for i in bad[:5]])
        # every frame is applied by at most one of the passes
        assert not np.any(((st1 >> 4) == B.WIRE_OK) & ((st2 >> 4) == B.WIRE_OK))
        seen += np.bincount(st2 >> 4, minlength=8)[:8]
        assert_columns_equal(a.read_columns(n), d.c, n, f"round {rnd}")
        if reads:
            cnt = np.zeros(1, np.uint64)
            a.d2h(cnt, d_cnt)
            rel = np.zeros(int(cnt[0]), B.READ_STATE_DTYPE)
            if len(rel):
                a.d2h(rel, d_rel)
            _released_equal(rel, want_rel, f"round {rnd}: released")
            n_rel += len(rel)
            R.queues_equal(a, d.q, n, f"round {rnd}")
        if inflights:           # sends fill the two-entry windows, so heartbeats free their first entries
            cells = rng.choice(8 * n, n // 2, replace=False)
            e = np.zeros(len(cells), B.SEND_ENTRY_DTYPE)
            e["group"], e["peer_slot"] = cells % n, cells // n
            e["next_idx"] = d.c.last_index[cells % n]
            assert np.array_equal(a.update_state(e), O.arena_update_state(d.c, e)), rnd
        li = rng.choice(N_NARROW, n // 100, replace=False)             # control: a re-election, some new log tails
        rows = []
        for g in li[: len(li) // 4].tolist():
            top = int(d.c.last_index[g]) + 1
            rows += [(B.CTL_RESET, g, 0, 0, (NO_TERM_START, top, int(d.c.committed[g]), top)), (B.CTL_BECOME_LEADER, g)]
        for g in li[len(li) // 4:].tolist():
            rows.append((B.CTL_SET_LOG_BOUNDS, g, 0, 0, (int(d.c.term_start[g]), int(d.c.last_index[g]) + 3)))
        _control(a, d, reads, cmds(*rows), f"round {rnd}: control")
    assert_columns_equal(a.read_columns(n), d.c, n, "end")
    ok_kinds = [B.WIRE_OK, B.WIRE_SKIP_TYPE, B.WIRE_TERM, B.WIRE_DUP, B.WIRE_CONTEXT]
    assert all(seen[x] > 100 for x in ok_kinds), seen
    if reads:
        assert n_rel > 1000, n_rel
    a.close()


# --------------------------------------------------------------------------- 3. frames against records at 1M groups

def test_frames_equal_records_at_1m():
    """cfg3, one tick: every follower answers the heartbeat that carries its group's last pending read id.  The 4M
    shuffled responses as MsgHeartbeatResponse frames, and as 24-byte records through raftgpu_heartbeat_resp +
    raftgpu_read_index_ack, leave identical arenas, result bytes and released reads."""
    n = 1_000_000
    s = B.Synth(n, 0x1A2B3, k_peers=5)
    arenas = []
    for _ in range(2):
        ar = B.Arena(n)
        ar.enable_read_index(P)
        assert ar.group_alloc_range(n) == 0
        ar.load_columns(s.initial)
        arenas.append(ar)
    rec_a, wire_a = arenas
    rng = np.random.default_rng(3)
    reqs = np.zeros(n, B.READ_REQ_DTYPE)
    reqs["group"], reqs["ctx"] = np.arange(n), np.arange(1, n + 1)
    for ar in arenas:
        ar.read_index_request(reqs)
    d_last = rec_a.device_alloc(8 * n)
    rec_a.read_index_last_ctx_device(0, n, d_last)
    last = np.zeros(n, np.uint64)
    rec_a.d2h(last, d_last)
    assert (last != 0).sum() > n // 10
    recs = np.zeros(4 * n, B.APPEND_RESP_DTYPE)
    recs["group"] = np.repeat(np.arange(n), 4)
    recs["peer_slot"] = np.tile(np.arange(1, 5), n)
    recs["flags"] = B.REC_HEARTBEAT | B.REC_READ_CTX
    recs["index"] = last[recs["group"]]
    recs["commit"] = rng.integers(0, 1 << 16, 4 * n)
    recs = recs[rng.permutation(4 * n)]
    cap = n * P
    # the record form
    d_rec, d_res = rec_a.device_alloc(recs.nbytes), rec_a.device_alloc(4 * n)
    d_rel1, d_cnt1 = rec_a.device_alloc(24 * cap), rec_a.device_alloc(8)
    rec_a.h2d(d_rec, recs)
    assert rec_a._L.raftgpu_heartbeat_resp_device(rec_a._h, None, d_rec, 4 * n, d_res, None) == B.OK
    assert rec_a._L.raftgpu_read_index_ack_device(rec_a._h, None, d_rec, 4 * n, d_rel1, cap, d_cnt1) == B.OK
    # the frame form
    wb = W.WireBuffers(wire_a, 4 * n, bytes_per_record=32)
    wb.encode_heartbeats(recs)
    assert wb.n == 4 * n
    d_bytes, d_off = wire_a.device_alloc(wb.n_bytes + 16), wire_a.device_alloc(4 * (4 * n + 1))
    d_st, d_rel2, d_cnt2 = wire_a.device_alloc(4 * n), wire_a.device_alloc(24 * cap), wire_a.device_alloc(8)
    wire_a.h2d(d_bytes, wb.bytes[: wb.n_bytes])
    wire_a.h2d(d_off, wb.offsets[: 4 * n + 1])
    wire_a.heartbeat_wire_device(d_bytes, wb.n_bytes, d_off, 4 * n, d_st, d_rel2, cap, d_cnt2)
    for ar in arenas:
        ar.synchronize()
    res, st = np.zeros(4 * n, np.uint8), np.zeros(4 * n, np.uint8)
    rec_a.d2h(res, d_res), wire_a.d2h(st, d_st)
    assert np.all((st >> 4) == B.WIRE_OK)
    assert np.array_equal(st & 0xF, res)
    rel = []
    for ar, d_rel, d_cnt in ((rec_a, d_rel1, d_cnt1), (wire_a, d_rel2, d_cnt2)):
        c = np.zeros(1, np.uint64)
        ar.d2h(c, d_cnt)
        r = np.zeros(int(c[0]), B.READ_STATE_DTYPE)
        ar.d2h(r, d_rel)
        rel.append(r)
    assert len(rel[0]) > n // 10
    _released_equal(rel[1], rel[0], "1M released")
    g1, g2 = rec_a.read_columns(n), wire_a.read_columns(n)
    for name in ("matched", "next_idx", "peer_committed", "pflags", "committed", "last_index"):
        assert checksum(getattr(g1, name)) == checksum(getattr(g2, name)), name
    q1, q2 = rec_a.read_index_read(0, n), wire_a.read_index_read(0, n)
    for x, y in zip(q1, q2):
        assert checksum(x) == checksum(y)
    wb.free()
    for ar in arenas:
        ar.close()


# --------------------------------------------------------------------------- 4. the AppendResponse step is unchanged

def test_step_begin_wire_leaves_heartbeat_frames_to_the_host():
    n = 1024
    s = B.Synth(n, 0x77, k_peers=5)
    a = B.Arena(n)
    assert a.group_alloc_range(n) == 0
    a.load_columns(s.initial)
    hb = np.zeros(3 * n, B.APPEND_RESP_DTYPE)
    hb["group"], hb["peer_slot"] = np.repeat(np.arange(n), 3), np.tile(np.arange(1, 4), n)
    hb["flags"] = B.REC_HEARTBEAT | B.REC_READ_CTX
    hb["index"], hb["commit"] = np.arange(3 * n) % 5, 7
    wb = W.WireBuffers(a, 3 * n).encode_heartbeats(hb)
    before = a.read_columns(n)
    a.step_begin_wire(wb, B.STEP_READ_COMMITTED)
    a.step_wait()
    assert np.all(a.wire_status() == B.WIRE_SKIP_TYPE << 4)
    after = a.read_columns(n)
    # the followers' cells (slots 1..7: the step's recompute updates the leader's own peer_committed in slot 0)
    for name in ("matched", "next_idx", "peer_committed", "pflags", "pending_request_snapshot"):
        assert np.array_equal(getattr(after, name)[1:], getattr(before, name)[1:]), name
    wb.free()
    a.close()


# --------------------------------------------------------------------------- 5. refusals

def test_refusals_before_any_launch():
    d = R.ArenaDriver(8)
    a = d.a
    for g in range(8):
        R.leader(d, g, 0b111)
    assert a.read_index_request(R.reqs((0, 1), (3, 2)))[0].tolist() == [B.READ_QUEUED] * 2
    fb = F.Frames([F.frame(0, 1, F.message(9, commit=1, context=F.ctx_bytes(1))),
                   F.frame(0, 2, F.message(9, commit=1, context=F.ctx_bytes(1))),
                   F.frame(3, 1, F.message(9, commit=1, context=F.ctx_bytes(2)))])
    L, h = a._L, a._h
    d_bytes, d_off, d_st = a.device_alloc(64 + fb.n_bytes), a.device_alloc(4 * 4), a.device_alloc(4)
    d_rel, d_cnt = a.device_alloc(24 * 3 * P), a.device_alloc(8)
    a.h2d(d_bytes, fb.bytes), a.h2d(d_off, fb.offsets)
    before = a.read_index_read(0, 8), a.read_columns(8)
    need = 3 * P
    refused = [
        L.raftgpu_heartbeat_wire_device(h, None, None, fb.n_bytes, d_off, 3, d_st, d_rel, need, d_cnt),
        L.raftgpu_heartbeat_wire_device(h, None, d_bytes, fb.n_bytes, None, 3, d_st, d_rel, need, d_cnt),
        L.raftgpu_heartbeat_wire_device(h, None, d_bytes, fb.n_bytes, d_off, 3, None, d_rel, need, d_cnt),
        L.raftgpu_heartbeat_wire_device(h, None, d_bytes, fb.n_bytes, d_off, 3, d_st, d_rel, need, None),
        L.raftgpu_heartbeat_wire_device(h, None, d_bytes + 4, fb.n_bytes, d_off, 3, d_st, d_rel, need, d_cnt),
        L.raftgpu_heartbeat_wire_device(h, None, d_bytes, fb.n_bytes, d_off, 3, d_st, d_rel, need - 1, d_cnt),
        L.raftgpu_heartbeat_wire_device(h, None, d_bytes, fb.n_bytes, d_off, 1 << 32, d_st, d_rel, need, d_cnt),
        L.raftgpu_heartbeat_wire_device(h, None, d_bytes, 1 << 32, d_off, 3, d_st, d_rel, need, d_cnt),
        L.raftgpu_heartbeat_wire(h, None, fb.n_bytes, fb.offsets.ctypes.data, 3, None, None, 0, None),
        L.raftgpu_heartbeat_wire(h, fb.bytes.ctypes.data, fb.n_bytes, fb.offsets.ctypes.data, 3, None,
                                 np.zeros(need, B.READ_STATE_DTYPE).ctypes.data, need - 1, C.byref(C.c_uint64())),
        L.raftgpu_heartbeat_wire(h, fb.bytes.ctypes.data, fb.n_bytes, fb.offsets.ctypes.data, 3, None, None, 0, None),
    ]
    assert refused == [B.ERR_INVALID] * len(refused), refused
    a.synchronize()
    after = a.read_index_read(0, 8), a.read_columns(8)
    for x, y in zip(before[0], after[0]):
        assert np.array_equal(x, y)
    assert_columns_equal(after[1], before[1], 8, "refusals")
    # with room, the same frames release both reads
    assert L.raftgpu_heartbeat_wire_device(h, None, d_bytes, fb.n_bytes, d_off, 3, d_st, d_rel, need, d_cnt) == B.OK
    a.synchronize()
    cnt = np.zeros(1, np.uint64)
    a.d2h(cnt, d_cnt)
    assert cnt.tolist() == [2]
    # an arena without read queues takes NULL release buffers, and a context there is the host's
    b = B.Arena(64)
    assert b.group_alloc_range(8) == 0
    st, rel = b.heartbeat_wire(fb)
    assert (st >> 4).tolist() == [B.WIRE_CONTEXT] * 3 and len(rel) == 0
    st, rel = b.heartbeat_wire(F.Frames([F.frame(0, 1, F.message(9, commit=1))]))
    assert st.tolist() == [B.RES_NO_PROGRESS] and len(rel) == 0
    b.close()
    a.close()
