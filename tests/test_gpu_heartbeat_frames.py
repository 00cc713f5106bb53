"""MsgHeartbeat frames built on the GPU (raftgpu_heartbeat_frames[_device]), byte-equal to the oracle
(oracle/hb_frames_oracle.c): random 100K-group arenas of every configuration, 1M groups after steps of synthetic
traffic, short capacities, the refusals, the frames fed back to raftgpu_heartbeat_wire, and the ReadIndex round trip
(requests -> frames -> the followers' echoed responses -> released reads).  Run with -m gpu."""
import numpy as np
import pytest

from oracle import hb_frames_oracle as HF
from oracle import hb_wire_oracle as H
from helpers import B
from control_cmds import cmds
import hb_frames as F
import pass_forms as PF
import read_cases as R

pytestmark = pytest.mark.gpu

P = 8
U64 = (1 << 64) - 1


def _ids(rng, n):
    ids = rng.integers(1, 1 << 63, (9, n), dtype=np.uint64)
    k = rng.random((9, n))
    ids[k < 0.05] = 0
    ids[(k > 0.05) & (k < 0.1)] = U64
    ids[(k > 0.1) & (k < 0.15)] = 128
    return ids


def _select(rng, cap, density):
    bits = rng.random(cap) < density
    return np.packbits(bits, bitorder="little").view(np.uint32).copy() if cap % 32 == 0 else None


def _check(a, c, q, first, n, ids, select, what):
    want = HF.bcast_heartbeats(c, q, first, n, ids, select)
    rc, blob, off, tot = a.heartbeat_frames(first, n, ids, select)
    assert rc == B.OK, what
    assert tot.tolist() == want[2].tolist(), (what, tot, want[2])
    assert np.array_equal(off, want[1]), what
    assert np.array_equal(blob, want[0]), (what, int(np.argmax(blob != want[0])) if len(blob) == len(want[0]) else None)
    dblob, doff, dtot = PF.broadcast(a, "heartbeat_frames", first, n, ids, select)
    assert dtot.tolist() == tot.tolist() and np.array_equal(doff, off) and np.array_equal(dblob, blob), what
    return want


# --------------------------------------------------------------------------- 1. random 100K-group arenas

N_NARROW, N_WIDE = 99_000, 500


def _setup(rng, reads):
    n = N_NARROW + 2 * N_WIDE
    a = B.Arena(n + 64)
    if reads:
        a.enable_read_index(P)
    assert a.group_alloc_range(N_NARROW) == 0
    for k in range(N_WIDE):
        assert a.group_alloc_wide() == N_NARROW + 2 * k
    d = R.OracleDriver(n, max_pending=P)
    for k in range(N_WIDE):
        lo = N_NARROW + 2 * k
        d.c.meta[lo], d.c.meta[lo + 1] = R.META_WIDE_LO, R.META_WIDE_HI
    setup = R.random_setup(rng, N_NARROW, N_WIDE)
    assert np.array_equal(a.control(setup), d.q.control(d.c, d.votes, setup))
    terms = rng.integers(1, 1 << 40, a.cap).astype(np.uint64)
    terms[rng.random(a.cap) < 0.08] = 0                                # leaders without a term
    terms[N_NARROW + 1:n:2] = 0                                        # (a high half's own term is not read)
    a.column_write(B.COL_TERM, 0, 0, terms[:n].copy())
    d.c.term[:] = 0
    d.c.term[:n] = terms[:n]
    if reads:
        reqs = R.random_requests(rng, n, 1.0, 1 << 40)
        res, _ = a.read_index_request(reqs)
        want, _ = d.q.request(d.c, reqs)
        assert np.array_equal(res, want) and (res == B.READ_QUEUED).sum() > n // 4
    return a, d, n


@pytest.mark.parametrize("reads", [True, False], ids=["read_queues", "no_read_queues"])
def test_random_arenas_vs_oracle(reads):
    rng = np.random.default_rng(0x4EB + reads)
    a, d, n = _setup(rng, reads)
    q = d.q if reads else None
    sel = _select(rng, a.cap, 0.3)
    ranges = [(0, n, None), (0, n, sel), (12_345, N_NARROW - 12_345 + 2 * 77, sel), (4_097, 2_001, None),
              (N_NARROW + 2 * 10, 2 * 40, sel), (0, a.cap, None), (n, a.cap - n, None)]
    kinds = np.zeros(3)
    for first, m, s in ranges:
        ids = _ids(rng, m)
        blob, off, tot = _check(a, d.c, q, first, m, ids, s, (first, m, s is not None))
        kinds += tot
    assert kinds[0] > 500_000 and kinds[2] > 5_000, kinds
    if reads:   # contexts went out
        blob, off, _ = HF.bcast_heartbeats(d.c, q, 0, 4096, _ids(rng, 4096))
        assert sum(1 for x in range(len(off) - 1) if blob[off[x + 1] - 10] == 0x62) > 300
    a.close()


# --------------------------------------------------------------------------- 2. 1M groups after synthetic traffic

def _oracle_queues(a, n, cap):
    cnt, ctx, _, _ = a.read_index_read(0, n)
    q = R.RO.ReadQueues(cap, P)
    q.allocated[:n] = 1
    q.count[:n], q.ctx[:n] = cnt, ctx
    return q


def test_1m_groups_after_steps():
    n = 1_000_000
    s = B.Synth(n, 0x4EB1, k_peers=5)
    a = B.Arena(n)
    a.enable_read_index(P)
    assert a.group_alloc_range(n) == 0
    a.load_columns(s.initial)
    rng = np.random.default_rng(5)
    terms = rng.integers(1, 1000, n).astype(np.uint64)
    terms[rng.random(n) < 0.01] = 0
    a.column_write(B.COL_TERM, 0, 0, terms)
    reqs = np.zeros(n, B.READ_REQ_DTYPE)
    reqs["group"], reqs["ctx"] = np.arange(n), rng.integers(1, 1 << 63, n, dtype=np.uint64)
    a.read_index_request(reqs)
    for _ in range(3):
        a.step_begin_records(s.next_round().copy(), B.STEP_READ_COMMITTED)
        a.step_wait()
    c = a.read_columns(n)
    c.term = np.zeros(c.cap, np.uint64)
    c.term[:n] = terms
    q = _oracle_queues(a, n, c.cap)
    assert (q.count[:n] > 0).sum() > n // 10
    ids = _ids(rng, n)
    want = _check(a, c, q, 0, n, ids, None, "1M")
    assert int(want[2][0]) > 3 * n
    a.close()


# --------------------------------------------------------------------------- 3. short capacities, refusals

def _small():
    d = R.ArenaDriver(64)
    a = d.a
    for g in range(40):
        R.leader(d, g, 0b11111)
        a.group_set_term(g, 7)
    R.leader(d, 40, 0b111)                                  # a leader without a term
    assert a.read_index_request(R.reqs(*[(g, 100 + g) for g in range(0, 40, 3)]))[0].tolist() == [B.READ_QUEUED] * 14
    wide = a.group_alloc_wide()
    assert a.control(cmds((B.CTL_SET_CONF, wide, 0, 0, (0x0F0F, 0, 0, 1)), (B.CTL_RESET, wide, 0, 0, (R.NO_TERM_START, 0, 0, 0)),
                          (B.CTL_BECOME_LEADER, wide)))["status"].tolist() == [B.OK] * 3
    a.group_set_term(wide, 9)
    return d, a, wide


def test_short_capacities_write_nothing():
    d, a, wide = _small()
    n = wide + 2
    ids = _ids(np.random.default_rng(1), n)
    rc, blob, off, tot = a.heartbeat_frames(0, n, ids)
    assert rc == B.OK and int(tot[0]) == 40 * 4 + 7 and int(tot[2]) == 1
    F_, N_ = int(tot[0]), int(tot[1])
    for bshort, fshort in ((1, 0), (0, 1), (1, 1)):
        bout = np.full(N_ + 64, 0xA5, np.uint8)
        oout = np.full(F_ + 8, 0x5A5A5A5A, np.uint32)
        rc, _, _, t = a.heartbeat_frames(0, n, ids, bytes_out=bout, offsets_out=oout, bytes_capacity=N_ - bshort,
                                         frames_capacity=F_ - fshort)
        assert rc == B.ERR_FULL and t.tolist() == tot.tolist()
        assert np.all(bout == 0xA5) and np.all(oout == 0x5A5A5A5A)
        # the device form: the guard patterns in device memory stay as they were
        d_ids, d_bytes, d_off, d_tot = a.device_alloc(ids.nbytes), a.device_alloc(N_ + 64), a.device_alloc(4 * (F_ + 8)), \
            a.device_alloc(24)
        a.h2d(d_ids, ids), a.h2d(d_bytes, bout), a.h2d(d_off, oout)
        a.heartbeat_frames_device(0, n, None, d_ids, d_bytes, N_ - bshort, d_off, F_ - fshort, d_tot)
        a.synchronize()
        gb, go, gt = np.zeros_like(bout), np.zeros_like(oout), np.zeros(3, np.uint64)
        a.d2h(gb, d_bytes), a.d2h(go, d_off), a.d2h(gt, d_tot)
        assert np.all(gb == 0xA5) and np.all(go == 0x5A5A5A5A) and gt.tolist() == tot.tolist()
        for p in (d_ids, d_bytes, d_off, d_tot):
            a.device_free(p)
    # exact capacities fit, and nothing is written past them
    bout = np.full(N_ + 64, 0xA5, np.uint8)
    oout = np.full(F_ + 8, 0x5A5A5A5A, np.uint32)
    rc, b2, o2, _ = a.heartbeat_frames(0, n, ids, bytes_out=bout, offsets_out=oout, bytes_capacity=N_, frames_capacity=F_)
    assert rc == B.OK and np.array_equal(b2, blob) and np.array_equal(o2, off)
    assert np.all(bout[N_:] == 0xA5) and np.all(oout[F_ + 1:] == 0x5A5A5A5A)
    a.close()


def test_refusals_before_any_launch():
    d, a, wide = _small()
    L, h = a._L, a._h
    ids = np.ones((9, 128), np.uint64)
    d_ids, d_bytes, d_off, d_tot = a.device_alloc(ids.nbytes), a.device_alloc(64 << 10), a.device_alloc(4 << 10), a.device_alloc(24)
    a.h2d(d_tot, np.full(3, 77, np.uint64))
    totals = np.zeros(3, np.uint64)
    bbuf, obuf = np.zeros(64 << 10, np.uint8), np.zeros(1 << 10, np.uint32)
    refused = [
        L.raftgpu_heartbeat_frames_device(h, None, wide + 1, 2, None, d_ids, d_bytes, 64 << 10, d_off, 1000, d_tot),  # starts at a high half
        L.raftgpu_heartbeat_frames_device(h, None, 0, wide + 1, None, d_ids, d_bytes, 64 << 10, d_off, 1000, d_tot),  # ends at a low half
        L.raftgpu_heartbeat_frames_device(h, None, 0, 8, None, d_ids, d_bytes + 4, 64 << 10, d_off, 1000, d_tot),    # unaligned
        L.raftgpu_heartbeat_frames_device(h, None, 0, 8, None, None, d_bytes, 64 << 10, d_off, 1000, d_tot),
        L.raftgpu_heartbeat_frames_device(h, None, 0, 8, None, d_ids, d_bytes, 64 << 10, d_off, 1000, None),
        L.raftgpu_heartbeat_frames_device(h, None, 0, 8, None, d_ids, None, 64, d_off, 1000, d_tot),
        L.raftgpu_heartbeat_frames(h, wide + 1, 2, None, ids.ctypes.data, bbuf.ctypes.data, len(bbuf), obuf.ctypes.data, 1000,
                                   totals.ctypes.data),
        L.raftgpu_heartbeat_frames(h, 0, 8, None, ids.ctypes.data, bbuf.ctypes.data, len(bbuf), obuf.ctypes.data, 1000, None),
    ]
    assert refused == [B.ERR_INVALID] * len(refused), refused
    assert L.raftgpu_heartbeat_frames_device(h, None, 0, a.cap + 1, None, d_ids, d_bytes, 1, d_off, 1, d_tot) == B.ERR_RANGE
    # (a range of 8_947_849 slots or more is refused too: its bound exceeds u32 offsets)
    assert B.heartbeat_frames_bound(8_947_848) < (1 << 32) <= B.heartbeat_frames_bound(8_947_849)
    a.synchronize()
    tot = np.zeros(3, np.uint64)
    a.d2h(tot, d_tot)
    assert tot.tolist() == [77] * 3           # nothing was launched
    a.close()


# --------------------------------------------------------------------------- 4. back through the wire entry points

def test_frames_through_heartbeat_wire_are_skip_type():
    d, a, wide = _small()
    n = wide + 2
    rc, blob, off, tot = a.heartbeat_frames(0, n, _ids(np.random.default_rng(2), n))
    assert rc == B.OK and int(tot[0]) > 100
    before = a.read_columns(n), a.read_index_read(0, n)
    fb = F.Frames([])
    fb.bytes, fb.offsets, fb.n, fb.n_bytes = blob, off, int(tot[0]), int(tot[1])
    status, rel = a.heartbeat_wire(fb)
    assert np.all(status == B.WIRE_SKIP_TYPE << 4) and len(rel) == 0
    after = a.read_columns(n), a.read_index_read(0, n)
    for name in ("matched", "next_idx", "peer_committed", "pflags", "committed"):
        assert np.array_equal(getattr(after[0], name), getattr(before[0], name)), name
    for x, y in zip(before[1], after[1]):
        assert np.array_equal(x, y)
    a.close()


# --------------------------------------------------------------------------- 5. the ReadIndex round trip

def _responses(blob, off, answering):
    """handle_heartbeat (raft.rs:2452-2464) at each follower that answers: to / from swapped, the context echoed,
    commit = the heartbeat's commit; framed for the leader as (group << 4 | slot)."""
    frames = []
    for k in range(len(off) - 1):
        lo, hi = int(off[k]), int(off[k + 1])
        hdr = int.from_bytes(bytes(blob[lo:lo + 4]), "little")
        g, s = hdr >> 4, hdr & 15
        if not answering[g, s]:
            continue
        m = H.decode_message(bytes(blob[lo + 4:hi]))
        assert m["msg_type"] == 8
        frames.append(F.frame(g, s, F.message(9, term=m["term"], commit=m["commit"], context=m["context"] or None,
                                              frm=m["to"])))
    return frames


@pytest.mark.parametrize("n_narrow,n_wide", [(20_000, 200)], ids=["20k"])
def test_read_round_trip(n_narrow, n_wide):
    rng = np.random.default_rng(0x4EB7)
    n = n_narrow + 2 * n_wide
    a = B.Arena(n + 64)
    a.enable_read_index(P)
    assert a.group_alloc_range(n_narrow) == 0
    for k in range(n_wide):
        assert a.group_alloc_wide() == n_narrow + 2 * k
    d = R.OracleDriver(n, max_pending=P)
    for k in range(n_wide):
        lo = n_narrow + 2 * k
        d.c.meta[lo], d.c.meta[lo + 1] = R.META_WIDE_LO, R.META_WIDE_HI
    setup = R.random_setup(rng, n_narrow, n_wide)
    assert np.array_equal(a.control(setup), d.q.control(d.c, d.votes, setup))
    terms = np.zeros(a.cap, np.uint64)
    terms[:n] = rng.integers(1, 50, n)
    terms[n_narrow + 1:n:2] = terms[n_narrow:n:2]
    a.column_write(B.COL_TERM, 0, 0, terms[:n].copy())
    d.c.term[:] = 0
    d.c.term[:n] = terms[:n]
    ids = _ids(rng, n)
    total = 0
    for rnd in range(4):
        reqs = R.random_requests(rng, n, 0.8, 1 << 40)
        res, rel = a.read_index_request(reqs)
        want_res, want_rel = d.q.request(d.c, reqs)
        assert np.array_equal(res, want_res), rnd
        sel_groups = np.unique(reqs["group"][np.isin(res, (B.READ_QUEUED, B.READ_DUP))]).astype(np.int64)
        select = np.zeros(a.cap // 32, np.uint32)
        np.bitwise_or.at(select, sel_groups // 32, np.left_shift(np.uint32(1), (sel_groups % 32).astype(np.uint32)))
        rc, blob, off, tot = a.heartbeat_frames(0, n, ids, select)
        wb, wo, wt = HF.bcast_heartbeats(d.c, d.q, 0, n, ids, select)
        assert rc == B.OK and np.array_equal(blob, wb) and np.array_equal(off, wo), rnd
        answering = rng.random((a.cap, 8)) < rng.choice([0.3, 0.6, 0.9])
        resp = _responses(blob, off, answering)
        assert len(resp) > 1000
        fb = F.Frames(resp)
        status, got = a.heartbeat_wire(fb)
        want_st, want = H.apply(d.c, d.q, fb.bytes[: fb.n_bytes], fb.offsets, terms)
        assert np.array_equal(status, want_st), rnd
        assert np.all((status >> 4) == B.WIRE_OK), rnd
        g, w = R.by_group(got), R.by_group(want)
        assert len(g) == len(w) and np.array_equal(g, w), rnd
        total += len(got)
        cnt, ctx, _, _ = a.read_index_read(0, n)
        assert np.array_equal(cnt, d.q.count[:n]), rnd
    assert total > 5000, total
    a.close()
