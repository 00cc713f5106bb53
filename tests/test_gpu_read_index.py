"""ReadIndex (ReadOnlyOption::Safe) on the GPU: the reference's read-only tests through the C-ABI, a randomized
differential test against the oracle over 100K groups (requests, shuffled ack batches, control lists with resets
and configuration changes, rechecks), the refusals, and that an arena with read queues steps exactly like one
without.  Run with -m gpu."""
import ctypes as C

import numpy as np
import pytest

from oracle import read_oracle as RO
from helpers import B, O, assert_columns_equal, bitmap_to_bool
from control_cmds import NO_TERM_START, META_WIDE_LO, META_WIDE_HI, cmds
import read_cases as R

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case", R.REFERENCE_CASES, ids=lambda f: f.__name__)
def test_reference_read_only_cases(case):
    d = R.ArenaDriver(4)
    case(d)
    d.a.close()


def test_edge_cases_and_group_lifecycle():
    d = R.ArenaDriver(2, max_pending=4)
    R.edge_cases(d, 2)
    a = d.a
    # a freed group leaves no queue behind, and a group allocated into its slot starts empty
    R.leader(d, 1, 0b111)
    assert a.read_index_request(R.reqs((1, 5), (1, 6)))[0].tolist() == [B.READ_QUEUED] * 2
    a.group_free(1)
    assert a.read_index_request(R.reqs((1, 7)))[0].tolist() == [B.READ_NO_GROUP]
    assert a.group_alloc() == 1
    assert a.read_index_get(1)[0].tolist() == []
    # a wide group: its high half is not a group of its own; peers 8..15 ack into the low half's queue
    w = a.group_alloc_wide()
    R.leader(d, w, 0x107)                      # voters 0, 1, 2 and 8: quorum 3
    res, _ = a.read_index_request(R.reqs((w, 11), (w + 1, 12)))
    assert res.tolist() == [B.READ_QUEUED, B.READ_NO_GROUP]
    assert R.pairs(a.read_index_ack(R.acks((w + 1, 0, 11)))) == []
    assert d.queue(w) == [(11, 1, 0x101)]
    assert R.pairs(a.read_index_ack(R.acks((w, 2, 11)))) == [(w, 11, 1)]
    a.close()


def test_refusals_apply_nothing():
    d = R.ArenaDriver(8)
    a = d.a
    for g in range(8):
        R.leader(d, g, 0b111)
    assert a.read_index_request(R.reqs((0, 1), (3, 2)))[0].tolist() == [B.READ_QUEUED] * 2
    before = a.read_index_read(0, 8)
    # out of group order: refused, nothing applied (host form: ERR_INVALID; device form: results 0, *d_bad bumped)
    with pytest.raises(B.RaftGpuError) as e:
        a.read_index_request(R.reqs((5, 3), (2, 4), (6, 5)))
    assert e.value.status == B.ERR_INVALID
    bad_reqs = R.reqs((1, 3), (7, 4), (2, 5))
    L, h = a._L, a._h
    d_req, d_res = a.device_alloc(bad_reqs.nbytes), a.device_alloc(len(bad_reqs))
    d_out, d_cnt, d_bad = a.device_alloc(24 * 16), a.device_alloc(8), a.device_alloc(4)
    a.h2d(d_req, bad_reqs)
    a.h2d(d_res, np.full(3, 0xAB, np.uint8))
    a.h2d(d_bad, np.array([7], np.uint32))
    assert L.raftgpu_read_index_request_device(h, None, d_req, 3, d_res, d_out, 8, d_cnt, d_bad) == B.OK
    a.synchronize()
    res, bad, cnt = np.zeros(3, np.uint8), np.zeros(1, np.uint32), np.zeros(1, np.uint64)
    a.d2h(res, d_res), a.d2h(bad, d_bad), a.d2h(cnt, d_cnt)
    assert res.tolist() == [0, 0, 0] and bad.tolist() == [8] and cnt.tolist() == [0]
    # capacities below what the pass could release: refused before any launch
    assert L.raftgpu_read_index_request_device(h, None, d_req, 3, d_res, d_out, 2, d_cnt, d_bad) == B.ERR_INVALID
    recs = R.acks((0, 1, 1), (3, 1, 2))
    d_rec = a.device_alloc(recs.nbytes)
    a.h2d(d_rec, recs)
    assert L.raftgpu_read_index_ack_device(h, None, d_rec, 2, d_out, 2 * 8 - 1, d_cnt) == B.ERR_INVALID
    out, n = np.zeros(4, B.READ_STATE_DTYPE), C.c_uint64()
    assert L.raftgpu_read_index_ack(h, recs.ctypes.data, 2, out.ctypes.data, 4, C.byref(n)) == B.ERR_INVALID
    assert L.raftgpu_read_index_recheck(h, np.array([0, 3], np.uint32).ctypes.data, 2, out.ctypes.data, 4,
                                        C.byref(n)) == B.ERR_INVALID
    after = a.read_index_read(0, 8)
    for x, y in zip(before, after):
        assert np.array_equal(x, y)
    # ... and with room, the same acks release both reads
    assert L.raftgpu_read_index_ack_device(h, None, d_rec, 2, d_out, 2 * 8, d_cnt) == B.OK
    a.synchronize()
    a.d2h(cnt, d_cnt)
    assert cnt.tolist() == [2]
    # an arena without read queues refuses the read calls
    b = B.Arena(64)
    one = R.reqs((0, 1))
    assert b._L.raftgpu_read_index_request(b._h, one.ctypes.data, 1, None, out.ctypes.data, 4, C.byref(n)) == B.ERR_INVALID
    assert b._L.raftgpu_read_index_ack(b._h, recs.ctypes.data, 2, out.ctypes.data, 4, C.byref(n)) == B.ERR_INVALID
    b.close()
    a.close()


# --------------------------------------------------------------------------- the randomized differential test

N_NARROW, N_WIDE = 99_000, 500     # 100K group slots: narrow groups, then wide pairs
P = 8


def _twin(rng):
    n = N_NARROW + 2 * N_WIDE
    a = B.Arena(n + 64)
    a.enable_read_index(P)
    assert a.group_alloc_range(N_NARROW) == 0
    for k in range(N_WIDE):
        assert a.group_alloc_wide() == N_NARROW + 2 * k
    d = R.OracleDriver(n, max_pending=P)
    for k in range(N_WIDE):
        lo = N_NARROW + 2 * k
        d.c.meta[lo], d.c.meta[lo + 1] = META_WIDE_LO, META_WIDE_HI
    setup = R.random_setup(rng, N_NARROW, N_WIDE)
    assert np.array_equal(a.control(setup), d.q.control(d.c, d.votes, setup))
    return a, d, n


def _compare_queues(a, d, n, what):
    got = a.read_index_read(0, n)
    want = R.oracle_queue_view(d.q, n)
    for name, x, y in zip(("count", "ctx", "index", "acks"), got, want):
        if not np.array_equal(x, y):
            g = int(np.argwhere(x != y)[0][0])
            raise AssertionError(f"{what}: queue {name} of group {g}: got {x[g]} want {y[g]}")


def _compare_released(got, want, what):
    g, w = R.by_group(got), R.by_group(want)
    assert len(g) == len(w), (what, len(g), len(w))
    assert np.array_equal(g, w), what


def _churn(rng, d, n):
    """A control list for ~1 % of the groups: re-elections (RESET + BECOME_LEADER + log bounds + commit), followers,
    and configuration changes that remove or add peers.  Returns (list, the groups whose configuration changed)."""
    rows, conf = [], []
    for g in rng.choice(np.arange(0, N_NARROW), n // 100, replace=False).tolist() + \
            [N_NARROW + 2 * int(k) for k in rng.choice(N_WIDE, 10, replace=False)]:
        wide = g >= N_NARROW
        lim = 0xFFFF if wide else 0xFF
        r = rng.random()
        if r < 0.5:     # drop or add a peer, keep the leader's slot
            lo, hi = int(d.c.meta[g]), int(d.c.meta[g + 1]) if wide else 0
            inc = (lo & 0xFF) | ((hi & 0xFF) << 8)
            out = ((lo >> 8) & 0xFF) | (((hi >> 8) & 0xFF) << 8)
            learn = ((lo >> 16) & 0xFF) | (((hi >> 16) & 0xFF) << 8)
            self_slot = ((lo >> 24) & 7) if lo & O.META_HAS_SELF else (8 + ((hi >> 24) & 7) if hi & O.META_HAS_SELF else B.CTL_NO_SELF)
            flip = 1 << int(rng.integers(0, 16 if wide else 8))
            if self_slot != B.CTL_NO_SELF and flip == 1 << self_slot:
                continue
            inc ^= flip
            learn &= ~flip
            out = 0 if rng.random() < 0.5 else out & ~flip
            if inc == 0:
                continue
            rows.append((B.CTL_SET_CONF, g, self_slot, 0, (inc & lim, out & lim, learn & lim, 5)))
            conf.append(g)
        elif r < 0.8:   # a new term
            li = int(d.c.last_index[g]) + 1
            rows += [(B.CTL_RESET, g, 0, 0, (NO_TERM_START, li, int(d.c.committed[g]), li)), (B.CTL_BECOME_LEADER, g),
                     (B.CTL_SET_LOG_BOUNDS, g, 0, 0, (li + 1, li + 3)), (B.CTL_COMMIT_TO, g, 0, 0, (li + 2,))]
        else:           # a follower
            rows.append((B.CTL_RESET, g, 0, 0, (NO_TERM_START, 9, 9, 9)))
    return cmds(*rows), conf


def test_randomized_differential_against_the_oracle():
    rng = np.random.default_rng(0x5EAD)
    a, d, n = _twin(rng)
    wide_hi = (d.c.meta[:d.c.cap] & META_WIDE_HI) != 0
    bad = list(range(n, n + 6)) + [N_NARROW + 1, N_NARROW + 3]     # unallocated groups, wide high halves
    n_rel = n_full = n_dup = n_ready = n_drop = 0
    for tick in range(6):
        reqs = R.random_requests(rng, n, 0.5 if tick else 4.0, 12, bad_groups=bad)
        res, rel = a.read_index_request(reqs)
        want_res, want_rel = d.q.request(d.c, reqs)
        assert np.array_equal(res, want_res), tick
        _compare_released(rel, want_rel, f"tick {tick}: requests")
        n_full += int((res == B.READ_FULL).sum())
        n_dup += int((res == B.READ_DUP).sum())
        n_ready += int((res == B.READ_READY).sum())
        n_drop += int((res == B.READ_DROPPED).sum())
        assert (res[np.isin(reqs["group"], bad)] == B.READ_NO_GROUP).all()
        _compare_queues(a, d, n, f"tick {tick}: requests")
        for k in range(2):
            recs = R.random_acks(rng, d.q, d.c.meta, n, 300_000, wide_hi)
            got = a.read_index_ack(recs)
            want = d.q.ack_seq(d.c, recs)          # the reference's order: one response at a time
            _compare_released(got, want, f"tick {tick}: ack batch {k}")
            n_rel += len(got)
            _compare_queues(a, d, n, f"tick {tick}: ack batch {k}")
        churn, conf = _churn(rng, d, n)
        assert np.array_equal(a.control(churn), d.q.control(d.c, d.votes, churn)), tick
        _compare_queues(a, d, n, f"tick {tick}: control list")
        got = a.read_index_recheck(conf)
        want = d.q.recheck(d.c, sorted(set(conf)))
        _compare_released(got, want, f"tick {tick}: recheck")
        _compare_queues(a, d, n, f"tick {tick}: recheck")
        # the ctx every group's heartbeat carries
        d_out = a.device_alloc(8 * n)
        a.read_index_last_ctx_device(0, n, d_out)
        last = np.zeros(n, np.uint64)
        a.d2h(last, d_out)
        a.device_free(d_out)
        cnt = d.q.count[:n].astype(np.int64)
        want_last = np.where(cnt > 0, d.q.ctx[np.arange(n), np.maximum(cnt - 1, 0)], 0)
        assert np.array_equal(last, want_last), tick
    # the workload reached every branch
    assert min(n_rel, n_full, n_dup, n_ready, n_drop) > 100, (n_rel, n_full, n_dup, n_ready, n_drop)
    a.close()


# --------------------------------------------------------------------------- no behaviour change

def _step_twins(n, seed):
    synth = B.Synth(n, seed=seed, k_peers=5)
    arenas = []
    for enabled in (True, False):
        ar = B.Arena(n)
        if enabled:
            ar.enable_read_index(8)
        assert ar.group_alloc_range(n) == 0
        ar.load_columns(synth.initial)
        arenas.append(ar)
    # the enabled arena holds pending reads while it steps
    reqs = np.zeros(n, B.READ_REQ_DTYPE)
    reqs["group"], reqs["ctx"] = np.arange(n), np.arange(1, n + 1)
    res, _ = arenas[0].read_index_request(reqs)
    assert (res == B.READ_QUEUED).sum() > n // 10
    return synth, arenas


def test_steps_are_identical_with_read_queues():
    n = 8192
    synth, (on, off) = _step_twins(n, 0xBEEF)
    pk = np.zeros((2 * 6 * n + 8, 2), np.uint64)
    bufs = {}
    for ar in (on, off):
        bufs[id(ar)] = (ar.device_alloc(pk.nbytes), ar.device_alloc(4 * (n // 256 + 2)), ar.device_alloc(4 * (n // 32 + 1)),
                        ar.device_alloc(8 * n))
    for rnd in range(6):
        recs = synth.next_round().copy()
        outs = []
        for ar in (on, off):
            if rnd % 3 == 0:      # the fused compact kernel, through the records API
                ar.step_begin_records(recs, B.STEP_READ_COMMITTED)
                ar.step_wait()
                bm, com = ar.step_results(n)
                adv = bitmap_to_bool(bm, n)
                outs.append((bm.copy(), np.where(adv, com, 0)))
            elif rnd % 3 == 1:    # the scatter kernels
                ar.enqueue(recs)
                ar.step(B.STEP_READ_COMMITTED)
                bm, com = ar.step_results(n)
                adv = bitmap_to_bool(bm, n)
                outs.append((bm.copy(), np.where(adv, com, 0)))
            else:                 # the device-resident fused tile kernel: every group's commit index
                d_pk, d_off, d_bm, d_com = bufs[id(ar)]
                k = ar.pack_records(recs, pk)
                tiles = B.tile_index(pk, k, n)
                ar.h2d(d_pk, pk[:k])
                ar.h2d(d_off, tiles)
                ar.step_sorted_device(d_pk, k, d_off, d_adv=d_bm, d_commit=d_com)
                bm, com = np.zeros(n // 32, np.uint32), np.zeros(n, np.uint64)
                ar.d2h(bm, d_bm), ar.d2h(com, d_com)
                outs.append((bm, com))
        assert np.array_equal(outs[0][0], outs[1][0]), rnd
        assert np.array_equal(outs[0][1], outs[1][1]), rnd
        assert_columns_equal(on.read_columns(n), off.read_columns(n), n, f"round {rnd}")
    assert on.counters() == off.counters()
    on.close()
    off.close()


def test_heartbeat_resp_ignores_read_ctx():
    n = 4096
    synth, (on, off) = _step_twins(n, 0xFACE)
    rng = np.random.default_rng(7)
    for _ in range(3):
        cells = rng.choice(n * 5, n * 2, replace=False)
        hb = np.zeros(len(cells), B.APPEND_RESP_DTYPE)
        hb["group"], hb["peer_slot"] = cells // 5, cells % 5
        hb["flags"] = B.REC_HEARTBEAT
        hb["commit"] = rng.integers(0, 1 << 20, len(cells))
        with_ctx = hb.copy()
        with_ctx["flags"] |= B.REC_READ_CTX
        with_ctx["index"] = rng.integers(1, n, len(cells))
        r_off = off.heartbeat_resp(hb)
        r_on = on.heartbeat_resp(with_ctx)
        assert np.array_equal(r_on, r_off)
        assert_columns_equal(on.read_columns(n), off.read_columns(n), n, "heartbeat")
        on.read_index_ack(with_ctx)     # the read pass over the same records leaves the tracker columns alone
        assert_columns_equal(on.read_columns(n), off.read_columns(n), n, "read pass")
    on.close()
    off.close()
