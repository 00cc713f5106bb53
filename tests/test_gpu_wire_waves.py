"""GPU parity of the passes at raftgpu_arena_set_wire_waves > 1 (DESIGN 3.19) against the wave oracle
(oracle/wire_waves_oracle.c), byte for byte: status bytes, from, appended records, responses, offsets, totals, the log
table and every arena column.  One wave against an arena that never called the setter; the wire step at 2, 4 and 64
waves on 100K leaders x 5 peers with and without leader runs, wide pairs, both step forms and the setter between a
begin and its wait; the follower's two append passes at 100K groups
in both forms; a round trip of k pipelined appends; and the edges: 10 000 frames of one cell, n = 0, the refusals."""
import importlib

import numpy as np
import pytest

from helpers import B, O, assert_columns_equal
from oracle import app_entries_oracle as AE
from oracle import app_follow_oracle as AL
from oracle import leader_runs_oracle as LR
from oracle import wire_waves_oracle as WW
import app_follow as A
import app_entries as E
import append_reject as R
import hb_follow as FL
import pass_forms as PF

pytestmark = pytest.mark.gpu

W = importlib.import_module("raft-rs_b200.wire")
N_LEADERS, PEERS = 100_000, range(1, 5)
WIDE_HI = 0x40000000  # RAFTGPU_META_WIDE_HI


def _leaders(seed, n=N_LEADERS):
    rng = np.random.default_rng(seed)
    logs = [R.random_log(rng, int(rng.integers(1, 7))) for _ in range(n)]
    c = R.leader_columns(logs, n, seed=seed)
    rows = np.zeros(n, LR.ROW_DTYPE)
    for k in range(3):
        sel = np.arange(k, n, 3)
        rows[sel] = R.rows_for([logs[g] for g in sel], np.ones(len(sel)), k)
    rows["group"] = np.arange(n)
    return rng, logs, c, rows


def _leader_batch(rng, c, n):
    frames = R.leader_frames(rng, c, range(n), PEERS, 6, needs_log=0.4)
    frames += [A.frame(5, 1, R.response(int(c.term[5]) + 1, index=1)), b"\x01\x02", A.frame(n + 7, 1, R.response(1)),
               A.frame(9, 2, b"\x08\x03")]                                      # TERM, hostile, another type
    return A.batch(frames)


def _step_host(a, blob, off):
    a.step_begin_wire(PF.host_batch(blob, off, len(blob)), B.STEP_READ_COMMITTED)
    a.step_wait()
    return a.wire_status().copy()


@pytest.mark.parametrize("runs", [False, True], ids=["no_runs", "runs"])
def test_leader_waves_100k_x5(runs):
    """100K leaders x 5 peers, 1-6 frames per cell (accepts, stale accepts, rejections with and without log_term,
    frames that need the log), through raftgpu_wire_apply_device at waves 2, 4 and RAFTGPU_WIRE_WAVES_MAX on one arena,
    then raftgpu_step_begin_wire at 4: statuses and columns against the wave oracle."""
    rng, logs, c, rows = _leaders(0x3A7E + runs)
    n = N_LEADERS
    a = R.leader_arena(c, n, runs)
    r = rows if runs else None
    if runs:
        assert (a.leader_runs_set(rows) == 0).all()
    ref = O.copy_columns(c)
    for waves in (2, 4, B.WIRE_WAVES_MAX):
        blob, off = _leader_batch(rng, ref, n)
        assert a.set_wire_waves(waves) == 0
        want = WW.leader(ref, r, blob, off, waves)
        got = PF.device(a, "wire_apply", blob, off)[0]
        bad = np.flatnonzero(got != want)
        assert len(bad) == 0, (waves, [(int(i), hex(got[i]), hex(want[i])) for i in bad[:5]])
        assert_columns_equal(a.read_columns(n), ref, n, f"device form, waves {waves}")
        st = want >> 4
        assert (st == B.WIRE_NEEDS_LOG).sum() > 1_000 and (st == B.WIRE_OK).sum() > 2 * n
        assert ((st == B.WIRE_DUP).sum() > 10_000) == (waves < 6)
    blob, off = _leader_batch(rng, ref, n)
    assert a.set_wire_waves(4) == 0
    want = WW.leader(ref, r, blob, off, 4)
    O.arena_recompute(ref)
    assert np.array_equal(_step_host(a, blob, off), want)
    assert_columns_equal(a.read_columns(n), ref, n, "host form")
    a.close()


def test_one_wave_is_the_arena_without_the_setter():
    """waves = 1 set explicitly gives exactly what an arena that never called the setter gives, on a batch with several
    frames per cell, in the wire step and in the follower's pass with entries."""
    rng, logs, c, rows = _leaders(0x1A1, 20_000)
    n = 20_000
    blob, off = _leader_batch(rng, c, n)
    a1, a0 = R.leader_arena(c, n, False), R.leader_arena(c, n, False)
    assert a1.set_wire_waves(5) == 0 and a1.set_wire_waves(1) == 0
    assert np.array_equal(PF.device(a1, "wire_apply", blob, off)[0], PF.device(a0, "wire_apply", blob, off)[0])
    assert_columns_equal(a1.read_columns(n), a0.read_columns(n), n, "one wave")
    a1.close(), a0.close()
    fa1, fc, _, table = E.world(rng, 20_000, 200, False)
    fa0 = E.world(np.random.default_rng(0), 20_000, 200, False)[0]
    _copy_state(fa1, fa0, fc.n_groups)
    fb, fo = _follower_batch(rng, fc, table, range(20_000), 4)
    assert fa1.set_wire_waves(1) == 0
    t1, t0 = table.copy(), table.copy()
    g1, g0 = PF.host(fa1, "follower_append_entries", fb, fo, t1), PF.host(fa0, "follower_append_entries", fb, fo, t0)
    for x, y in zip(g1, g0):
        assert np.array_equal(x, y)
    assert np.array_equal(t1, t0)
    fa1.close(), fa0.close()


def _copy_state(src, dst, n):
    for col in (B.COL_TERM, B.COL_LAST_INDEX, B.COL_COMMITTED, B.COL_TERM_START):
        dst.column_write(col, 0, 0, src.column_read(col, 0, 0, n, np.uint64))


def _follower_batch(rng, c, table, groups, per_group, entries=True, junk=True):
    """1..per_group pipelined MsgAppend frames per listed group (a pair by its low half), built from its state, the groups
    interleaved; with junk, a stale frame, a gap (NEEDS_LOG) or an over-commit (COMMIT_RANGE) in the middle of some
    groups' frames."""
    per = []
    for g in groups:
        wide = bool(c.meta[g] & E.WIDE_LO)
        last = int(max(c.last_index[g], c.last_index[g + 1])) if wide else int(c.last_index[g])
        com = int(max(c.committed[g], c.committed[g + 1])) if wide else int(c.committed[g])
        run_term, term = int(table["run_term"][g]), int(c.term[g])
        if int(table["run_start"][g]) > last or run_term > term:
            continue
        bodies = [b for b, _ in R.pipelined_appends(rng, last, run_term, term, com, int(rng.integers(1, per_group + 1)),
                                                    entries)]
        if junk and len(bodies) > 1 and rng.random() < 0.2:
            k = int(rng.integers(1, len(bodies)))
            kind = int(rng.integers(0, 3))
            if kind == 0:                                                       # stale
                bad = A.message(3, term=term, log_term=1, index=max(com, 1) - 1, commit=com, frm=3)
            elif kind == 1:                                                     # a gap: NEEDS_LOG
                bad = A.message(3, term=term, log_term=0, index=last + 50, commit=com, frm=3,
                                entries=[(term, last + 51)] if entries else None)
            else:                                                               # COMMIT_RANGE
                bad = A.message(3, term=term, log_term=0, index=last + 50, commit=last + 50, frm=3)
            bodies.insert(k, bad)
        per.append((g, [A.frame(g, int(rng.integers(16)), b) for b in bodies]))
    return A.batch(R.interleave(rng, per))


@pytest.mark.parametrize("entries", [False, True], ids=["entry_less", "entries"])
@pytest.mark.parametrize("device", [True, False], ids=["device", "host"])
def test_follower_waves_100k(entries, device):
    """100K follower groups (and 500 wide pairs), 1-6 pipelined MsgAppend frames per group, with stale, NEEDS_LOG and
    COMMIT_RANGE frames among them, at waves 3 and RAFTGPU_WIRE_WAVES_MAX: every output, the table and the group columns
    against the wave oracle."""
    rng = np.random.default_rng(0xF0 + 2 * entries + device)
    a, c, q, table = E.world(rng, E.N_NARROW, E.N_WIDE, False)
    n = c.n_groups
    lows = [g for g in range(n) if not (c.meta[g] & WIDE_HI)]
    for waves in (3, B.WIRE_WAVES_MAX):
        blob, off = _follower_batch(rng, c, table, lows, 6, entries)
        assert a.set_wire_waves(waves) == 0
        want_table = table.copy()
        want = WW.follower(c, q, want_table, blob, off, waves, entries)
        if entries:
            got = PF.run(a, "follower_append_entries", blob, off, table, device=device)
            got = tuple(got[:2]) + (got[2].view(AE.APPENDED_DTYPE),) + tuple(got[3:])
            PF.equal(want, got, E.NAMES, ("waves", waves))
            assert np.array_equal(table, want_table)
        else:
            got = PF.device(a, "follower_append", blob, off, table) if device else A.host_form(a, blob, off, table)
            PF.equal(want[:2] + want[3:], got, A.NAMES, ("waves", waves))
        for name, col in FL.group_state(a, n).items():
            assert np.array_equal(col, getattr(c, name)[:n]), (waves, name)
        st = want[0] >> 4
        assert (st == B.WIRE_COMMIT_RANGE).sum() > 100 and ((st == B.WIRE_NEEDS_LOG).sum() > 100) == entries
        assert (st == B.WIRE_DUP).sum() > 1_000 and (want[0] & B.RES_OK).sum() > len(lows)
    a.close()


def test_round_trip_k_pipelined_appends():
    """A leader arena pipelines k = 4 MsgAppend frames with entries to each follower, built from its state; the followers
    (one arena per peer slot) answer all of them in one raftgpu_follower_append_entries_device call at waves = k and the
    leader applies all k responses per cell in one raftgpu_step_begin_wire at waves = k.  Every leader's committed and
    every cell's matched, next_idx and state equal k rounds at waves = 1."""
    rng = np.random.default_rng(0x2017)
    n, P, k = 20_000, 5, 4
    term = 7
    last0 = rng.integers(10, 1000, n).astype(np.uint64)
    lc = O.new_columns(n, n)
    lc.term[:n], lc.term_start[:n], lc.last_index[:n], lc.committed[:n] = term, last0, last0, last0 - 1
    lc.meta[:n] = O.make_meta((1 << P) - 1, self_slot=0)
    lc.matched[0, :n] = last0
    for s in range(1, P):
        lc.matched[s, :n] = last0 - 1
        lc.next_idx[s, :n] = last0
        lc.pflags[s, :n] = B.STATE_REPLICATE
    cnt = rng.integers(1, 4, (n, k))                                             # entries per frame
    ends = last0[:, None] + np.cumsum(cnt, axis=1).astype(np.uint64)            # each frame's last index
    lc.last_index[:n] = ends[:, -1]
    lc.matched[0, :n] = ends[:, -1]
    ids = rng.integers(1, 1 << 40, (P, n), dtype=np.uint64)
    resp_by_round = [[] for _ in range(k)]
    for s in range(1, P):
        fc = O.new_columns(n, n)
        fc.term_start[:] = A.NO_TERM_START
        fc.term[:n], fc.last_index[:n], fc.committed[:n] = term, last0 - 1, last0 - 2
        table = np.zeros(n, AL.LOG_DTYPE)
        table["id"], table["flags"], table["run_start"], table["run_term"] = ids[s], AL.SELECT, 1, term
        frames = []
        for g in range(n):
            idx = int(last0[g]) - 1
            for j in range(k):
                ents = [(term, idx + e + 1) for e in range(int(cnt[g, j]))]
                frames.append(A.frame(g, s, A.message(3, term=term, log_term=term, index=idx, commit=int(last0[g]) - 1,
                                                      frm=int(ids[0, g]), entries=ents, to=int(ids[s, g]))))
                idx += len(ents)
        blob, off = A.batch(frames)
        fa = B.Arena(n)
        assert fa.group_alloc_range(n) == 0 and fa.set_wire_waves(k) == 0
        for col, name in ((B.COL_TERM, "term"), (B.COL_LAST_INDEX, "last_index"), (B.COL_COMMITTED, "committed"),
                          (B.COL_TERM_START, "term_start")):
            fa.column_write(col, 0, 0, getattr(fc, name)[:n].copy())
        st, frm, app, rb, ro, tot = PF.device(fa, "follower_append_entries", blob, off, table)
        fa.close()
        assert ((st >> 4) == B.WIRE_OK).all() and int(tot[0]) == n * k
        resp = [bytes(rb[x:y]) for x, y in zip(ro[:-1].tolist(), ro[1:].tolist())]
        for i, r in enumerate(resp):                                             # frame order: group g's j-th at g * k + j
            resp_by_round[i % k].append(r)
    # k rounds at one wave on a twin
    twin = R.leader_arena(lc, n, False)
    for j in range(k):
        b1, o1 = A.batch(resp_by_round[j])
        assert ((_step_host(twin, b1, o1) >> 4) == B.WIRE_OK).all()
    la = R.leader_arena(lc, n, False)
    assert la.set_wire_waves(k) == 0
    allb, allo = A.batch([r for g in range(len(resp_by_round[0])) for r in (x[g] for x in resp_by_round)])
    assert ((_step_host(la, allb, allo) >> 4) == B.WIRE_OK).all()
    got, want = la.read_columns(n), twin.read_columns(n)
    assert np.array_equal(got.committed[:n], want.committed[:n]) and (got.committed[:n] > lc.committed[:n]).all()
    for name in ("matched", "next_idx"):
        assert np.array_equal(getattr(got, name)[:, :n], getattr(want, name)[:, :n]), name
    assert np.array_equal(got.pflags[:, :n] & 3, want.pflags[:, :n] & 3)
    assert (got.matched[1:P, :n] == ends[:, -1] - 1).all()                    # (the followers began one entry behind)
    la.close(), twin.close()


def test_setter_between_begin_and_wait():
    """Two wire steps in flight with the setter called between a begin and its wait: the step begun at 1 wave keeps it,
    the one begun after the setter runs at 4 waves."""
    rng, logs, c, rows = _leaders(0x5E7, 20_000)
    n = 20_000
    a = R.leader_arena(c, n, False)
    ref = O.copy_columns(c)
    ba, bb = _leader_batch(rng, c, n), _leader_batch(rng, c, n)
    wa, wb = PF.host_batch(*ba, len(ba[0])), PF.host_batch(*bb, len(bb[0]))
    a.step_begin_wire(wa, B.STEP_READ_COMMITTED)
    assert a.set_wire_waves(4) == 0
    a.step_begin_wire(wb, B.STEP_READ_COMMITTED)
    a.step_wait()
    want_a = WW.leader(ref, None, *ba, 1)
    O.arena_recompute(ref)
    assert np.array_equal(a.wire_status().copy(), want_a)
    a.step_wait()
    want_b = WW.leader(ref, None, *bb, 4)
    O.arena_recompute(ref)
    assert np.array_equal(a.wire_status().copy(), want_b)
    assert_columns_equal(a.read_columns(n), ref, n, "setter in flight")
    a.close()


def test_wide_pairs():
    """Leaders of 2 000 narrow groups and 1 000 wide pairs, 1-5 frames per cell to both halves of every pair (accepts and
    rejections with log_term 0), at 4 waves: statuses and columns against the wave oracle."""
    rng = np.random.default_rng(0x91DE)
    n_narrow, n_wide = 2_000, 1_000
    n = n_narrow + 2 * n_wide
    a = B.Arena(n + 64)
    assert a.group_alloc_range(n_narrow) == 0
    for g in range(n_narrow):
        a.group_set_conf(g, 0x1F, 0, 0, 0, 1)
    for _ in range(n_wide):
        g = a.group_alloc_wide()
        a.group_set_conf(g, 0x0707, 0, 0, 0, 1)
    last = rng.integers(100, 1000, n).astype(np.uint64)
    hi = np.arange(n_narrow + 1, n, 2)
    last[hi] = last[hi - 1] + rng.integers(0, 3, len(hi)).astype(np.uint64)
    a.column_write(B.COL_TERM, 0, 0, np.full(n, 3, np.uint64))
    a.column_write(B.COL_TERM_START, 0, 0, last - 5)
    a.column_write(B.COL_LAST_INDEX, 0, 0, last)
    for s in range(B.SLOTS):
        a.column_write(B.COL_NEXT_IDX, s, 0, last + 1)
    c = a.read_columns(n)
    c.term = a.column_read(B.COL_TERM, 0, 0, n, np.uint64)
    cells = []
    for g in range(n):
        for s in (1, 2):
            cells.append([A.frame(g, s, R.response(3, index=int(rng.integers(0, int(last[g]) + 1)), reject=rng.random() < 0.2,
                                                   hint=int(rng.integers(0, int(last[g])))))
                          for _ in range(int(rng.integers(1, 6)))])
    blob, off = A.batch(R.interleave(rng, list(enumerate(cells))))
    assert a.set_wire_waves(4) == 0
    want = WW.leader(c, None, blob, off, 4)
    got = PF.device(a, "wire_apply", blob, off)[0]
    assert np.array_equal(got, want)
    assert ((want >> 4) == B.WIRE_DUP).sum() > 100 and ((want >> 4) == B.WIRE_OK).sum() > 4 * n
    assert_columns_equal(a.read_columns(n), c, n, "wide pairs")
    a.close()


def test_edges():
    """One cell with 10 000 frames at 4 waves: exactly 4 applied, the rest DUP; n = 0; the setter's refusals."""
    rng, logs, c, rows = _leaders(0xED6E, 64)
    a = R.leader_arena(c, 64, False)
    assert a.set_wire_waves(4) == 0
    last = int(c.last_index[3])
    frames = [A.frame(3, 1, R.response(int(c.term[3]), index=min(i, last))) for i in range(10_000)]
    blob, off = A.batch(frames)
    ref = O.copy_columns(c)
    want = WW.leader(ref, None, blob, off, 4)
    got = PF.device(a, "wire_apply", blob, off)[0]
    assert np.array_equal(got, want)
    assert ((got[:4] >> 4) == B.WIRE_OK).all() and ((got[4:] >> 4) == B.WIRE_DUP).all()
    assert_columns_equal(a.read_columns(64), ref, 64, "one cell")
    assert len(PF.device(a, "wire_apply", np.zeros(16, np.uint8), np.zeros(1, np.uint32))[0]) == 0
    for bad in (0, B.WIRE_WAVES_MAX + 1, 1 << 31):
        assert a.set_wire_waves(bad) == B.ERR_INVALID
    assert B.lib().raftgpu_arena_set_wire_waves(None, 2) == B.ERR_INVALID
    assert a.set_wire_waves(B.WIRE_WAVES_MAX) == 0
    a.close()
