"""GPU parity of the wire step on arenas with leader runs (raftgpu_arena_enable_leader_runs, raftgpu_leader_runs_set):
rejected MsgAppendResponse frames with log_term > 0 decided on the device, against the oracle's batch form
(oracle/leader_runs_oracle.c) applied through the records every wire test uses, byte for byte: statuses and every
column.  Random 100K-leader arenas with and without runs in both step forms, stale anchors and the setter's refusals,
wide pairs, the edges of the 16-bit next_idx window, the setter between raftgpu_step_begin_wire and its wait, and the
round trip after a store-wide election against the literal walk."""
import importlib
import json
import os

import numpy as np
import pytest

from helpers import B, O, assert_columns_equal
from oracle import leader_runs_oracle as LR
from oracle import app_entries_oracle as AE
from oracle import app_follow_oracle as AL
import app_entries as E
import app_follow as A
import append_reject as R
import pass_forms as PF

pytestmark = pytest.mark.gpu

W = importlib.import_module("raft-rs_b200.wire")
HERE = os.path.dirname(os.path.abspath(__file__))


def _random_batch(rng, logs, c, n_frames, golden=True):
    n = len(logs)
    frames = []
    for _ in range(n_frames):
        g = int(rng.integers(0, n))
        last = len(logs[g]) - 1
        k = int(rng.integers(0, 8))
        term = int(c.term[g]) if k else int(c.term[g]) + 1
        idx = int(c.next_idx[1, g]) - 1 if k >= 4 and rng.random() < 0.7 else int(rng.integers(0, last + 2))
        body = R.response(term, index=idx, reject=k >= 3, hint=int(rng.integers(0, last + 3)),
                          log_term=int(rng.integers(1, 40)) if k >= 4 else 0, commit=int(rng.integers(0, last + 1)),
                          snap=int(rng.integers(1, 5)) if k == 7 and rng.random() < 0.2 else 0)
        frames.append(A.frame(g, int(rng.integers(1, 6)), body))
    if golden:
        with open(os.path.join(HERE, "golden", "wire", "append_responses.json")) as f:
            for i, v in enumerate(json.load(f)["responses"]):
                frames.append(A.frame(int(rng.integers(0, n)), 1 + i % 7, bytes.fromhex(v["hex"])))
    frames.append(b"\x01\x02")                                        # hostile: shorter than the header
    frames.append(A.frame(n + 5, 1, R.response(1)))                  # a group past the arena
    frames.append(A.frame(0, 1, b"\x08\x04\x28"))                     # truncated varint
    return A.batch(frames)


def _leaders(rng, n):
    logs = [R.random_log(rng, int(rng.integers(1, 7))) for _ in range(n)]
    c = R.leader_columns(logs, n, seed=int(rng.integers(0, 1 << 30)))
    # a mix of 0, 1 and 2 stated runs
    rows = np.zeros(n, LR.ROW_DTYPE)
    for k in range(3):
        sel = np.arange(k, n, 3)
        rows[sel] = R.rows_for([logs[g] for g in sel], np.ones(len(sel)), k)
    rows["group"] = np.arange(n)
    return logs, c, rows


def test_random_leaders_host_and_device_forms_against_the_oracle():
    """100K leaders with 1-6 term runs and 0-2 stated runs; a batch of accepts, rejections with log_term 0 and > 0
    (most at the probe's index), term mismatches, several frames per cell, the golden response vectors and hostile
    frames.  The twin without runs gives exactly the wire oracle's statuses; the arena with runs the batch form's, both
    through raftgpu_wire_apply_device and raftgpu_step_begin_wire."""
    rng = np.random.default_rng(0xA11)
    n = 100_000
    logs, c, rows = _leaders(rng, n)
    blob, off = _random_batch(rng, logs, c, 300_000)
    with_runs, without = R.leader_arena(c, n, True), R.leader_arena(c, n, False)
    assert (with_runs.leader_runs_set(rows) == 0).all()
    ref, ref0 = O.copy_columns(c), O.copy_columns(c)
    want = R.oracle_step(ref, rows, blob, off)
    want0 = R.oracle_step(ref0, None, blob, off)
    got = PF.device(with_runs, "wire_apply", blob, off)[0]
    got0 = PF.device(without, "wire_apply", blob, off)[0]
    assert np.array_equal(got0, want0)
    bad = np.nonzero(got != want)[0]
    assert len(bad) == 0, [(int(i), hex(got[i]), hex(want[i])) for i in bad[:5]]
    assert_columns_equal(with_runs.read_columns(n), ref, n, "runs, device form")
    assert_columns_equal(without.read_columns(n), ref0, n, "no runs, device form")
    decided = ((want0 >> 4) == B.WIRE_NEEDS_LOG) & ((want >> 4) == B.WIRE_OK)
    assert decided.sum() > 10_000 and ((want >> 4) == B.WIRE_NEEDS_LOG).sum() > 1_000
    # the host form on the arena with runs: a second batch, then Raft::maybe_commit
    blob2, off2 = _random_batch(rng, logs, c, 200_000, golden=False)
    frames = [bytes(blob2[off2[i]:off2[i + 1]]) for i in range(len(off2) - 1)]
    wb = W.WireBuffers(with_runs, len(frames) + 8, bytes_per_record=64)
    wb.set_frames(frames)
    with_runs.step_begin_wire(wb, B.STEP_READ_COMMITTED)
    with_runs.step_wait()
    want2 = R.oracle_step(ref, rows, wb.bytes[: wb.n_bytes], wb.offsets[: wb.n + 1])
    O.arena_recompute(ref)
    assert np.array_equal(with_runs.wire_status().copy(), want2)
    assert_columns_equal(with_runs.read_columns(n), ref, n, "runs, host form")
    wb.free()
    for a in (with_runs, without):
        a.close()


def test_stale_anchors_and_refusals():
    """A row is inert once its group's (term, term_start) moves: reset, become_leader, set_log_bounds, a term bump, a
    free / alloc cycle (which also clears the row); a row restated for the new anchor decides again.  Statuses and
    columns against the oracle on the arena's own columns.  The setter's refusals are the oracle's row check."""
    n = 64
    logs = [[0, 1, 1, 3, 3, 3, 5, 5, 7, 7, 7] for _ in range(n)]
    c = R.leader_columns(logs, n)
    a = R.leader_arena(c, n, True)
    rows = R.rows_for(logs, np.ones(n), 2)
    assert (a.leader_runs_set(rows) == 0).all()
    a.group_reset(1, 9, 10, 0, 0)
    a.group_become_leader(2)
    a.group_set_log_bounds(3, 9, 10)
    a.group_set_term(4, 8)
    a.group_free(5)
    assert a.group_alloc() == 5
    a.group_set_log_bounds(5, 8, 10)                # the old anchor again, but the row was cleared
    rows[5] = np.zeros(1, LR.ROW_DTYPE)[0]
    a.group_reset(6, 9, 10, 0, 0)                   # moved, then restated for its new anchor
    rows[6] = LR.row(6, 7, 9, [(6, 5), (3, 3)])
    assert (a.leader_runs_set(rows[6:7]) == 0).all()
    ref = a.read_columns(n)
    ref.term[:n] = a.column_read(B.COL_TERM, 0, 0, n, np.uint64)
    assert int(ref.term[4]) == 8
    # rejected at the probe's index with (hint 9, log_term 4): on the stated log the walk goes 9 (7), 7 (5), 5 (3) -> 5
    frames = [A.frame(g, 1, R.response(int(ref.term[g]), index=max(int(ref.next_idx[1, g]) - 1, 0), reject=True, hint=9,
                                       log_term=4)) for g in range(n)]
    blob, off = A.batch(frames)
    want = R.oracle_step(ref, rows, blob, off)
    got = PF.device(a, "wire_apply", blob, off)[0]
    assert np.array_equal(got, want), [(g, hex(got[g]), hex(want[g])) for g in range(n) if got[g] != want[g]]
    st = got >> 4
    assert (st[[1, 2, 3, 4, 5]] == B.WIRE_NEEDS_LOG).all() and st[0] == B.WIRE_OK and (st[6:] == B.WIRE_OK).all()
    assert_columns_equal(a.read_columns(n), ref, n, "stale anchors")
    assert int(ref.next_idx[1, 0]) == 6
    # refusals
    bad = np.array([LR.row(n + 3, 7, 9), LR.row(0, 0, 9), LR.row(0, 7, 9, [(9, 5)]), LR.row(0, 7, 9, [(5, 5), (6, 3)]),
                    LR.row(0, 7, 9, [(5, 7)]), LR.row(0, 7, 9, [(0, 0), (2, 1)])], LR.ROW_DTYPE)
    st = a.leader_runs_set(bad)
    assert st.tolist() == [B.ERR_RANGE] + [B.ERR_INVALID] * 5
    assert st.tolist() == [LR.row_status(r, allocated=r["group"] < n) for r in bad]
    plain = B.Arena(8)
    with pytest.raises(Exception):
        plain.leader_runs_set(bad[:1])
    plain.close()
    a.close()


# --------------------------------------------------------------------------- wide pairs

WIDE_LO, WIDE_HI = 0x20000000, 0x40000000  # RAFTGPU_META_WIDE_LO / _HI


def test_wide_pairs():
    """Leaders of 2 000 narrow groups and 1 000 wide pairs, frames to both halves of every pair (peer 8 + s is cell
    (g + 1, s)).  A pair reads its low half's row with the larger last_index of its halves: half the pairs have the
    larger one on the high half, and hints fall between the two.  A row stated on a high half is refused."""
    rng = np.random.default_rng(0x3A1D)
    n_narrow, n_wide = 2_000, 1_000
    n = n_narrow + 2 * n_wide
    a = B.Arena(n + 64)
    a.enable_leader_runs()
    assert a.group_alloc_range(n_narrow) == 0
    for g in range(n_narrow):
        a.group_set_conf(g, 0x1F, 0, 0, 0, 1)            # 5 voters, self slot 0
    for k in range(n_wide):
        g = a.group_alloc_wide()
        assert g == n_narrow + 2 * k
        a.group_set_conf(g, 0x0707, 0, 0, 0, 1)          # voters: slots 0-2 of each half, self slot 0
    logs = [R.random_log(rng, int(rng.integers(2, 7))) for _ in range(n)]
    for k in range(n_wide):                              # a pair is one leader: one log, on its low half
        logs[n_narrow + 2 * k + 1] = logs[n_narrow + 2 * k]
    term = np.array([t[-1] for t in logs], np.uint64)
    ts = np.array([LR.runs_of_log(t, 1, 0)[1] for t in logs], np.uint64)
    top = np.array([len(t) - 1 for t in logs], np.uint64)   # the group's (the pair's) last_index
    hi = np.arange(n_narrow + 1, n, 2)
    # one half of a pair holds top, the other lags by 0-5 (not below term_start)
    last = top.copy()
    lag = np.minimum(rng.integers(0, 6, n_wide).astype(np.uint64), top[hi] - ts[hi])
    on_hi = rng.random(n_wide) < 0.5
    last[hi - 1] = np.where(on_hi, top[hi] - lag, top[hi])
    last[hi] = np.where(on_hi, top[hi], top[hi] - lag)
    assert (lag > 0).sum() > 100
    for col, arr in ((B.COL_TERM, term), (B.COL_TERM_START, ts), (B.COL_LAST_INDEX, last)):
        a.column_write(col, 0, 0, arr)
    for s in range(B.SLOTS):
        a.column_write(B.COL_NEXT_IDX, s, 0, top + 1)
    rows = R.rows_for(logs, np.ones(n), 2, cap=n)
    rows_hi = rows[hi].copy()
    rows[hi] = np.zeros(len(hi), LR.ROW_DTYPE)
    assert (a.leader_runs_set(rows[:n_narrow]) == 0).all()
    assert (a.leader_runs_set(rows[hi - 1]) == 0).all()
    assert (a.leader_runs_set(rows_hi) == B.ERR_RANGE).all()      # a pair's row lives on its low half
    c = a.read_columns(n)
    c.term = a.column_read(B.COL_TERM, 0, 0, n, np.uint64)
    assert ((c.meta[hi] & WIDE_HI) != 0).all() and ((c.meta[hi - 1] & WIDE_LO) != 0).all()
    frames = []
    for _ in range(40_000):
        g = int(rng.integers(0, n))
        lo = g - 1 if c.meta[g] & WIDE_HI else g
        tp = int(top[g])
        h = int(rng.integers(max(int(ts[lo]) - 1, 0), tp + 2)) if rng.random() < 0.5 else int(rng.integers(0, tp + 2))
        lt = int(rng.integers(1, int(term[lo]) + 1))
        reject = rng.random() < 0.8
        frames.append(A.frame(g, int(rng.integers(1, 3)), R.response(int(term[g]), index=tp, reject=reject, hint=h,
                                                                      log_term=lt if reject else 0)))
    blob, off = A.batch(frames)
    want = R.oracle_step(c, rows, blob, off)
    got = PF.device(a, "wire_apply", blob, off)[0]
    bad = np.nonzero(got != want)[0]
    assert len(bad) == 0, [(int(i), hex(got[i]), hex(want[i])) for i in bad[:5]]
    assert_columns_equal(a.read_columns(n), c, n, "wide pairs")
    hdr = np.array([int.from_bytes(f[:4], "little") >> 4 for f in frames])
    rej = np.array([O.wire_decode_message(f[4:])["reject"] for f in frames], bool)
    decided = ((want >> 4) == B.WIRE_OK) & rej
    assert (decided & np.isin(hdr, hi)).sum() > 1_000 and (decided & np.isin(hdr, hi - 1)).sum() > 1_000
    assert ((want >> 4) == B.WIRE_NEEDS_LOG).sum() > 100
    a.close()


# --------------------------------------------------------------------------- the 16-bit next_idx window

def test_next_idx_offset_window_edges():
    """next_idx is stored as a 16-bit offset from matched, escaped outside [-32767, 32767] (k_common.cuh).  Probing
    cells whose next_idx sits at the window's edges take decided rejections whose new next_idx lands at each edge, above
    and below matched, through the leader's own segment and through a stated run.  Columns (the u64 values the codec
    decodes) against the oracle."""
    M, W = 1_000_000, 32767
    edges = [W - 1, W, W + 1, W + 2]
    starts = [M + d for d in edges] + [M - d for d in edges] + [M + 5]        # next_idx before the frame
    targets = [M + d for d in edges] + [M - d for d in edges] + [M + 1]       # next_idx the decision leads to
    cases = [(n0, t) for n0 in starts for t in targets if t < n0]
    n = len(cases)
    term, ts, rt0 = 9, M + 20_000, 4
    c = O.new_columns(n, n)
    c.term[:n], c.term_start[:n], c.last_index[:n] = term, ts, M + 50_000
    c.meta[:n] = O.make_meta(0x1F, self_slot=0)
    c.matched[1, :n] = M
    a = B.Arena(n)
    a.enable_leader_runs()
    assert a.group_alloc_range(n) == 0
    frames = []
    for g, (n0, t) in enumerate(cases):
        c.next_idx[1, g] = n0
        # the decided conflict index is t - 1: through the top segment (log_term >= term) when t - 1 >= term_start,
        # else through run 1 = [1, term_start - 1] at rt0 (log_term = rt0)
        lt = term if t - 1 >= ts else rt0
        frames.append(A.frame(g, 1, R.response(term, index=n0 - 1, reject=True, hint=t - 1, log_term=lt)))
    a.load_columns(c)
    a.column_write(B.COL_TERM, 0, 0, c.term[:n].copy())
    rows = np.zeros(n, LR.ROW_DTYPE)
    for g in range(n):
        rows[g] = LR.row(g, term, ts, [(1, rt0)])
    assert (a.leader_runs_set(rows) == 0).all()
    blob, off = A.batch(frames)
    want = R.oracle_step(c, rows, blob, off)
    assert ((want >> 4) == B.WIRE_OK).all()
    got = PF.device(a, "wire_apply", blob, off)[0]
    assert np.array_equal(got, want)
    got_c = a.read_columns(n)
    assert_columns_equal(got_c, c, n, "offset window edges")
    assert sorted(set(int(x) - M for x in c.next_idx[1, :n])) == sorted(set(t - M for _, t in cases))
    a.close()


# --------------------------------------------------------------------------- the setter with steps in flight

def test_setter_between_begin_and_wait():
    """raftgpu_leader_runs_set between raftgpu_step_begin_wire and its wait takes effect in submission order: the step
    begun before it sees the old rows (none: its rejections stay NEEDS_LOG), the step begun after it the new ones.
    Statuses and columns against the oracle, step by step, with Raft::maybe_commit after each."""
    rng = np.random.default_rng(0x5E7)
    n = 20_000
    logs = [R.random_log(rng, int(rng.integers(2, 7))) for _ in range(n)]
    c = R.leader_columns(logs, n)
    a = R.leader_arena(c, n, True)
    rows = R.rows_for(logs, np.ones(n), 2)
    none = np.zeros(n, LR.ROW_DTYPE)
    ref = O.copy_columns(c)

    def batch(slot):
        fr = []
        for g in range(n):
            last = len(logs[g]) - 1
            fr.append(A.frame(g, slot, R.response(int(c.term[g]), index=last, reject=True,
                                                  hint=int(rng.integers(0, last + 1)), log_term=int(rng.integers(1, 40)))))
        wb = W.WireBuffers(a, len(fr) + 8, bytes_per_record=64)
        wb.set_frames(fr)
        return wb

    wa, wb2 = batch(1), batch(2)
    a.step_begin_wire(wa, B.STEP_READ_COMMITTED)
    assert (a.leader_runs_set(rows) == 0).all()
    a.step_begin_wire(wb2, B.STEP_READ_COMMITTED)
    a.step_wait()
    want_a = R.oracle_step(ref, none, wa.bytes[: wa.n_bytes], wa.offsets[: wa.n + 1])
    O.arena_recompute(ref)
    assert np.array_equal(a.wire_status().copy(), want_a)
    assert ((want_a >> 4) == B.WIRE_NEEDS_LOG).all()
    a.step_wait()
    want_b = R.oracle_step(ref, rows, wb2.bytes[: wb2.n_bytes], wb2.offsets[: wb2.n + 1])
    O.arena_recompute(ref)
    assert np.array_equal(a.wire_status().copy(), want_b)
    assert ((want_b >> 4) == B.WIRE_OK).sum() > n // 4
    assert_columns_equal(a.read_columns(n), ref, n, "setter in flight")
    wa.free(), wb2.free()
    a.close()


# --------------------------------------------------------------------------- the round trip after an election

def _follower_log(rng, leader, ts):
    """A follower of a leader whose log is `leader` (terms, entry 0 first; the leader's own entry at ts): it holds the
    leader's log up to ts - 1 but for its last 0-3 term runs, of which it may keep a part, and may then carry a
    divergent tail of terms the leader never had."""
    starts = [i for i in range(1, ts) if leader[i] != leader[i - 1]]          # the first index of each earlier run
    d = int(rng.integers(0, min(3, len(starts) - 1) + 1))
    if d == 0:
        return list(leader[:ts])
    cut = starts[len(starts) - d]                                             # the first run the follower misses
    end = starts[len(starts) - d + 1] if d > 1 else ts                        # where that run ends (+1)
    out = list(leader[:cut]) + list(leader[cut: cut + int(rng.integers(0, end - cut))])   # maybe a part of it
    if rng.random() < 0.5:                                                    # a divergent tail
        lo = out[-1]
        taken = set(leader)
        free = [t for t in range(lo + 1, leader[ts]) if t not in taken]
        if free:
            out += [int(rng.choice(free))] * int(rng.integers(1, 5))
    return out


def test_round_trip_after_an_election_100k_x5():
    """100K groups x 5 peers after a store-wide election: every leader has just appended its empty entry at term_start
    and states its last two earlier runs; every follower lags by 0-3 of the leader's term runs or diverges.  The leader's
    probes (index = term_start - 1, the empty entry) go through raftgpu_follower_append_entries on the device, one
    follower arena per slot; the frames that pass hands back as NEEDS_LOG are answered on the host by the reference's
    rule.  All responses go back as one wire batch through raftgpu_step_begin_wire on the leader arena with runs: the
    NEEDS_LOG frames there are exactly those the oracle's batch form leaves undecided.  Those are resolved by the literal
    find_conflict_by_term and submitted as REJECT + EXT records with the next step.  Then every cell's next_idx, state
    and paused equal the literal oracle's, which walks each leader's whole log."""
    rng = np.random.default_rng(0xE1EC)
    n, P = 100_000, 5
    leaders = []
    for g in range(n):
        t = R.random_log(rng, int(rng.integers(2, 7)))
        leaders.append(t + [t[-1] + int(rng.integers(1, 4))])                 # become_leader's empty entry
    term = np.array([t[-1] for t in leaders], np.uint64)
    ts = np.array([len(t) - 1 for t in leaders], np.uint64)
    c = O.new_columns(n, n)
    c.term[:n], c.term_start[:n], c.last_index[:n] = term, ts, ts
    c.meta[:n] = O.make_meta((1 << P) - 1, self_slot=0)
    c.next_idx[:, :n] = ts                                                   # reset(): last_index + 1 before the append
    c.matched[0, :n] = ts
    la = R.leader_arena(c, n, True)
    rows = R.rows_for(leaders, np.ones(n), 2)
    assert (la.leader_runs_set(rows) == 0).all()
    ids = rng.integers(1, 1 << 40, (P, n), dtype=np.uint64)
    resp_frames = []
    needs_host = 0
    for sl in range(1, P):
        flogs = [_follower_log(rng, leaders[g], int(ts[g])) for g in range(n)]
        fl_last = np.array([len(f) - 1 for f in flogs], np.uint64)
        fc = O.new_columns(n, n)
        fc.term_start[:] = A.NO_TERM_START
        fc.term[:n], fc.last_index[:n] = term, fl_last
        table = np.zeros(n, AL.LOG_DTYPE)
        table["id"], table["flags"] = ids[sl], AL.SELECT
        for g, f in enumerate(flogs):
            table["run_start"][g], table["run_term"][g] = A.run_of(np.array(f, np.uint64), len(f) - 1)
        probes = []
        for g in range(n):
            i0 = int(ts[g]) - 1
            probes.append(A.frame(g, sl, E.message(int(term[g]), leaders[g][i0], i0, 0, int(ids[0, g]),
                                                    [E.record(E.entry(int(term[g]), i0 + 1))], to=int(ids[sl, g]))))
        fblob, foff = A.batch(probes)
        fa = B.Arena(n)
        assert fa.group_alloc_range(n) == 0
        for col, name in ((B.COL_TERM, "term"), (B.COL_LAST_INDEX, "last_index"), (B.COL_COMMITTED, "committed"),
                          (B.COL_TERM_START, "term_start")):
            fa.column_write(col, 0, 0, getattr(fc, name)[:n].copy())
        want_table = table.copy()
        w = AE.batch(fc, None, want_table, fblob, foff)
        got = PF.device(fa, "follower_append_entries", fblob, foff, table)
        PF.equal(w, tuple(got[:2]) + (got[2].view(AE.APPENDED_DTYPE),) + tuple(got[3:]), E.NAMES, ("slot", sl))
        fa.close()
        st = w[0] >> 4
        assert set(np.unique(st).tolist()) <= {B.WIRE_OK, B.WIRE_NEEDS_LOG}
        resp_frames += [bytes(w[3][a0:b0]) for a0, b0 in zip(w[4][:-1].tolist(), w[4][1:].tolist())]
        for g in np.flatnonzero(st == B.WIRE_NEEDS_LOG).tolist():             # handle_append_entries on the host
            f, i0 = flogs[g], int(ts[g]) - 1
            hint = LR.find_conflict_by_term(f, 1, min(i0, len(f) - 1), leaders[g][i0])
            resp_frames.append(A.frame(g, sl, R.response(int(term[g]), index=i0, reject=True, hint=hint,
                                                         log_term=int(f[hint]), frm=int(ids[sl, g]))))
            needs_host += 1
    assert needs_host > 1_000
    blob, off = A.batch(resp_frames)
    # the literal oracle: the reference's walk over each leader's whole log, every frame applied
    lit = O.copy_columns(c)
    lst, lrecs, lhint, lsnap = LR.literal_batch(leaders, np.ones(n), term, blob, off)
    assert (lst == O.WIRE_OK).all()
    seq = []
    for i in range(len(lst)):
        seq.append(tuple(lrecs[i]))
        if lrecs["flags"][i] & B.REC_REJECT:
            seq.append((lrecs["group"][i], lrecs["peer_slot"][i], B.REC_EXT, 0, lhint[i], lsnap[i]))
    O.arena_apply(lit, np.array(seq, B.APPEND_RESP_DTYPE), mode=0)
    # the leader arena: one wire step, then the NEEDS_LOG frames as records
    ref = O.copy_columns(c)
    want = R.oracle_step(ref, rows, blob, off)
    O.arena_recompute(ref)
    la.step_begin_wire(PF.host_batch(blob, off, len(blob)), B.STEP_READ_COMMITTED)
    la.step_wait()
    got = la.wire_status().copy()
    assert np.array_equal(got, want)
    undecided = np.flatnonzero((got >> 4) == B.WIRE_NEEDS_LOG)
    bst, _, _, _ = LR.decode_batch(c, rows, blob, off)
    assert np.array_equal(undecided, np.flatnonzero(bst == O.WIRE_NEEDS_LOG))
    rej = np.array([O.wire_decode_message(f[4:])["reject"] for f in resp_frames], bool)
    assert len(undecided) > 1_000 and ((got >> 4) == B.WIRE_OK)[rej].sum() > 50_000
    recs = []
    for i in undecided.tolist():
        recs.append(tuple(lrecs[i]))
        recs.append((lrecs["group"][i], lrecs["peer_slot"][i], B.REC_EXT, 0, lhint[i], lsnap[i]))
    rb = PF.host_batch(np.zeros(0, np.uint8), np.zeros(1, np.uint32), 0)
    rb.records = np.array(recs, B.APPEND_RESP_DTYPE)
    rb.n_records = len(rb.records)
    la.step_begin_wire(rb, B.STEP_READ_COMMITTED)
    la.step_wait()
    lc = la.read_columns(n)
    assert np.array_equal(lc.next_idx[:, :n], lit.next_idx[:, :n])
    assert np.array_equal(lc.pflags[:, :n] & 3, lit.pflags[:, :n] & 3)                        # state
    assert np.array_equal(lc.pflags[:, :n] & B.PF_PAUSED, lit.pflags[:, :n] & B.PF_PAUSED)    # paused
    assert np.array_equal(lc.matched[:, :n], lit.matched[:, :n])
    la.close()
