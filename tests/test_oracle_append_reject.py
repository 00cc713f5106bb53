"""The leader's side of a rejected MsgAppendResponse on the oracle (oracle/leader_runs_oracle.c): find_conflict_by_term
(raft_log.rs:209-235) on the whole term array (the literal form) against the device rule over the arena and a row of at
most two earlier term runs (the batch form), and the setter's row check."""
import numpy as np
import pytest

from helpers import B, O
from oracle import leader_runs_oracle as LR
import app_follow as A
import append_reject as R

# test_raft.rs:5574 (test_fast_log_rejection), the leader's side: (leader log terms, the follower's log_term, its
# reject_hint, next_append_term, next_append_index)
FAST_LOG_REJECTION = [
    ([1, 2, 2, 4, 4, 4, 4], 3, 7, 2, 3),
    ([1, 2, 2, 3, 4, 4, 4, 5], 3, 8, 3, 4),
    ([1, 1, 1, 1], 1, 1, 1, 1),
    ([1, 1, 1, 1, 1, 1], 1, 1, 1, 1),
    ([1, 1, 1, 1], 1, 1, 1, 1),
    ([1, 1, 1, 4, 5], 4, 4, 4, 4),
    ([2, 5, 5, 5, 5, 5, 5, 5, 5], 4, 6, 2, 1),
    ([2, 2, 2, 2, 2], 2, 1, 2, 1),
]


@pytest.mark.parametrize("n_runs, decided", [(0, []), (1, [2, 3, 4, 7]), (2, [0, 2, 3, 4, 5, 6, 7])])
def test_fast_log_rejection_leader_probe(n_runs, decided):
    """Every case of test_fast_log_rejection: the follower's (reject_hint, log_term) reaches the leader, which has
    appended its become_leader entry.  The reference's leader is at term 1 after become_candidate, so that entry's term
    is 1; the walk never reaches it, and a leader at a term above its log gives the same probe.  The literal form gives
    the reference's next probe (its index and the leader's term there).  The batch form, with the runs the leader's log
    implies, gives the same probe in the cases it decides, and leaves the others NEEDS_LOG."""
    got = []
    for k, (leader, lt, hint, wterm, windex) in enumerate(FAST_LOG_REJECTION):
        for own in (1, max(leader) + 1):
            terms = [0] + leader + [own]
            probe = LR.find_conflict_by_term(terms, 1, hint, lt)
            assert (probe, terms[probe]) == (windex, wterm), k
        terms = [0] + leader + [max(leader) + 1]
        term, ts, runs = LR.runs_of_log(terms, 1, n_runs)
        assert len(runs) == min(n_runs, len(set(leader)))
        # through the frames: one leader, the follower at slot 1 probing at next_idx = last_index + 1 = the rejected index
        c = R.leader_columns([terms], 8)
        c.next_idx[1, 0] = len(leader) + 1
        rows = np.zeros(8, LR.ROW_DTYPE)
        rows[0] = LR.row(0, term, ts, runs)
        blob, off = A.batch([A.frame(0, 1, R.response(term, index=len(leader), reject=True, hint=hint, log_term=lt))])
        st, _, h, _ = LR.decode_batch(c, rows, blob, off)
        lst, _, lh, _ = LR.literal_batch([terms], [1], [term], blob, off)
        assert lst[0] == O.WIRE_OK and lh[0] == windex
        if st[0] == O.WIRE_OK:
            assert h[0] == windex
            R.oracle_step(c, rows, blob, off)
            # maybe_decr_to: next_idx = min(rejected, hint + 1); the next MsgAppend goes at index next_idx - 1
            assert int(c.next_idx[1, 0]) - 1 == windex and terms[windex] == wterm
            got.append(k)
        else:
            assert st[0] == O.WIRE_NEEDS_LOG
    assert got == decided


def _hints(terms, first_index):
    """Every hint the random test tries: 0, each run's edges and inside, last_index, above it."""
    last = len(terms) - 1
    hs = {0, 1, last, last + 1, last + 7, max(first_index - 1, 0), first_index}
    for i in range(1, last + 1):
        if terms[i] != terms[i - 1] or i == last or (i + 1 <= last and terms[i + 1] != terms[i]):
            hs.update({i - 1, i, i + 1})
    return sorted(h for h in hs if h >= 0)


def test_batch_form_agrees_with_the_literal_walk_on_random_leaders():
    """Random leader logs of 1-6 term runs, some compacted (first_index > 1, the rows restated so that every run is at
    or above first_index - 1), hints at 0, inside and at the edges of every run, at last_index and above, log terms below,
    at and above every run's term: wherever the batch form decides, at 0, 1 or 2 stated runs, its next probe is the
    literal form's.  Stale and mismatched anchors decide nothing."""
    rng = np.random.default_rng(0xB0B)
    decided = {0: 0, 1: 0, 2: 0}
    total = 0
    for trial in range(300):
        terms = R.random_log(rng, int(rng.integers(1, 7)))
        last = len(terms) - 1
        fi = 1 if trial % 3 else int(rng.integers(1, last + 1))
        lit = [0 if i + 1 < fi else t for i, t in enumerate(terms)]  # what RaftLog::term reads below first_index - 1
        term_vals = sorted(set(terms))
        lts = sorted({max(1, t + d) for t in term_vals for d in (-1, 0, 1)})
        for n_runs in (0, 1, 2):
            term, ts, runs = LR.runs_of_log(terms, fi, n_runs)
            for s, t in runs:
                assert s >= fi - 1 and all(terms[i] == t for i in range(s, (runs[runs.index((s, t)) - 1][0] if runs.index((s, t)) else ts)))
            r = LR.row(0, term, ts, runs)
            assert LR.row_status(r) == 0
            for h in _hints(terms, fi):
                for lt in lts:
                    want = LR.find_conflict_by_term(lit, fi, h, lt)
                    got = LR.probe_by_runs(term, ts, last, r, h, lt)
                    total += n_runs == 0
                    if got is not None:
                        assert got == want, (terms, fi, runs, h, lt)
                        decided[n_runs] += 1
                    # a stale anchor (another term or term_start), no row, a follower: undecided
                    assert LR.probe_by_runs(term + 1, ts, last, r, h, lt) is None
                    assert LR.probe_by_runs(term, ts + 1, last, r, h, lt) is None
                    assert LR.probe_by_runs(term, ts, last, None, h, lt) is None
                    assert LR.probe_by_runs(term, LR.NO_TERM_START, last, r, h, lt) is None
    assert decided[0] < decided[1] < decided[2] < total


def test_batch_form_through_frames_against_the_literal_form():
    """Frames of 200 random leaders, several per cell: accepts, rejections with log_term 0 and > 0, term mismatches,
    other types.  The batch form's statuses equal the literal form's except for the rejections it leaves NEEDS_LOG, which
    claim no cell (a later frame of that cell then goes first); every decided hint equals the literal one."""
    rng = np.random.default_rng(7)
    n = 200
    logs = [R.random_log(rng, int(rng.integers(1, 7))) for _ in range(n)]
    c = R.leader_columns(logs, n)
    rows = R.rows_for(logs, np.ones(n, np.uint64), 2)
    frames = []
    for _ in range(1500):
        g = int(rng.integers(0, n))
        last = len(logs[g]) - 1
        k = int(rng.integers(0, 6))
        term = int(c.term[g]) if k else int(c.term[g]) + 1
        body = R.response(term, index=int(rng.integers(0, last + 2)), reject=k >= 3, hint=int(rng.integers(0, last + 3)),
                          log_term=int(rng.integers(0, 40)) if k >= 4 else 0, commit=int(rng.integers(0, last + 1)))
        frames.append(A.frame(g, int(rng.integers(1, 5)), body))
    blob, off = A.batch(frames)
    st, recs, h, _ = LR.decode_batch(c, rows, blob, off)
    lst, lrecs, lh, _ = LR.literal_batch(logs, np.ones(n), c.term[:n], blob, off)
    needs = st == O.WIRE_NEEDS_LOG
    assert needs.any() and (st == O.WIRE_OK).sum() > 100
    # without undecided frames the two agree frame for frame
    keep = np.nonzero(~needs)[0]
    frames2 = [frames[i] for i in keep]
    blob2, off2 = A.batch(frames2)
    st2, _, h2, _ = LR.decode_batch(c, rows, blob2, off2)
    lst2, _, lh2, _ = LR.literal_batch(logs, np.ones(n), c.term[:n], blob2, off2)
    assert np.array_equal(st2, lst2) and np.array_equal(h2[st2 == 0], lh2[lst2 == 0])
    # without rows: exactly the wire oracle's statuses
    st0, _, h0, _ = LR.decode_batch(c, None, blob, off)
    wst, _, wh, _ = O.wire_decode_batch(blob, off, n, c.term[:n].copy())
    assert np.array_equal(st0, wst) and np.array_equal(h0, wh)


def test_row_check_refusals():
    """The setter's refusals, row by row."""
    ok = LR.row(0, 9, 20, [(10, 5), (4, 2)])
    assert LR.row_status(ok) == 0
    assert LR.row_status(LR.row(0, 9, 20)) == 0
    assert LR.row_status(LR.row(0, 9, 20, [(1, 8)])) == 0
    assert LR.row_status(ok, allocated=False) == B.ERR_RANGE
    assert LR.row_status(ok, wide_hi=True) == B.ERR_RANGE
    bad = [LR.row(0, 0, 20), LR.row(0, 9, 0), LR.row(0, 9, LR.NO_TERM_START),
           LR.row(0, 9, 20, [(0, 0), (4, 2)]),                       # run 2 without run 1
           LR.row(0, 9, 20, [(20, 5)]), LR.row(0, 9, 20, [(25, 5)]),  # run 1 not below term_start
           LR.row(0, 9, 20, [(10, 5), (10, 2)]), LR.row(0, 9, 20, [(10, 5), (12, 2)]),
           LR.row(0, 9, 20, [(10, 0)]), LR.row(0, 9, 20, [(10, 9)]), LR.row(0, 9, 20, [(10, 12)]),
           LR.row(0, 9, 20, [(10, 5), (4, 5)]), LR.row(0, 9, 20, [(10, 5), (4, 0)]), LR.row(0, 9, 20, [(10, 5), (4, 7)])]
    for r in bad:
        assert LR.row_status(r) == B.ERR_INVALID, r
