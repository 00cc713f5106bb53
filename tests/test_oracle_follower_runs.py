"""The follower's earlier term runs on the oracle (oracle/follower_runs_oracle.c, DESIGN 3.22): the batch form -- the
device's rule over the arena view, the table and a row of at most two runs below the table's run -- against the
literal form, which steps every frame over each group's whole term array as the reference does; without an anchored
row against the passes' own batch oracles; and the setter's row check."""
import numpy as np
import pytest

from helpers import B, O
from oracle import app_entries_oracle as AE
from oracle import app_follow_oracle as AL
from oracle import follower_runs_oracle as FR
import app_follow as A
import follower_runs as F

WIDE_LO, WIDE_HI = 0x20000000, 0x40000000  # RAFTGPU_META_WIDE_LO / _HI

assert FR.ROW_DTYPE == B.FOLLOWER_RUNS_DTYPE and B.FOLLOWER_RUNS_DTYPE.itemsize == 56

# test_raft.rs:5574 (test_fast_log_rejection): (leader log terms, follower log terms, the follower's log_term and
# reject_hint, next_append_term, next_append_index)
FAST_LOG_REJECTION = [
    ([1, 2, 2, 4, 4, 4, 4], [1, 2, 2, 3, 3, 3, 3, 3, 3, 3, 3], 3, 7, 2, 3),
    ([1, 2, 2, 3, 4, 4, 4, 5], [1, 2, 2, 3, 3, 3, 3, 3, 3, 3, 3], 3, 8, 3, 4),
    ([1, 1, 1, 1], [1, 2, 2, 4], 1, 1, 1, 1),
    ([1, 1, 1, 1, 1, 1], [1, 2, 2, 4], 1, 1, 1, 1),
    ([1, 1, 1, 1], [1, 2, 2, 4, 4, 4], 1, 1, 1, 1),
    ([1, 1, 1, 4, 5], [1, 1, 1, 4], 4, 4, 4, 4),
    ([2, 5, 5, 5, 5, 5, 5, 5, 5], [2, 4, 4, 4, 4, 4], 4, 6, 2, 1),
    ([2, 2, 2, 2, 2], [2, 4, 4, 4, 4, 4, 4, 4], 2, 1, 2, 1),
]


def _one(follower, term):
    """One follower (group 0) with the literal log follower: (literal groups, literal terms, columns)."""
    f = F.Followers.__new__(F.Followers)
    f.n, f.log_cap = 1, 64
    f.groups = np.zeros(1, AL.GROUP_DTYPE)
    f.terms = np.zeros((1, 64), np.uint64)
    f.terms[0, 1:len(follower) + 1] = follower
    f.groups["last_index"], f.groups["term"], f.groups["id"], f.groups["flags"] = len(follower), term, 2, AL.FOLLOWER
    return f


@pytest.mark.parametrize("n_runs, rejected, probed", [(0, [0, 1, 5, 6], [1, 5]), (1, [0, 1, 5, 6, 7], [0, 1, 5, 6, 7]),
                                                      (2, list(range(8)), list(range(8)))])
def test_fast_log_rejection_follower(n_runs, rejected, probed):
    """Every case of test_fast_log_rejection at the follower.  The leader (term max + 1 of both logs) probes at its
    last index with its become_leader entry behind it; that entry's term is max + 1 here, not the reference's 1, which
    would make the leader's log non-monotone.  The literal form answers with the reference's (reject_hint, log_term);
    the batch form, with n_runs runs stated below the follower's table run, answers the same where it decides.  Then
    the leader's next probe (next_append_index, next_append_term, and the leader's entries behind it) goes through the
    entries pass: where it is decided the follower's log is the leader's, and the table and the row state its top."""
    got_rej, got_probe = [], []
    for k, (leader, follower, rh_term, rh_index, next_term, next_index) in enumerate(FAST_LOG_REJECTION):
        term = max(leader + follower) + 1
        lead = [0] + leader + [term]  # the leader's log, the become_leader entry last
        f = _one(follower, term)
        table, rows = f.state(n_runs)
        last_l = len(leader)
        body = A.message(3, term=term, log_term=lead[last_l], index=last_l, frm=1, entries=[(term, last_l + 1)])
        blob, off = A.batch([A.frame(0, 1, body)])
        groups, terms = f.groups.copy(), f.terms.copy()
        outcome, lb, lo, _ = AL.literal(groups, terms, blob, off)
        assert outcome[0] == AL.ANSWERED
        want = AL.encode_response(1, 2, term, rh_term, last_l, 0, True, rh_index)
        assert bytes(lb[4:]) == want, k
        c = f.columns()
        st, _, _, rb, ro, _ = FR.batch(c, None, table, rows, blob, off, entries=True)
        if st[0] >> 4 == B.WIRE_OK:
            assert bytes(rb[4:]) == want
            got_rej.append(k)
        else:
            assert st[0] >> 4 == B.WIRE_NEEDS_LOG
        # the next probe, from the follower's unchanged log
        ents = [(lead[i], i) for i in range(next_index + 1, last_l + 2)]
        body = A.message(3, term=term, log_term=next_term, index=next_index, frm=1, entries=ents)
        blob, off = A.batch([A.frame(0, 1, body)])
        groups, terms = f.groups.copy(), f.terms.copy()
        outcome, lb, _, _ = AL.literal(groups, terms, blob, off)
        assert outcome[0] == AL.ANSWERED and list(terms[0, :last_l + 2]) == lead
        c = f.columns()
        st, _, app, rb, _, _ = FR.batch(c, None, table, rows, blob, off, entries=True)
        if st[0] >> 4 == B.WIRE_OK:
            assert bytes(rb) == bytes(lb)
            assert int(c.last_index[0]) == last_l + 1
            assert FR.stated_ok(terms[0], table[0], rows[0], last_l + 1)
            segs = FR.segments(terms[0, :last_l + 2])
            assert (int(table["run_start"][0]), int(table["run_term"][0])) == segs[0]
            stated = [(int(rows["run_start"][0, j]), int(rows["run_term"][0, j])) for j in range(2) if rows["run_start"][0, j]]
            assert stated == segs[1:1 + len(stated)]
            got_probe.append(k)
        else:
            assert st[0] >> 4 == B.WIRE_NEEDS_LOG
    assert (got_rej, got_probe) == (rejected, probed)


def _check_against_literal(f, table, rows, frames, entries):
    """One batch of at most one frame per group through the batch form and the literal form: every frame the batch
    form decides is answered byte for byte as the literal form answers it, and the groups it changed state segments
    that hold at every index of the literal log.  Returns the statuses."""
    blob, off = A.batch(frames)
    groups, terms = f.groups.copy(), f.terms.copy()
    outcome, lb, lo, _ = AL.literal(groups, terms, blob, off)
    c = f.columns()
    st, frm, app, rb, ro, _ = FR.batch(c, None, table, rows, blob, off, entries=entries)
    mine, lit = F.responses_by_frame(st, rb, ro), F.literal_by_frame(outcome, lb, lo)
    for i, s in enumerate(st.tolist()):
        g = int.from_bytes(frames[i][:4], "little") >> 4
        if s >> 4 == B.WIRE_OK:
            assert mine[i] == lit[i], i
            assert int(c.last_index[g]) == int(groups["last_index"][g]) and int(c.committed[g]) == int(groups["committed"][g])
            assert F.FR.stated_ok(terms[g], table[g], rows[g] if rows is not None else None, int(groups["last_index"][g]))
            if s & AE.APPENDED:
                assert (int(app["run_start"][i]), int(app["run_term"][i])) == (int(table["run_start"][g]),
                                                                               int(table["run_term"][g]))
        elif s >> 4 == AL.WIRE_COMMIT_RANGE:
            assert outcome[i] == AL.FATAL
        else:
            assert s >> 4 == B.WIRE_NEEDS_LOG, (i, s)
    return st


@pytest.mark.parametrize("entries", [False, True])
def test_batch_form_agrees_with_the_literal_form_on_random_followers(entries):
    """Followers of 1-6 term runs, some compacted (the runs stated at or above first_index - 1), some rows anchored
    elsewhere; entry-less probes that match in every segment, rejections at random log terms and (the entries pass)
    appends that truncate into the table's run, run 1 and run 2 with 1-3 new terms.  At 0, 1 and 2 stated runs every
    decided frame agrees with the literal form, the stated segments hold, and more runs decide more."""
    rng = np.random.default_rng(0xF011 + entries)
    decided = {}
    for n_runs in (0, 1, 2):
        total = 0
        for trial in range(6):
            f = F.Followers(rng, 300)
            fi = np.where(rng.random(f.n) < 0.3, rng.integers(1, 8, f.n), 1)
            table, rows = f.state(n_runs, fi, rng, stale=0.1)
            cut = set(F.truncate(rng, f, table, 0.05).tolist())  # table runs emptied, rows still anchored to them
            kinds = ["match", "reject", "append"] if entries else ["match", "reject"]
            frames = [A.frame(g, 1, F.probe(rng, f, g, kinds[int(rng.integers(0, len(kinds)))])) for g in range(f.n)]
            st = _check_against_literal(f, table, rows, frames, entries)
            for g in cut:  # an empty table run states nothing: every frame that reads a term at or below last_index
                idx = int(O.wire_decode_message(frames[g][4:])["index"])
                if int(f.groups["committed"][g]) <= idx <= f.last(g):
                    assert st[g] >> 4 == B.WIRE_NEEDS_LOG, g
            total += int((st >> 4 == B.WIRE_OK).sum())
        decided[n_runs] = total
    assert decided[0] < decided[1] < decided[2]


def test_waves_and_wide_pairs_keep_the_segments_true():
    """Several frames per group decided in 4 waves, on wide pairs too: after every call the table and the rows state
    only segments the literal log holds, and the batch's state is the literal form's for the groups it answered."""
    rng = np.random.default_rng(0x4A7E)
    f = F.Followers(rng, 200)
    table, rows = f.state(2)
    c = f.columns()
    wide = np.arange(0, 40, 2)
    c.meta[wide] |= WIDE_LO
    c.meta[wide + 1] |= WIDE_HI
    for k in ("committed", "last_index", "term"):  # a pair's high half: a copy, its own log unused
        getattr(c, k)[wide + 1] = getattr(c, k)[wide]
    frames = []
    for _ in range(3):
        for g in range(f.n):
            if g in set((wide + 1).tolist()):
                continue
            frames.append(A.frame(g, 1, F.probe(rng, f, g, "append" if rng.random() < 0.6 else "match")))
    order = rng.permutation(len(frames))
    frames = [frames[i] for i in order]
    blob, off = A.batch(frames)
    st, frm, app, rb, ro, tot = FR.waves(c, None, table, rows, blob, off, True, 4)
    assert (st >> 4 == B.WIRE_OK).sum() > len(frames) // 3
    # each group's literal log after the frames the waves applied, in their order
    groups, terms = f.groups.copy(), f.terms.copy()
    ok = [i for i in range(len(frames)) if st[i] >> 4 == B.WIRE_OK]
    b2, o2 = A.batch([frames[i] for i in ok])
    outcome, lb, lo, _ = AL.literal(groups, terms, b2, o2)
    assert (outcome == AL.ANSWERED).all()
    assert bytes(rb) == bytes(lb)
    for g in range(f.n):
        if g in set((wide + 1).tolist()):
            continue
        last = int(max(c.last_index[g], c.last_index[g + 1])) if g in set(wide.tolist()) else int(c.last_index[g])
        if any(st[i] >> 4 in (B.WIRE_NEEDS_LOG, AL.WIRE_COMMIT_RANGE) and int.from_bytes(frames[i][:4], "little") >> 4 == g
               for i in range(len(frames))):
            continue  # the host resolves it first
        assert last == int(groups["last_index"][g])
        assert FR.stated_ok(terms[g], table[g], rows[g], last)


def test_without_an_anchored_row_the_passes_oracles_decide():
    """With follower runs off, or on but with no row anchored, the batch form's statuses, from, appended records,
    responses, table and columns are those of the entry-less and the entries passes' batch oracles."""
    rng = np.random.default_rng(0x0A0A)
    for entries in (False, True):
        f = F.Followers(rng, 400)
        table, _ = f.state(0)
        kinds = ["match", "reject", "append"]
        frames = [A.frame(g, 1, F.probe(rng, f, g, kinds[int(rng.integers(0, 3))])) for g in range(f.n) for _ in range(2)]
        blob, off = A.batch(frames)
        for rows in (None, FR.rows_for(f.n)):
            t1, t2 = table.copy(), table.copy()
            c1, c2 = f.columns(), f.columns()
            got = FR.batch(c1, None, t1, rows, blob, off, entries)
            if entries:
                want = AE.batch(c2, None, t2, blob, off)
            else:
                s, fr, rb, ro, tot = AL.batch(c2, None, t2, blob, off)
                want = (s, fr, np.zeros(len(s), AE.APPENDED_DTYPE), rb, ro, tot)
            for w, g in zip(want, got):
                assert np.array_equal(w, g)
            assert np.array_equal(t1, t2)
            for k in ("committed", "last_index"):
                assert np.array_equal(getattr(c1, k), getattr(c2, k))


def test_row_check_refusals():
    """The setter's refusals, row by row: the leader rows' check with the anchor in place of (term, term_start)."""
    ok = FR.row(0, 20, 9, [(10, 5), (4, 2)])
    assert FR.row_status(ok) == 0
    assert FR.row_status(FR.row(0, 20, 9)) == 0
    assert FR.row_status(FR.row(0, 20, 9, [(1, 8)])) == 0
    assert FR.row_status(ok, allocated=False) == B.ERR_RANGE
    assert FR.row_status(ok, wide_hi=True) == B.ERR_RANGE
    bad = [FR.row(0, 20, 0), FR.row(0, 0, 9), FR.row(0, A.NO_TERM_START, 9),
           FR.row(0, 20, 9, [(0, 0), (4, 2)]),                        # run 2 without run 1
           FR.row(0, 20, 9, [(20, 5)]), FR.row(0, 20, 9, [(25, 5)]),  # run 1 not below anchor_start
           FR.row(0, 20, 9, [(10, 5), (10, 2)]), FR.row(0, 20, 9, [(10, 5), (12, 2)]),
           FR.row(0, 20, 9, [(10, 0)]), FR.row(0, 20, 9, [(10, 9)]), FR.row(0, 20, 9, [(10, 12)]),
           FR.row(0, 20, 9, [(10, 5), (4, 5)]), FR.row(0, 20, 9, [(10, 5), (4, 0)]), FR.row(0, 20, 9, [(10, 5), (4, 7)])]
    for r in bad:
        assert FR.row_status(r) == B.ERR_INVALID, r


@pytest.mark.parametrize("follower_runs", [True, False], ids=["follower_runs", "no_follower_runs"])
def test_election_dialogue_on_the_oracles(follower_runs):
    """The election dialogue (follower_runs.Dialogue) on 2K groups x 5 peers, the oracles at both ends: every follower
    ends with its leader's log.  With two runs stated at both ends no frame goes to the host; without the follower's
    runs the follower's end hands frames back."""
    import pass_forms as PF
    d = F.Dialogue(np.random.default_rng(0xD1A1), 2000, follower_runs)
    d.run(PF)
    if follower_runs:
        assert (d.host_follower, d.host_leader) == (0, 0)
    else:
        assert d.host_follower > 0
