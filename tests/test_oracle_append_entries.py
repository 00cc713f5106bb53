"""The batch oracle of raftgpu_follower_append_entries (oracle/app_entries_oracle.c): its entry decode against
python-protobuf's golden vectors, the reference's maybe_append and follower tests restated on it, and the batch form
against the literal form (oracle/app_follow_oracle.c, which appends entries literally) on random logs."""
import json
import os

import numpy as np
import pytest

from helpers import O
from oracle import app_entries_oracle as AE
from oracle import app_follow_oracle as AL
import app_entries as E
import app_follow as A

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "wire", "append_entries.json")
NEEDS_LOG, OK = O.WIRE_NEEDS_LOG, O.WIRE_OK


def test_golden_decode_verdict_entries_and_spans():
    vectors = json.load(open(GOLDEN))["vectors"]
    assert len(vectors) >= 90
    for v in vectors:
        got = AE.decode(bytes.fromhex(v["hex"]))
        assert (got is not None) == v["parses"], v["name"]
        if got is None:
            continue
        ents = got[1][got[1]["ld"] == 1]
        assert [[int(e["term"]), int(e["index"]), int(e["off"]), int(e["end"])] for e in ents] == v["entries"], v["name"]


def _one(last_terms, committed, run, term, frame_body, n_groups=1):
    """One follower (group 0) whose log has terms last_terms[1:] (index 0 the dummy), its run table and one frame ->
    (status, appended record, columns, table)."""
    last = len(last_terms) - 1
    c = O.new_columns(8, n_groups)
    c.term_start[:] = A.NO_TERM_START
    c.term[0], c.last_index[0], c.committed[0] = term, last, committed
    t = np.zeros(n_groups, AL.LOG_DTYPE)
    t["id"], t["flags"], t["run_start"], t["run_term"] = 1, AL.SELECT, run[0], run[1]
    blob, off = A.batch([A.frame(0, 0, frame_body)])
    st, _, app, rb, ro, tot = AE.batch(c, None, t, blob, off)
    return int(st[0]), app[0], c, t, rb


# raft_log.rs:681 test_log_maybe_append: log [1:1, 2:2, 3:3], committed 1; (log_term, index, commit, [(index, term)],
# the result: None = no match, else (last_new, committed after)).  On the batch form a match needs term(index) inside
# the run [3, 3] or above last_index; the reference's fatal case (a conflict at committed) comes with m.index below
# committed and is answered stale by handle_append_entries before maybe_append.
MAYBE_APPEND = [
    (2, 3, 3, [(4, 4)], "needs_log"),  # find_conflict_by_term walks below the run
    (3, 4, 3, [(5, 4)], None),
    (3, 3, 3, [], (3, 3)),
    (3, 3, 4, [], (3, 3)),
    (3, 3, 2, [], (3, 2)),
    (3, 3, 0, [], (3, 1)),
    (0, 0, 3, [], "stale"),
    (3, 3, 3, [(4, 4)], (4, 3)),
    (3, 3, 4, [(4, 4)], (4, 4)),
    (3, 3, 5, [(4, 4)], (4, 4)),
    (3, 3, 5, [(4, 4), (5, 4)], (5, 5)),
    (2, 2, 3, [(3, 4)], "needs_log"),
    (1, 1, 3, [(2, 4)], "needs_log"),
    (0, 0, 3, [(1, 4)], "stale"),
    (1, 1, 3, [(2, 4), (3, 4)], "needs_log"),
]


@pytest.mark.parametrize("case", range(len(MAYBE_APPEND)))
def test_log_maybe_append(case):
    log_term, index, commit, ents, want = MAYBE_APPEND[case]
    body = E.message(5, log_term, index, commit, 2, [E.record(E.entry(t, i)) for i, t in ents])
    st, app, c, t, rb = _one([0, 1, 2, 3], 1, (3, 3), 5, body)
    if want == "needs_log":
        assert st >> 4 == NEEDS_LOG
    elif want == "stale":
        assert st == (OK << 4 | AL.RES_OK | AL.STALE)
    elif want is None:
        assert st == (OK << 4 | AL.RES_OK | AL.REJECT)
        assert int(c.last_index[0]) == 3
    else:
        last_new, committed = want
        appended = any(i > 3 for i, _ in ents)
        assert st == (OK << 4 | AL.RES_OK | (AE.APPENDED if appended else 0)), st
        assert int(c.committed[0]) == committed
        assert int(c.last_index[0]) == (last_new if appended else 3)
        assert int(app["last_index"]) == (last_new if appended else 0)
        if appended:
            assert (int(t["run_start"][0]), int(t["run_term"][0])) == (4, 4)
            assert int(app["first_index"]) == 4


def _literal_log(log_terms, body):
    """The literal form's log after one frame to a follower at term 5 with log_terms (committed 0) -> terms[1..last]."""
    groups = np.zeros(1, AL.GROUP_DTYPE)
    groups["id"], groups["term"], groups["last_index"], groups["flags"] = 1, 5, len(log_terms) - 1, AL.FOLLOWER
    terms = np.zeros((1, 32), np.uint64)
    terms[0, :len(log_terms)] = log_terms
    blob, off = A.batch([A.frame(0, 0, body)])
    AL.literal(groups, terms, blob, off)
    return terms[0, :int(groups["last_index"][0]) + 1]


# raft_log.rs:767 test_find_conflict, restated where the run decides: m.index in the run, entries from m.index + 1 on.
# (log, m.index, [(index, term)], conflict): no conflict (every entry matched), the first entry past the log, or a
# conflict at or below last_index inside the run (a truncation).  None: entries that do not follow m.index.
@pytest.mark.parametrize("log,index,ents,conflict", [
    ([0, 1, 2, 3], 3, [], 0),
    ([0, 1, 2, 3], 3, [(3, 3)], None),
    ([0, 1, 2, 3], 3, [(4, 4), (5, 4)], 4),
    ([0, 1, 2, 3], 3, [(4, 5)], 4),
    ([0, 1, 2, 3], 3, [(4, 3), (5, 3)], 4),
    ([0, 1, 3, 3, 3, 3], 2, [(3, 3), (4, 3)], 0),
    ([0, 1, 3, 3, 3, 3], 2, [(3, 3), (4, 4), (5, 4)], 4),
    ([0, 1, 3, 3, 3, 3], 3, [(4, 4)], 4),
])
def test_find_conflict(log, index, ents, conflict):
    last = len(log) - 1
    body = E.message(5, 3, index, 0, 2, [E.record(E.entry(t, i)) for i, t in ents])
    st, app, c, t, _ = _one(log, 0, A.run_of(np.array(log, np.uint64), last), 5, body)
    if conflict is None:          # (3, 3) does not follow index 3: the indexes are the host's
        assert st >> 4 == NEEDS_LOG
        return
    assert st >> 4 == OK
    assert int(app["first_index"]) == conflict
    assert int(c.last_index[0]) == (index + len(ents) if conflict else last)
    lit = _literal_log(log, body)
    assert len(lit) - 1 == int(c.last_index[0])


# raft_log.rs:1279 test_append on the batch form, with the log's last run kept in the table: entries of the run's term
# past the log extend the run; a new term starts a new one at its first entry; a conflict inside the run truncates the
# log there and the run starts at the trailing block of the last term.  The literal form's log agrees.
@pytest.mark.parametrize("log,run,index,ents,want_last,want_run", [
    ([0, 1, 2], (2, 2), 2, [(3, 2)], 3, (2, 2)),
    ([0, 1, 2], (2, 2), 2, [(3, 3)], 3, (3, 3)),
    ([0, 1, 2], (2, 2), 2, [(3, 2), (4, 3), (5, 3)], 5, (4, 3)),
    ([0, 1, 2, 2, 2, 2], (2, 2), 2, [(3, 3)], 3, (3, 3)),                    # truncation at 3 inside the run
    ([0, 1, 2, 2, 2, 2], (2, 2), 3, [(4, 2), (5, 3), (6, 3)], 6, (5, 3)),    # matches 4, truncates at 5
    ([0, 1, 2, 2, 2, 2], (3, 2), 3, [(4, 2), (5, 2), (6, 2)], 6, (3, 2)),    # a shortened run, extended past the log
])
def test_append(log, run, index, ents, want_last, want_run):
    body = E.message(5, 2, index, 0, 2, [E.record(E.entry(t, i)) for i, t in ents])
    st, app, c, t, _ = _one(log, 0, run, 5, body)
    assert st & AE.APPENDED
    assert int(c.last_index[0]) == want_last
    assert (int(t["run_start"][0]), int(t["run_term"][0])) == want_run == (int(app["run_start"]), int(app["run_term"]))
    lit = _literal_log(log, body)
    assert len(lit) - 1 == want_last
    true_start, true_term = A.run_of(lit, want_last)
    assert want_run[1] == true_term and want_run[0] >= true_start   # a suffix of the true last run


def test_follower_append_entries():
    """test_raft_paper.rs:709: a follower at term 2 with the log [1:1, 2:2].  The case the run decides appends as the
    reference does; the three that match below the run come back NEEDS_LOG, and the literal form (the reference's
    steps) ends with the reference's logs."""
    cases = [(2, 2, [(3, 3)], [1, 2, 3]), (1, 1, [(2, 3), (3, 4)], [1, 3, 4]), (0, 0, [(1, 1)], [1, 2]),
             (0, 0, [(1, 3)], [3])]
    for k, (index, log_term, ents, wlog) in enumerate(cases):
        body = E.message(2, log_term, index, 0, 2, [E.record(E.entry(t, i)) for i, t in ents])
        st, app, c, t, _ = _one([0, 1, 2], 0, (2, 2), 2, body)
        assert (st >> 4 == 0) == (k == 0), (k, st)
        groups = np.zeros(1, AL.GROUP_DTYPE)
        groups["id"], groups["term"], groups["last_index"], groups["flags"] = 1, 2, 2, AL.FOLLOWER
        terms = np.zeros((1, 16), np.uint64)
        terms[0, 1:3] = [1, 2]
        blob, off = A.batch([A.frame(0, 0, body)])
        AL.literal(groups, terms, blob, off)
        assert terms[0, 1:int(groups["last_index"][0]) + 1].tolist() == wlog, k
        if k == 0:
            assert int(c.last_index[0]) == 3 and int(app["first_index"]) == 3


def _decode_spans(blob, off, st, app):
    """python-protobuf's reading of every appended span -> {frame: [(term, index)]}."""
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
    from gen_wire_golden import build_classes
    Message = build_classes()
    out = {}
    for i in np.flatnonzero(st & AE.APPENDED).tolist():
        a, n = int(app["span_off"][i]), int(app["span_len"][i])
        m = Message()
        m.ParseFromString(bytes(blob[a:a + n]))
        out[i] = [(e.term, e.index) for e in m.entries]
    return out


@pytest.mark.parametrize("shorten", [0.0, 0.4])
def test_batch_against_literal_on_random_logs(shorten):
    """Random literal logs with full or shortened runs, one random frame each (overlaps, truncations inside the run,
    all-matching frames, stale and rejected frames, gaps, hostile entries): every frame the batch form decides leaves
    the literal form's state (last_index, committed, response), its appended span decodes to the entries the literal
    log took, and the run it leaves is a suffix of the literal log's last run."""
    rng = np.random.default_rng(0xAE50 + int(shorten * 10))
    n = 3000
    w = A.World(rng, n, log_cap=160, max_last=60)
    runs = w.runs(rng, shorten)
    c, table = w.columns(), w.table(runs)
    c.term = w.groups["term"].copy()
    frames = []
    for g in range(n):
        s, rt = runs[g]
        body = E.random_frame(rng, int(w.groups["last_index"][g]), s, rt, int(w.groups["term"][g]),
                              int(w.groups["committed"][g]), hostile=0.05)
        frames.append(A.frame(g, 0, body))
    blob, off = A.batch(frames)
    st, frm, app, rb, ro, tot = AE.batch(c, None, table, blob, off)
    lit = w.copy()
    outcome, lrb, lro, _ = AL.literal(lit.groups, lit.terms, blob, off)
    decided = (st >> 4) == OK
    assert decided.sum() > n // 2 and np.count_nonzero(st & AE.APPENDED) > n // 5
    spans = _decode_spans(blob, off, st, app)
    bresp = A.split_responses(rb, ro)
    lresp = A.split_responses(lrb, lro)
    # the literal form answers every frame; map its responses to frames in order
    lmap, k = {}, 0
    for i in range(n):
        if outcome[i] == AL.ANSWERED:
            lmap[i] = lresp[k]
            k += 1
    bk = 0
    for i in range(n):
        if not decided[i]:
            continue
        assert outcome[i] == AL.ANSWERED, i
        assert bresp[bk] == lmap[i], i
        bk += 1
        g = i
        last = int(lit.groups["last_index"][g])
        assert int(c.last_index[g]) == last and int(c.committed[g]) == int(lit.groups["committed"][g]), i
        if st[i] & AE.APPENDED:
            a = app[i]
            assert int(a["last_index"]) == last
            took = [(int(lit.terms[g, j]), j) for j in range(int(a["first_index"]), last + 1)]
            assert spans[i] == took, i
            assert int(w.terms[g, int(a["first_index"])]) != int(lit.terms[g, int(a["first_index"])]) or \
                int(a["first_index"]) > int(w.groups["last_index"][g])
        rs, rt = int(table["run_start"][g]), int(table["run_term"][g])
        true_s, true_t = A.run_of(lit.terms[g], last)
        assert rs > last or (rt == true_t and rs >= true_s), (i, rs, rt, true_s, true_t)
