"""The follower MsgAppend oracle (oracle/app_follow_oracle.c): its encoder against python-protobuf's bytes
(tests/golden/wire/append_responses.json, scripts/gen_wire_append_resp_golden.py), the entries flag on golden MsgAppend
bytes, the reference's follower append cases on the literal form, the batch form against the literal form on random
logs with full and shortened runs, the resubmission loop, and the commit loop through three oracles."""
import json
import os

import numpy as np

from oracle import app_follow_oracle as AL
from oracle import app_frames_oracle as AF
from helpers import B, O
import app_follow as A

HERE = os.path.dirname(os.path.abspath(__file__))
U64 = A.U64
EDGES = {0, 1, 127, 128, 1 << 32, 1 << 63, U64}


def _golden():
    with open(os.path.join(HERE, "golden", "wire", "append_responses.json")) as f:
        return json.load(f)


def test_golden_responses_encode_byte_for_byte_and_decode_back():
    vs = _golden()["responses"]
    names = ("to", "from", "term", "log_term", "index", "commit", "reject", "reject_hint")
    for v in vs:
        got = AL.encode_response(*[v[k] for k in names])
        assert got.hex() == v["hex"], v
        assert len(got) + 4 <= AL.FRAME_MAX
        m = O.wire_decode_message(got)
        assert m["msg_type"] == 4 and [m["from" if k == "from" else k] for k in names] == [v[k] for k in names], v
    for name in names:
        assert (EDGES if name != "reject" else {0, 1}) <= {v[name] for v in vs}, name
    assert any(v["reject"] and v["reject_hint"] == 0 and v["log_term"] == 0 for v in vs)


def test_golden_appends_entries_flag():
    """0, 1 and 3 entries, an empty Entry among them: the field-7 count and each Entry's term and index."""
    seen = set()
    for v in _golden()["appends"]:
        n7, ents = AL.fields7(bytes.fromhex(v["hex"]))
        assert n7 == len(v["entries"]) and [list(e) for e in ents] == v["entries"], v
        seen.add(n7)
        assert A.message(3, v["term"], v["log_term"], v["index"], v["commit"], to=0,
                         entries=[tuple(e) for e in v["entries"]]).hex() == v["hex"]
    assert seen == {0, 1, 3}


def _literal_one(log, term, committed, msg, lower_reply=False):
    """One follower (id 1) with log terms [dummy 0] + log, stepped with msg from id 2 -> (outcome, response fields, group)."""
    g = np.zeros(1, AL.GROUP_DTYPE)
    g["id"], g["term"], g["committed"], g["last_index"] = 1, term, committed, len(log)
    g["flags"] = AL.FOLLOWER | (AL.LOWER_REPLY if lower_reply else 0)
    t = np.zeros((1, 64), np.uint64)
    t[0, 1:len(log) + 1] = log
    out, rb, ro, tot = AL.literal(g, t, *A.batch([A.frame(0, 5, msg)]))
    resp = [O.wire_decode_message(b) for h, b in A.split_responses(rb, ro)]
    assert all(h == 5 for h, _ in A.split_responses(rb, ro))
    return int(out[0]), resp, g[0], t[0]


def test_follower_check_msg_append():
    """test_raft_paper.rs:645 (test_follower_check_msg_append): log [(1, 1), (2, 2)], committed 1, term 2."""
    cases = [(0, 0, 1, 1, False, 0, 0), (1, 1, 1, 1, False, 0, 0), (2, 2, 2, 1, False, 0, 0), (1, 2, 2, 1, True, 1, 1),
             (3, 3, 3, 1, True, 2, 2)]
    for log_term, index, windex, wcommit, wreject, whint, wlt in cases:
        out, resp, _, _ = _literal_one([1, 2], 2, 1, A.message(3, term=2, log_term=log_term, index=index, frm=2))
        assert out == AL.ANSWERED and len(resp) == 1
        m = resp[0]
        assert (m["msg_type"], m["to"], m["from"], m["term"], m["index"], m["commit"]) == (4, 2, 1, 2, windex, wcommit)
        assert (bool(m["reject"]), m["reject_hint"], m["log_term"]) == (wreject, whint if wreject else 0,
                                                                       wlt if wreject else 0)
        # the batch form with the run the log implies decides it the same way
        c = O.new_columns(8, 1)
        c.term_start[:] = A.NO_TERM_START
        c.term[0], c.last_index[0], c.committed[0] = 2, 2, 1
        tab = np.zeros(1, AL.LOG_DTYPE)
        tab["id"], tab["run_start"], tab["run_term"], tab["flags"] = 1, 2, 2, AL.SELECT
        st, frm, rb, ro, _ = AL.batch(c, None, tab, *A.batch([A.frame(0, 5, A.message(3, term=2, log_term=log_term,
                                                                                    index=index, frm=2))]))
        if st[0] >> 4 == B.WIRE_OK:
            assert [O.wire_decode_message(b) for _, b in A.split_responses(rb, ro)] == resp and frm[0] == 2
        else:  # the decision reads a term below the run [2, 2]
            assert st[0] >> 4 == B.WIRE_NEEDS_LOG and A.reads_outside([0, 1, 2], 2, 1, 2, index, log_term)


def test_handle_msg_append():
    """test_raft.rs:1281 (test_handle_msg_append): log [(1, 1), (2, 2)], committed 0, term 2 -> last_index, committed,
    reject.  The reference calls handle_append_entries directly; here every message is at the follower's term."""
    cases = [((3, 2, 3, None), 2, 0, True), ((3, 3, 3, None), 2, 0, True), ((1, 1, 1, None), 2, 1, False),
             ((0, 0, 1, [(2, 1)]), 1, 1, False), ((2, 2, 3, [(2, 3), (2, 4)]), 4, 3, False),
             ((2, 2, 4, [(2, 3)]), 3, 3, False), ((1, 1, 4, [(2, 2)]), 2, 2, False), ((1, 1, 3, None), 2, 1, False),
             ((1, 1, 3, [(2, 2)]), 2, 2, False), ((2, 2, 3, None), 2, 2, False), ((2, 2, 4, None), 2, 2, False)]
    for (log_term, index, commit, ents), wlast, wcommit, wreject in cases:
        msg = A.message(3, term=2, log_term=log_term, index=index, commit=commit, frm=2, entries=ents)
        out, resp, g, _ = _literal_one([1, 2], 2, 0, msg)
        assert out == AL.ANSWERED and len(resp) == 1
        assert (int(g["last_index"]), int(g["committed"]), bool(resp[0]["reject"])) == (wlast, wcommit, wreject)


# test_raft.rs:5574 (test_fast_log_rejection): (leader log terms, follower log terms, reject_hint's term, reject_hint)
FAST_LOG_REJECTION = [
    ([1, 2, 2, 4, 4, 4, 4], [1, 2, 2, 3, 3, 3, 3, 3, 3, 3, 3], 3, 7),
    ([1, 2, 2, 3, 4, 4, 4, 5], [1, 2, 2, 3, 3, 3, 3, 3, 3, 3, 3], 3, 8),
    ([1, 1, 1, 1], [1, 2, 2, 4], 1, 1),
    ([1, 1, 1, 1, 1, 1], [1, 2, 2, 4], 1, 1),
    ([1, 1, 1, 1], [1, 2, 2, 4, 4, 4], 1, 1),
    ([1, 1, 1, 4, 5], [1, 1, 1, 4], 4, 4),
    ([2, 5, 5, 5, 5, 5, 5, 5, 5], [2, 4, 4, 4, 4, 4], 4, 6),
    ([2, 2, 2, 2, 2], [2, 4, 4, 4, 4, 4, 4, 4], 2, 1),
]


def test_fast_log_rejection_follower_hints():
    """The follower side of every case of test_raft.rs:5574 (test_fast_log_rejection): the new leader's probe (index =
    its last index, log_term = its last term, its new entry) gets the reference's (reject_hint, log_term) on the literal
    form, whose find_conflict_by_term walks the follower's whole log.  On the batch form, with the run the follower's
    log implies, the probe is NEEDS_LOG (it carries an entry); without the entry it is decided with the same hint where
    the walk stays in the run (the first two cases, where it starts and stops there, and the sixth and seventh, where
    it starts above last_index), and is NEEDS_LOG where it walks below the run (the others)."""
    decided = []
    for leader, follower, wterm, whint in FAST_LOG_REJECTION:
        index, log_term = len(leader), leader[-1]
        msg = A.message(3, term=5, log_term=log_term, index=index, frm=1, entries=[(5, index + 1)])
        _, resp, g, _ = _literal_one(follower, 5, 0, msg)
        assert resp[0]["reject"] and (resp[0]["reject_hint"], resp[0]["log_term"]) == (whint, wterm)
        assert int(g["last_index"]) == len(follower)                  # a rejection appends nothing
        row = np.array([0] + follower, np.uint64)
        run_start, run_term = A.run_of(row, len(follower))
        c = O.new_columns(8, 1)
        c.term_start[:] = A.NO_TERM_START
        c.term[0], c.last_index[0] = 5, len(follower)
        tab = np.zeros(1, AL.LOG_DTYPE)
        tab["id"], tab["run_start"], tab["run_term"], tab["flags"] = 2, run_start, run_term, AL.SELECT
        st, _, _, _, tot = AL.batch(c, None, tab, *A.batch([A.frame(0, 0, msg)]))
        assert st[0] >> 4 == B.WIRE_NEEDS_LOG and int(tot[0]) == 0
        bare = A.message(3, term=5, log_term=log_term, index=index, frm=1)
        st, _, rb, ro, _ = AL.batch(c, None, tab, *A.batch([A.frame(0, 0, bare)]))
        if A.reads_outside(row, len(follower), 0, run_start, index, log_term):
            assert st[0] >> 4 == B.WIRE_NEEDS_LOG
        else:
            m = O.wire_decode_message(A.split_responses(rb, ro)[0][1])
            assert st[0] == (A.LOG_STATUS_OK | AL.REJECT) and (m["reject_hint"], m["log_term"]) == (whint, wterm)
            decided.append(FAST_LOG_REJECTION.index((leader, follower, wterm, whint)))
    assert decided == [0, 1, 5, 6]


def test_lower_and_higher_terms_on_the_literal_form():
    out, resp, _, _ = _literal_one([1, 2], 3, 1, A.message(3, term=2, index=2, frm=2), lower_reply=True)
    assert out == AL.ANSWERED and resp[0]["term"] == 3 and resp[0]["index"] == 0 and not resp[0]["reject"]
    out, resp, _, _ = _literal_one([1, 2], 3, 1, A.message(3, term=2, index=2, frm=2))
    assert out == AL.DROPPED and resp == []
    out, resp, g, _ = _literal_one([1, 2], 2, 1, A.message(3, term=4, log_term=2, index=2, commit=2, frm=2))
    assert out == AL.ANSWERED and int(g["term"]) == 4 and int(g["committed"]) == 2 and resp[0]["term"] == 4


def _decide_vs_literal(seed, shorten):
    rng = np.random.default_rng(seed)
    n = 3000
    w = A.World(rng, n)
    runs = w.runs(rng, shorten)
    gs = rng.permutation(n)
    frames = [A.frame(int(g), int(rng.integers(16)), A.random_append(rng, w, int(g), entries_p=0.1)) for g in gs]
    blob, off = A.batch(frames)
    c = w.columns()
    before = A.state(c, n)
    st, frm, rb, ro, tot = AL.batch(c, None, w.table(runs), blob, off)
    lw = w.copy()
    out, lrb, lro, _ = AL.literal(lw.groups, lw.terms, blob, off)
    lresp = A.split_responses(lrb, lro)
    assert np.all(out != AL.NONE)
    answered = np.cumsum(out == AL.ANSWERED) - 1                       # frame -> its literal response
    bresp = iter(A.split_responses(rb, ro))
    kinds = np.bincount(st >> 4, minlength=16)
    for i, g in enumerate(gs.tolist()):
        s, f = int(st[i]) >> 4, AL.fields7(frames[i][4:])[0]
        m = O.wire_decode_message(frames[i][4:])
        outside = f > 0 or A.reads_outside(w.terms[g], int(w.groups["last_index"][g]), int(w.groups["committed"][g]),
                                          runs[g][0], m["index"], m["log_term"])
        assert (s == B.WIRE_NEEDS_LOG) == outside, (i, s, m, runs[g])
        if s == B.WIRE_OK:
            assert out[i] == AL.ANSWERED and next(bresp) == lresp[answered[i]], i
            assert c.committed[g] == lw.groups["committed"][g] and frm[i] == m["from"]
        else:
            assert c.committed[g] == before["committed"][g] and frm[i] == 0      # a non-OK frame changes nothing
            if s == B.WIRE_COMMIT_RANGE:
                assert out[i] == AL.FATAL
    assert next(bresp, None) is None
    for k in ("last_index", "term", "term_start"):
        assert np.array_equal(A.state(c, n)[k], before[k])
    return kinds


def test_batch_decides_as_the_literal_form_full_runs():
    kinds = _decide_vs_literal(0xAF01, 0.0)
    assert kinds[B.WIRE_OK] > 1200 and kinds[B.WIRE_NEEDS_LOG] > 200 and kinds[B.WIRE_COMMIT_RANGE] > 10, kinds


def test_batch_decides_as_the_literal_form_shortened_runs():
    kinds = _decide_vs_literal(0xAF02, 0.7)
    assert kinds[B.WIRE_OK] > 800 and kinds[B.WIRE_NEEDS_LOG] > 500, kinds


def test_statuses_before_the_decision_change_nothing():
    rng = np.random.default_rng(0xAF03)
    n = 500
    w = A.World(rng, n)
    tab = w.table(w.runs())
    tab["flags"][rng.random(n) < 0.2] = 0
    c = w.columns()
    c.term_start[:n][rng.random(n) < 0.1] = 3
    frames = []
    for g in range(n):
        t = int(w.groups["term"][g])
        frames += [A.frame(g, 1, A.message(3, term=t + int(rng.choice([-1, 1])), index=1, frm=2)),
                   A.frame(g, 1, A.message(int(rng.choice([4, 8, 9])), term=t, frm=2)),
                   A.frame(g, 1, A.message(3, term=0, frm=2)), A.frame(g, 1, bytes([0xff, 0xff])),
                   A.frame(n + 5 + g, 1, A.message(3, term=t))]
    before = A.state(c, n)
    st, frm, rb, ro, tot = AL.batch(c, None, tab, *A.batch(frames))
    assert set((st >> 4).tolist()) <= {B.WIRE_TERM, B.WIRE_SKIP_TYPE, B.WIRE_ROLE, B.WIRE_MALFORMED}
    assert {B.WIRE_TERM, B.WIRE_SKIP_TYPE, B.WIRE_ROLE, B.WIRE_MALFORMED} <= set((st >> 4).tolist())
    assert tot.tolist() == [0, 0] and not frm.any()
    after = A.state(c, n)
    assert all(np.array_equal(before[k], after[k]) for k in before)


def resubmission_loop(w, runs_of, frames, step):
    """Run frames through `step` (the batch form or the device) until none is DUP; the host takes every frame the pass
    leaves (NEEDS_LOG, COMMIT_RANGE) through the literal form, in frame order between rounds.  step(c, table, blob, off)
    -> (status, from, response blob, response offsets, totals) and leaves the arena in c.  Returns (final status per
    frame, responses per group, rounds)."""
    final = np.full(len(frames), 0xFF, np.uint8)
    per_group = {}
    pending = list(range(len(frames)))
    rounds = 0
    while pending:
        rounds += 1
        c = w.columns()
        st, _, rb, ro, _ = step(c, w.table(runs_of(w)), *A.batch([frames[i] for i in pending]))
        w.groups["committed"] = c.committed[: w.n]
        resp = iter(A.split_responses(rb, ro))
        nxt = []
        for k, i in enumerate(pending):
            s = int(st[k]) >> 4
            g = int.from_bytes(frames[i][:4], "little") >> 4
            if s == B.WIRE_DUP:
                nxt.append(i)
                continue
            final[i] = st[k]
            if s == B.WIRE_OK:
                per_group.setdefault(g, []).append(next(resp))
            else:
                out, lrb, lro, _ = AL.literal(w.groups, w.terms, *A.batch([frames[i]]))
                assert out[0] == AL.ANSWERED
                per_group.setdefault(g, []).extend(A.split_responses(lrb, lro))
        pending = nxt
    return final, per_group, rounds


def test_resubmission_loop_equals_the_literal_form():
    rng = np.random.default_rng(0xAF04)
    n = 800
    w = A.World(rng, n)
    frames = []
    for g in range(n):
        frames += [(g, A.frame(g, int(rng.integers(16)), A.random_append(rng, w, g, entries_p=0.15, safe=True)))
                   for _ in range(int(rng.integers(1, 5)))]
    frames = [f for _, f in (frames[i] for i in rng.permutation(len(frames)))]
    want_w = w.copy()
    out, lrb, lro, _ = AL.literal(want_w.groups, want_w.terms, *A.batch(frames))
    assert np.all(out == AL.ANSWERED)
    want = {}
    lresp = A.split_responses(lrb, lro)
    for i, f in enumerate(frames):
        want.setdefault(int.from_bytes(f[:4], "little") >> 4, []).append(lresp[i])
    for shorten in (0.0, 0.5):
        w2 = w.copy()
        srng = np.random.default_rng(7)
        final, got, rounds = resubmission_loop(w2, lambda x: x.runs(srng, shorten), frames,
                                               lambda c, t, b, o: AL.batch(c, None, t, b, o))
        assert rounds >= 4 and got == want
        assert np.array_equal(w2.groups, want_w.groups) and np.array_equal(w2.terms, want_w.terms)
        assert set((final >> 4).tolist()) <= {B.WIRE_OK, B.WIRE_NEEDS_LOG}
        assert np.count_nonzero(final >> 4 == B.WIRE_OK) > len(frames) // 3


def test_commit_loop_through_the_oracles():
    """app_frames_oracle's commit broadcast -> the follower oracle at each of four followers -> the wire oracle (the
    leader's handle_append_response) at the leader.  Every follower is caught up: every frame is OK and every response
    WIRE_OK at the leader, whose peers' matched and peer_committed move to the followers' answers."""
    rng = np.random.default_rng(0xAF05)
    n = 2000
    c = O.new_columns(n, n)
    c.meta[:] = O.make_meta(0b11111, 0, 0, 0)
    c.term[:n] = rng.integers(1, 1 << 40, n)
    c.term_start[:n] = 1
    c.last_index[:n] = rng.integers(1, 1 << 30, n)
    c.committed[:n] = c.last_index[:n] - rng.integers(0, 5, n).astype(np.uint64)
    c.next_idx[:, :n] = c.last_index[:n] + 1
    c.matched[:, :n] = c.last_index[:n]
    c.peer_committed[:, :n] = c.committed[:n] - np.minimum(c.committed[:n], 3)
    c.pflags[:, :n] = B.STATE_REPLICATE
    ids = rng.integers(1, 1 << 63, (9, n), dtype=np.uint64)
    blob, off, rest, tot = AF.bcast_append(c, None, 0, n, ids)
    assert int(tot[0]) == 4 * n and len(rest) == 0
    hdr = np.array([int.from_bytes(bytes(blob[a:a + 4]), "little") for a in off[:-1].tolist()], np.uint32)
    back = []
    for s in range(1, 5):
        sel = np.flatnonzero((hdr & 15) == s)
        frames = [bytes(blob[off[i]:off[i + 1]]) for i in sel]       # follower slot g: the header stays (g << 4 | s)
        fc = O.new_columns(n + 8, n)
        fc.term_start[:] = A.NO_TERM_START
        fc.term[:n], fc.last_index[:n] = c.term[:n], c.last_index[:n]
        fc.committed[:n] = c.peer_committed[s, :n]
        tab = np.zeros(n, AL.LOG_DTYPE)
        tab["id"], tab["flags"] = ids[s], AL.SELECT
        tab["run_start"], tab["run_term"] = c.last_index[:n] - np.minimum(c.last_index[:n], 2), c.term[:n]
        st, frm, rb, ro, rt = AL.batch(fc, None, tab, *A.batch(frames))
        leader_ids = [O.wire_decode_message(f[4:])["from"] for f in frames]
        assert np.all(st == A.LOG_STATUS_OK) and frm.tolist() == leader_ids and int(rt[0]) == n
        assert np.array_equal(fc.committed[:n], c.committed[:n])
        back += [np.array([h], "<u4").tobytes() + b for h, b in A.split_responses(rb, ro)]
    wblob, woff = A.batch(back)
    wst, recs, hint, snap = O.wire_decode_batch(wblob, woff, n, c.term[:n])
    assert np.all(wst == B.WIRE_OK)
    O.arena_apply(c, recs, mode=0)
    assert np.array_equal(c.peer_committed[1:5, :n], np.broadcast_to(c.committed[:n], (4, n)))
    assert np.array_equal(c.matched[1:5, :n], np.broadcast_to(c.last_index[:n], (4, n)))


def test_log_table_mirror_matches_the_header():
    """raftgpu_follower_log's C layout (from the header text) against binding.FOLLOWER_LOG_DTYPE and the oracle's."""
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(HERE), "scripts"))
    import gen_rust_stub as G
    size, offs = G.struct_layouts()["raftgpu_follower_log"]
    assert size == B.FOLLOWER_LOG_DTYPE.itemsize == AL.LOG_DTYPE.itemsize == 32
    assert [(f, o) for f, o, _ in offs] == [(f, B.FOLLOWER_LOG_DTYPE.fields[f][1]) for f in B.FOLLOWER_LOG_DTYPE.names]
    assert B.FOLLOWER_LOG_DTYPE == AL.LOG_DTYPE
    assert (B.FOLLOWER_SELECT, B.FAPP_REJECT, B.FAPP_STALE) == (AL.SELECT, AL.REJECT, AL.STALE)
    assert B.follower_append_bound(3) == 3 * AL.FRAME_MAX
