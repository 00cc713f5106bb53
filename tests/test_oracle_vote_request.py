"""The vote-request oracle (oracle/vote_request_oracle.c) on the CPU: the encoder goldens, the reference's voter tables
restated on the literal form and through the batch form, and the exactness of the batch form's resubmission loop against
the literal form."""
import json
import os

import numpy as np
import pytest

from oracle import oracle as O
from oracle import control_oracle as CO
from oracle import hb_wire_oracle as H
from oracle import vote_request_oracle as VR
from helpers import B
import hb_frames as F
import vote_request_frames as Q

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "wire", "vote_requests.json")
FIELDS = ("to", "from", "term", "log_term", "index", "commit", "commit_term", "priority")


def _golden():
    with open(GOLDEN, encoding="utf-8") as f:
        return json.load(f)["vectors"]


# --------------------------------------------------------------------------- 1. the encoders and the decoder


def test_test_encoder_and_oracle_decoder_match_python_protobuf():
    vs = _golden()
    assert len(vs) > 500
    for v in vs:
        ctx = bytes.fromhex(v["context"])
        got = Q.request(v["msg_type"], v["term"], v["log_term"], v["index"], v["commit"], v["commit_term"], v["priority"],
                        ctx, to=v["to"], frm=v["from"])
        assert got.hex() == v["hex"], v
        m = H.decode_message(got)   # fields 5, 6, 12, 14 and 15 read back
        assert m["msg_type"] == v["msg_type"] and m["context"] == ctx
        assert all(m[k] == v[k] for k in FIELDS), v


def test_synth_encoder_matches_python_protobuf():
    vs = _golden()
    e = np.zeros(len(vs), B.SYNTH_VOTE_REQUEST_DTYPE)
    for i, v in enumerate(vs):
        e[i]["hdr"] = (i % 1000) << 4 | (i % 16)
        e[i]["msg_type"] = v["msg_type"]
        for k in FIELDS:
            e[i][k] = v[k]
        ctx = bytes.fromhex(v["context"])
        e[i]["context"][: len(ctx)] = np.frombuffer(ctx, np.uint8)
        e[i]["context_len"] = len(ctx)
    blob, off = B.synth_encode_vote_requests(e)
    for i, v in enumerate(vs):
        fr = blob[off[i]:off[i + 1]].tobytes()
        assert fr[:4] == np.array([(i % 1000) << 4 | (i % 16)], "<u4").tobytes()
        assert fr[4:].hex() == v["hex"], v


def test_response_encoder_is_the_vote_response_encoding():
    """vro_encode_response writes what tests/vote_frames.py (pinned by vote_responses.json) writes."""
    import vote_frames as V
    rng = np.random.default_rng(5)
    for _ in range(500):
        t, to, fr, term, c, ct = int(rng.choice([6, 18])), *[int(rng.choice([0, 1, rng.integers(1 << 62)])) for _ in range(5)]
        rej = bool(rng.random() < 0.5)
        assert VR.encode_response(t, to, fr, term, c, rej, ct) == V.message(t, term, rej, c, ct, to=to, frm=fr)


# --------------------------------------------------------------------------- 2. one group at a time


def _one(role, term, vote, last_index, last_term, leader=False, lease=False, check_quorum=False, voters=0b1,
         committed=None, commit_term=0, priority=0):
    """One group (slot 0 = self, id 1) in `role` at `term` with the given log -> (columns, votes, role, table)."""
    c = O.new_columns(8, 1)
    c.meta[0] = B.make_meta(voters, 0, 0, 0)
    c.term[0], c.last_index[0] = term, last_index
    c.committed[0] = last_index if committed is None else committed
    c.term_start[0] = last_index if role == Q.LEADER else B.NO_TERM_START
    t = np.zeros(1, VR.VOTER_DTYPE)
    t["id"], t["vote"], t["last_term"], t["commit_term"], t["persisted"], t["priority"] = \
        1, vote, last_term, commit_term, last_index, priority
    t["flags"] = (VR.SELECT if role != Q.LEADER else 0) | (VR.LEADER if leader else 0) | (VR.LEASE if lease else 0) | \
        (VR.CHECK_QUORUM if check_quorum else 0)
    return c, np.zeros((O.SLOTS, c.cap), np.uint8), np.array([role], np.uint8), t


def _responses(blob, off):
    return [H.decode_message(blob[off[k] + 4:off[k + 1]].tobytes()) for k in range(len(off) - 1)]


def _literal(state, frames):
    c, vt, role, t = state
    blob, off = F.batch(frames)
    rb, ro, _ = VR.literal(c, None, vt, role, t, blob, off)
    return _responses(rb, ro)


def _batch(state, frames):
    c, vt, _, t = state
    blob, off = F.batch(frames)
    st, out, rb, ro, _ = VR.batch(c, None, vt, blob, off, t)
    return st, _responses(rb, ro)


# test_raft.rs:1537-1605: (role, index, log_term, vote, want reject) against a log of two entries at term 2
RECV_VOTE = [
    (Q.FOLLOWER, 0, 0, 0, True), (Q.FOLLOWER, 0, 1, 0, True), (Q.FOLLOWER, 0, 2, 0, True), (Q.FOLLOWER, 0, 3, 0, False),
    (Q.FOLLOWER, 1, 0, 0, True), (Q.FOLLOWER, 1, 1, 0, True), (Q.FOLLOWER, 1, 2, 0, True), (Q.FOLLOWER, 1, 3, 0, False),
    (Q.FOLLOWER, 2, 0, 0, True), (Q.FOLLOWER, 2, 1, 0, True), (Q.FOLLOWER, 2, 2, 0, False), (Q.FOLLOWER, 2, 3, 0, False),
    (Q.FOLLOWER, 3, 0, 0, True), (Q.FOLLOWER, 3, 1, 0, True), (Q.FOLLOWER, 3, 2, 0, False), (Q.FOLLOWER, 3, 3, 0, False),
    (Q.FOLLOWER, 3, 2, 2, False), (Q.FOLLOWER, 3, 2, 1, True), (Q.LEADER, 3, 3, 1, True), (Q.PRE_CANDIDATE, 3, 3, 1, True),
    (Q.CANDIDATE, 3, 3, 1, True),
]


def recv_vote_case(row):
    role, index, log_term, vote, _ = row
    term = max(2, log_term)
    return _one(role, term, vote, 2, 2), [F.frame(0, 0, Q.request(Q.VOTE, term, log_term, index, frm=2))]


@pytest.mark.parametrize("row", range(len(RECV_VOTE)))
def test_recv_msg_request_vote(row):
    state, frames = recv_vote_case(RECV_VOTE[row])
    want = RECV_VOTE[row][4]
    r = _literal(state, frames)
    assert len(r) == 1 and r[0]["msg_type"] == 6 and bool(r[0]["reject"]) == want
    state, _ = recv_vote_case(RECV_VOTE[row])
    st, rb = _batch(state, frames)
    if RECV_VOTE[row][0] == Q.LEADER:   # a leader is the host's
        assert st.tolist() == [VR.WIRE_ROLE << 4] and rb == []
    else:
        assert st.tolist() == [(0 if want else VR.GRANTED | VR.VOTED)] and bool(rb[0]["reject"]) == want


# test_raft_paper.rs:962-1006: (log as (term, index) entries, m.log_term, m.index, want reject) at m.term 3
VOTER = [([(1, 1)], 1, 1, False), ([(1, 1)], 1, 2, False), ([(1, 1), (1, 2)], 1, 1, True),
         ([(1, 1)], 2, 1, False), ([(1, 1)], 2, 2, False), ([(1, 1), (1, 2)], 2, 1, False),
         ([(2, 1)], 1, 1, True), ([(2, 1)], 1, 2, True), ([(2, 1), (1, 2)], 1, 1, True)]


def voter_case(row):
    ents, log_term, index, _ = row
    # a new Raft at term 0 over that log (term 0 is the host's: the pass needs a known term, so the group sits at 1)
    state = _one(Q.FOLLOWER, 1, 0, len(ents), ents[-1][0], voters=0b11)
    return state, [F.frame(0, 0, Q.request(Q.VOTE, 3, log_term, index, frm=2))]


@pytest.mark.parametrize("row", range(len(VOTER)))
def test_voter(row):
    want = VOTER[row][3]
    for form in ("literal", "batch"):
        state, frames = voter_case(VOTER[row])
        r = _literal(state, frames) if form == "literal" else _batch(state, frames)[1]
        assert len(r) == 1 and r[0]["msg_type"] == 6 and bool(r[0]["reject"]) == want and r[0]["term"] == 3, form
        assert state[0].term[0] == 3   # the higher term was taken either way


def any_state_case(role, typ):
    """test_raft.rs:655-760: three voters, term 1 (a Follower whose leader is 3, a PreCandidate), 2 (a Candidate or a
    Leader, who voted for themselves; the leader appended its empty entry); a request from 2 at term + 1."""
    term = 2 if role in (Q.CANDIDATE, Q.LEADER) else 1
    vote = 1 if role in (Q.CANDIDATE, Q.LEADER) else 0
    last = 1 if role == Q.LEADER else 0
    state = _one(role, term, vote, last, term if last else 0, leader=role in (Q.FOLLOWER, Q.LEADER), voters=0b111)
    return state, [F.frame(0, 0, Q.request(typ, term + 1, term + 1, 42, frm=2))]


@pytest.mark.parametrize("typ", [Q.VOTE, Q.PRE_VOTE], ids=["vote", "prevote"])
@pytest.mark.parametrize("role", [Q.FOLLOWER, Q.CANDIDATE, Q.PRE_CANDIDATE, Q.LEADER])
def test_vote_from_any_state(role, typ):
    state, frames = any_state_case(role, typ)
    c, _, r_role, t = state
    orig = int(c.term[0])
    r = _literal(state, frames)
    assert len(r) == 1 and r[0]["msg_type"] == typ + 1 and not r[0]["reject"]
    if typ == Q.VOTE:
        assert (r_role[0], c.term[0], t["vote"][0]) == (Q.FOLLOWER, orig + 1, 2)
        assert c.term_start[0] == B.NO_TERM_START
    else:
        assert (r_role[0], c.term[0]) == (role, orig) and t["vote"][0] in (0, 1)
    state, frames = any_state_case(role, typ)
    st, rb = _batch(state, frames)
    if role == Q.LEADER:
        assert st.tolist() == [VR.WIRE_ROLE << 4]
    else:
        want = VR.GRANTED | (VR.VOTED | VR.BUMPED if typ == Q.VOTE else 0)
        assert st.tolist() == [want] and len(rb) == 1 and not rb[0]["reject"]


def test_lease_and_priority_cases():
    """The voter side of test_leader_election_with_check_quorum / test_prevote_with_check_quorum (a follower that heard
    from its leader ignores a higher-term request unless it is a transfer) and test_election_with_priority_log (a
    candidate with the same log but a lower priority is rejected; a longer log wins whatever the priority)."""
    for typ in (Q.VOTE, Q.PRE_VOTE):
        for ctx, dropped in ((b"", True), (Q.ELECTION, True), (Q.TRANSFER, False)):
            for form in ("literal", "batch"):
                state = _one(Q.FOLLOWER, 1, 0, 1, 1, leader=True, lease=True, check_quorum=True, voters=0b111)
                frames = [F.frame(0, 0, Q.request(typ, 2, 1, 1, context=ctx, frm=3))]
                if form == "literal":
                    r = _literal(state, frames)
                    assert len(r) == (0 if dropped else 1)
                else:
                    st, r = _batch(state, frames)
                    assert (st[0] >> 4 == VR.WIRE_IGNORED) == dropped and len(r) == (0 if dropped else 1)
                if not dropped:
                    assert not r[0]["reject"]
    for index, prio, want in ((1, 2, True), (1, 3, False), (1, 9, False), (2, 0, False)):
        for form in ("literal", "batch"):
            state = _one(Q.FOLLOWER, 1, 0, 1, 1, priority=3, voters=0b111)
            frames = [F.frame(0, 0, Q.request(Q.VOTE, 2, 1, index, priority=prio, frm=2))]
            r = _literal(state, frames) if form == "literal" else _batch(state, frames)[1]
            assert bool(r[0]["reject"]) == want, (index, prio, form)


def test_statuses_in_order():
    """Every status, each at the first check that fails, against a hand-built arena."""
    meta = B.make_meta(0b111, 0, 0, 0)
    c = O.new_columns(16, 6)
    c.term_start[:] = B.NO_TERM_START
    c.meta[:6] = meta
    c.term[:6] = [5, 5, 5, 0, 5, 5]
    c.last_index[:6], c.committed[:6] = 10, 8
    c.term_start[2] = 9
    t = np.zeros(6, VR.VOTER_DTYPE)
    t["id"], t["last_term"], t["flags"], t["commit_term"] = 1, 4, VR.SELECT, 3
    t["flags"][1] = 0
    t["flags"][5] = VR.SELECT | VR.LEADER | VR.LEASE
    frames = [F.frame(99, 0, Q.request(Q.VOTE, 6)),                       # MALFORMED: past the arena
              F.frame(0, 0, b"\x08"),                                    # MALFORMED: truncated
              F.frame(0, 0, Q.request(6, 6)),                            # SKIP_TYPE
              F.frame(1, 0, Q.request(Q.VOTE, 6)),                       # ROLE: not selected
              F.frame(2, 0, Q.request(Q.VOTE, 6)),                       # ROLE: a leader
              F.frame(3, 0, Q.request(Q.VOTE, 6)),                       # TERM: unknown term
              F.frame(0, 0, Q.request(Q.VOTE, 0)),                       # TERM: a local message
              F.frame(0, 0, Q.request(Q.VOTE, 4)),                       # IGNORED: lower-term vote
              F.frame(0, 0, Q.request(Q.VOTE, 6, 4, 10, frm=2)),         # DUP
              F.frame(4, 0, Q.request(Q.VOTE, 5, 3, 10, 9, 4, frm=2)),   # COMMIT_VOTE: stale log, commit ahead
              F.frame(5, 0, Q.request(Q.PRE_VOTE, 6, 4, 10, frm=2)),     # IGNORED: lease
              F.frame(5, 0, Q.request(Q.PRE_VOTE, 6, 4, 10, frm=2))]     # DUP
    blob, off = F.batch(frames)
    vt = np.zeros((O.SLOTS, c.cap), np.uint8)
    st, out, rb, ro, totals = VR.batch(c, None, vt, blob, off, t)
    W = B
    want = [W.WIRE_MALFORMED, W.WIRE_MALFORMED, W.WIRE_SKIP_TYPE, W.WIRE_ROLE, W.WIRE_ROLE, W.WIRE_TERM, W.WIRE_TERM,
            W.WIRE_IGNORED, W.WIRE_DUP, W.WIRE_COMMIT_VOTE, W.WIRE_IGNORED, W.WIRE_DUP]
    assert (st >> 4).tolist() == want and totals.tolist() == [0, 0] and not out.any()
    assert c.term[:6].tolist() == [5, 5, 5, 0, 5, 5]


# --------------------------------------------------------------------------- 3. the resubmission loop is exact


def state_of(s):
    c = O.new_columns(s.n + 8, s.n)
    c.term_start[:] = B.NO_TERM_START
    c.meta[s.n_narrow:s.n:2], c.meta[s.n_narrow + 1:s.n:2] = Q.META_WIDE_LO, Q.META_WIDE_HI   # the allocated pairs
    vt = np.zeros((O.SLOTS, c.cap), np.uint8)
    assert np.all(CO.arena_control(c, vt, s.setup)["status"] == 0)
    return c, vt


def caller_update(table, role, status, out, frames):
    """What the caller does with an applied frame's flags (INTEGRATION.md section 6)."""
    for i in np.flatnonzero(status >> 4 == B.WIRE_OK):
        g = int(np.frombuffer(frames[i][:4], "<u4")[0]) >> 4
        if status[i] & B.VREQ_BUMPED:   # become_follower(m.term, INVALID_ID)'s host side
            table["vote"][g] = 0
            table["flags"][g] &= ~np.uint32(VR.LEADER | VR.LEASE)
            role[g] = Q.FOLLOWER
        if status[i] & B.VREQ_VOTED:    # vote = m.from, election_elapsed = 0
            table["vote"][g] = out[i][0]
            if table["flags"][g] & VR.LEADER and table["flags"][g] & VR.CHECK_QUORUM:
                table["flags"][g] |= VR.LEASE


@pytest.mark.parametrize("seed", range(8))
def test_resubmission_loop_equals_the_literal_form(seed):
    rng = np.random.default_rng(0x7100 + seed)
    s = Q.Scenario(rng, 300, 40, p_role=(0.6, 0.2, 0.2, 0.0), p_select=1.0)
    for g in s.lows:   # some groups check the quorum
        if rng.random() < 0.5:
            s.table["flags"][g] |= VR.CHECK_QUORUM
    frames = s.frames(rng, per_group=(1, 4), noise=False, only_decided=True)
    frames = [frames[i] for i in rng.permutation(len(frames))]
    # the literal form, every frame in order
    c1, v1 = state_of(s)
    t1, r1 = s.table.copy(), s.role.copy()
    blob, off = F.batch(frames)
    rb, ro, _ = VR.literal(c1, None, v1, r1, t1, blob, off)
    lit = {}
    for k in range(len(ro) - 1):
        fr = rb[ro[k]:ro[k + 1]].tobytes()
        lit.setdefault(int(np.frombuffer(fr[:4], "<u4")[0]) >> 4, []).append(fr)
    # the batch form, DUP frames resubmitted in order until none is left
    c2, v2 = state_of(s)
    t2, r2 = s.table.copy(), s.role.copy()
    pending, rounds, got = frames, 0, {}
    while pending:
        blob, off = F.batch(pending)
        st, out, rb, ro, _ = VR.batch(c2, None, v2, blob, off, t2)
        assert np.all(np.isin(st >> 4, (B.WIRE_OK, B.WIRE_DUP, B.WIRE_IGNORED))), np.unique(st >> 4)
        for k in range(len(ro) - 1):
            fr = rb[ro[k]:ro[k + 1]].tobytes()
            got.setdefault(int(np.frombuffer(fr[:4], "<u4")[0]) >> 4, []).append(fr)
        caller_update(t2, r2, st, out, pending)
        pending = [pending[i] for i in np.flatnonzero(st >> 4 == B.WIRE_DUP)]
        rounds += 1
    assert rounds > 1 and got == lit
    for name in ("term", "term_start", "committed", "last_index", "matched", "next_idx", "peer_committed", "pflags"):
        assert np.array_equal(getattr(c1, name), getattr(c2, name)), name
    assert np.array_equal(v1, v2)
    assert np.array_equal(t1["vote"], t2["vote"]) and np.array_equal(t1["flags"], t2["flags"])
    assert np.array_equal(r1, r2)
