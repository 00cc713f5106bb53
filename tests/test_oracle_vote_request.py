"""The vote-request oracle (oracle/vote_request_oracle.c) on the CPU: the encoder goldens, the reference's voter tables
restated on the literal form and through the batch form, and the exactness of the batch form's resubmission loop against
the literal form."""
import json
import os

import numpy as np
import pytest

from oracle import oracle as O
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


@pytest.mark.parametrize("row", range(len(Q.RECV_VOTE)))
def test_recv_msg_request_vote(row):
    state, frames = Q.recv_vote_case(Q.RECV_VOTE[row])
    want = Q.RECV_VOTE[row][4]
    r = _literal(state, frames)
    assert len(r) == 1 and r[0]["msg_type"] == 6 and bool(r[0]["reject"]) == want
    state, _ = Q.recv_vote_case(Q.RECV_VOTE[row])
    st, rb = _batch(state, frames)
    if Q.RECV_VOTE[row][0] == Q.LEADER:   # a leader is the host's
        assert st.tolist() == [VR.WIRE_ROLE << 4] and rb == []
    else:
        assert st.tolist() == [(0 if want else VR.GRANTED | VR.VOTED)] and bool(rb[0]["reject"]) == want


@pytest.mark.parametrize("row", range(len(Q.VOTER)))
def test_voter(row):
    want = Q.VOTER[row][3]
    for form in ("literal", "batch"):
        state, frames = Q.voter_case(Q.VOTER[row])
        r = _literal(state, frames) if form == "literal" else _batch(state, frames)[1]
        assert len(r) == 1 and r[0]["msg_type"] == 6 and bool(r[0]["reject"]) == want and r[0]["term"] == 3, form
        assert state[0].term[0] == 3   # the higher term was taken either way


@pytest.mark.parametrize("typ", [Q.VOTE, Q.PRE_VOTE], ids=["vote", "prevote"])
@pytest.mark.parametrize("role", [Q.FOLLOWER, Q.CANDIDATE, Q.PRE_CANDIDATE, Q.LEADER])
def test_vote_from_any_state(role, typ):
    state, frames = Q.any_state_case(role, typ)
    c, _, r_role, t = state
    orig = int(c.term[0])
    r = _literal(state, frames)
    assert len(r) == 1 and r[0]["msg_type"] == typ + 1 and not r[0]["reject"]
    if typ == Q.VOTE:
        assert (r_role[0], c.term[0], t["vote"][0]) == (Q.FOLLOWER, orig + 1, 2)
        assert c.term_start[0] == B.NO_TERM_START
    else:
        assert (r_role[0], c.term[0]) == (role, orig) and t["vote"][0] in (0, 1)
    state, frames = Q.any_state_case(role, typ)
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
                state = Q.one(Q.FOLLOWER, 1, 0, 1, 1, leader=True, lease=True, check_quorum=True, voters=0b111)
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
            state = Q.one(Q.FOLLOWER, 1, 0, 1, 1, priority=3, voters=0b111)
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
    c1, v1 = Q.state_of(s)
    t1, r1 = s.table.copy(), s.role.copy()
    blob, off = F.batch(frames)
    rb, ro, _ = VR.literal(c1, None, v1, r1, t1, blob, off)
    lit = {}
    for k in range(len(ro) - 1):
        fr = rb[ro[k]:ro[k + 1]].tobytes()
        lit.setdefault(int(np.frombuffer(fr[:4], "<u4")[0]) >> 4, []).append(fr)
    # the batch form, DUP frames resubmitted in order until none is left
    c2, v2 = Q.state_of(s)
    t2, r2 = s.table.copy(), s.role.copy()
    pending, rounds, got = frames, 0, {}
    while pending:
        blob, off = F.batch(pending)
        st, out, rb, ro, _ = VR.batch(c2, None, v2, blob, off, t2)
        assert np.all(np.isin(st >> 4, (B.WIRE_OK, B.WIRE_DUP, B.WIRE_IGNORED))), np.unique(st >> 4)
        for k in range(len(ro) - 1):
            fr = rb[ro[k]:ro[k + 1]].tobytes()
            got.setdefault(int(np.frombuffer(fr[:4], "<u4")[0]) >> 4, []).append(fr)
        Q.caller_update(t2, r2, st, out, pending)
        pending = [pending[i] for i in np.flatnonzero(st >> 4 == B.WIRE_DUP)]
        rounds += 1
    assert rounds > 1 and got == lit
    for name in ("term", "term_start", "committed", "last_index", "matched", "next_idx", "peer_committed", "pflags"):
        assert np.array_equal(getattr(c1, name), getattr(c2, name)), name
    assert np.array_equal(v1, v2)
    assert np.array_equal(t1["vote"], t2["vote"]) and np.array_equal(t1["flags"], t2["flags"])
    assert np.array_equal(r1, r2)
