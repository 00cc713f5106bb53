"""The vote-response oracle (oracle/vote_wire_oracle.c) on the CPU: the encoder goldens, the reference's election
tables restated through frames, each status, and the batch form against the literal one -- the first decided result
of every group in many orders, and the caller's recipe (batch form, then the transition lists) against the reference's
transitions."""
import json
import os

import numpy as np
import pytest

from oracle import oracle as O
from oracle import control_oracle as CO
from oracle import hb_wire_oracle as H
from oracle import vote_wire_oracle as VW
from helpers import B
from control_cmds import cmds
import hb_frames as F
import vote_frames as V

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "wire", "vote_responses.json")


def _golden():
    with open(GOLDEN, encoding="utf-8") as f:
        return json.load(f)["vectors"]


# --------------------------------------------------------------------------- 1. the encoders


def test_test_encoder_matches_python_protobuf():
    vs = _golden()
    assert len(vs) > 800
    for v in vs:
        got = V.message(v["msg_type"], v["term"], v["reject"], v["commit"], v["commit_term"], to=v["to"], frm=v["from"])
        assert got.hex() == v["hex"], v
        m = H.decode_message(got)   # the oracle's decoder reads every field back
        assert (m["msg_type"], m["term"], bool(m["reject"]), m["commit"], m["commit_term"]) == \
            (v["msg_type"], v["term"], v["reject"], v["commit"], v["commit_term"])


def test_synth_encoder_matches_python_protobuf():
    vs = _golden()
    e = np.zeros(len(vs), B.SYNTH_VOTE_DTYPE)
    for i, v in enumerate(vs):
        e[i]["hdr"] = (i % 1000) << 4 | (i % 16)
        for k in ("msg_type", "to", "from", "term", "commit", "commit_term"):
            e[i][k] = v[k]
        e[i]["reject"] = v["reject"]
    blob, off = B.synth_encode_votes(e)
    for i, v in enumerate(vs):
        fr = blob[off[i]:off[i + 1]].tobytes()
        assert fr[:4] == np.array([(i % 1000) << 4 | (i % 16)], "<u4").tobytes()
        assert fr[4:].hex() == v["hex"], v


# --------------------------------------------------------------------------- 2. one group at a time


def same_decisions(outs, first):
    """The pass's outcomes against the literal form's first decided words: the same groups and VoteResults (the counts
    differ where votes came in after the decision: the pass tallies once, after the batch)."""
    want = VW.outcomes_of(first)
    return np.array_equal(outs["group"], want["group"]) and np.array_equal(outs["result"] & 0xFF, want["result"] & 0xFF)


def one_round_case(size, votes):
    """The case on a fresh arena: the campaign list of INTEGRATION.md section 6 (term 0 -> 1, self vote in slot 0),
    then the responses as frames (peer id k in slot k - 1) -> (campaign's VOTE_RESULT word, frames, columns, votes)."""
    c, vt = V.candidates([B.make_meta((1 << size) - 1, 0, 0, 0)], [0])
    camp = cmds((B.CTL_RESET, 0, 0, 0, (B.NO_TERM_START, 10, 5, 10)), (B.CTL_SET_TERM, 0, 0, 0, (1,)),
                (B.CTL_RESET_VOTES, 0), (B.CTL_RECORD_VOTE, 0, 0, 1), (B.CTL_VOTE_RESULT, 0))
    first = int(CO.arena_control(c, vt, camp)["value"][-1])
    frames = [F.frame(0, k - 1, V.message(6, 1, not v, to=1, frm=k)) for k, v in votes.items()]
    return first, frames, c, vt


@pytest.mark.parametrize("case", range(len(V.ONE_ROUND)))
def test_leader_election_in_one_round_rpc(case):
    size, votes, state = V.ONE_ROUND[case]
    first, frames, c, vt = one_round_case(size, votes)
    st, outs, tallied = V.run_batch(c, vt, frames, [True])
    assert np.all(st == (B.WIRE_OK << 4 | B.RES_OK))
    assert tallied == (1 if frames else 0)
    # a single voter wins on its own vote: the campaign list decides it, and there is no frame to pass
    assert V.expected_state(first, outs) == state
    assert len(outs) == (state != "Candidate" and bool(frames))
    assert int(c.term[0]) == 1
    # the literal form agrees
    _, frames, c2, vt2 = one_round_case(size, votes)
    role = np.array([V.CANDIDATE], np.uint8)
    blob, off = F.batch(frames)
    got = VW.literal(c2, vt2, role, blob, off)
    assert same_decisions(outs, got)
    if frames:   # and its transitions leave the role the table names
        assert {V.LEADER: "Leader", V.FOLLOWER: "Follower", V.CANDIDATE: "Candidate"}[int(role[0])] == state


def test_statuses_in_order():
    """Each check of raftgpu.h on a candidate (group 0, term 7), a PreCandidate (group 1, term 7), a leader (2) and an
    unselected group (3); committed 5."""
    meta = B.make_meta(0x1F, 0, 0, 0)
    c, vt = V.candidates([meta] * 4, [7, 7, 7, 7])
    c.term_start[2] = 11
    sel, pre = [True, True, True, False], [False, True, False, False]
    rows = [
        (F.frame(9, 1, V.message(6, 7)), B.WIRE_MALFORMED),                       # group past the arena
        (F.frame(0, 1, b"\x08"), B.WIRE_MALFORMED),                               # truncated protobuf
        (F.frame(0, 1, V.message(4, 7)), B.WIRE_SKIP_TYPE),                       # MsgAppendResponse
        (F.frame(0, 1, V.message(9, 7)), B.WIRE_SKIP_TYPE),                       # MsgHeartbeatResponse
        (F.frame(3, 1, V.message(6, 7)), B.WIRE_ROLE),                            # not selected
        (F.frame(2, 1, V.message(6, 7)), B.WIRE_ROLE),                            # a leader
        (F.frame(0, 1, V.message(18, 7)), B.WIRE_ROLE),                           # pre-vote response at a Candidate
        (F.frame(1, 1, V.message(6, 7)), B.WIRE_ROLE),                            # vote response at a PreCandidate
        (F.frame(0, 1, V.message(6, 0)), B.WIRE_TERM),                            # m.term 0
        (F.frame(0, 1, V.message(6, 8)), B.WIRE_TERM),                            # Candidate: higher
        (F.frame(0, 1, V.message(6, 6)), B.WIRE_TERM),                            # Candidate: lower
        (F.frame(1, 1, V.message(18, 6)), B.WIRE_TERM),                           # PreCandidate: lower
        (F.frame(1, 1, V.message(18, 8, True)), B.WIRE_TERM),                     # PreCandidate: higher rejection
        (F.frame(0, 2, V.message(6, 7, commit=6, commit_term=7)), B.WIRE_COMMIT_VOTE),
        (F.frame(0, 2, V.message(6, 7, commit=6)), B.WIRE_OK),                    # commit_term 0: no maybe_commit_by_vote
        (F.frame(0, 3, V.message(6, 7, commit=5, commit_term=7)), B.WIRE_OK),     # not beyond committed
        (F.frame(0, 2, V.message(6, 7, True)), B.WIRE_DUP),                       # the cell's second frame
        (F.frame(1, 1, V.message(18, 8)), B.WIRE_OK),                             # granted pre-vote at term + 1
        (F.frame(1, 2, V.message(18, 7, True)), B.WIRE_OK),                       # pre-vote rejection at the term
        (F.frame(1, 9, V.message(18, 7)), B.WIRE_OK),                             # slot 9: no such peer
    ]
    st, outs, tallied = V.run_batch(c, vt, [f for f, _ in rows], sel, pre)
    assert (st >> 4).tolist() == [s for _, s in rows]
    assert st[-1] & 0xF == B.RES_NO_PROGRESS and st[-2] & 0xF == B.RES_OK and st[-6] & 0xF == B.RES_OK
    assert vt[:, 0].tolist()[:4] == [0, 0, 2, 2] and vt[:, 1].tolist()[:3] == [0, 2, 1]
    # group 0: slots 2 and 3 granted of 5 voters, pending; group 1: slot 1 granted, slot 2 rejected, pending
    assert tallied == 2 and outs.tolist() == []
    # the same frames, the rejected cell already voted before the batch: or_insert keeps the old vote, result 0
    c, vt = V.candidates([meta] * 4, [7, 7, 7, 7])
    c.term_start[2] = 11
    vt[2, 0] = 1
    st, _, _ = V.run_batch(c, vt, [f for f, _ in rows], sel, pre)
    assert st[14] == (B.WIRE_OK << 4) and vt[2, 0] == 1


def test_group_without_voters_is_role():
    """A selected group slot without voters -- freed (meta 0, its term left behind) or not configured yet -- is the
    host's: the pass neither records nor tallies it, so only allocated groups reach the outcome list."""
    meta = B.make_meta(0b11, 0, 0, 0)
    c, vt = V.candidates([meta, 0, 0], [4, 4, 4])
    vt[0, 0] = 2                                               # group 0's self vote
    frames = [F.frame(g, 1, V.message(6, 4)) for g in (1, 0, 2)]
    st, outs, tallied = V.run_batch(c, vt, frames, [True, True, True])
    assert (st >> 4).tolist() == [B.WIRE_ROLE, B.WIRE_OK, B.WIRE_ROLE]
    assert outs.tolist() == [(0, B.VOTE_WON | 2 << 8)] and tallied == 1
    assert np.count_nonzero(vt[:, 1:3]) == 0


def test_pre_vote_terms_and_commit_by_vote():
    """A PreCandidate at term 5 with 3 voters: granted pre-votes from term 6 win without changing the term; a rejection
    at a higher term is the host's.  test_advance_commit_index_by_vote_response's shape (test_raft.rs:4646-4800): a
    response whose commit is beyond committed with a commit_term is COMMIT_VOTE and records nothing."""
    meta = B.make_meta(0b111, 0, 0, 0)
    c, vt = V.candidates([meta, meta], [5, 5], committed=[3, 3])
    vt[0, 0] = vt[0, 1] = 2                                    # both self votes
    frames = [F.frame(0, 1, V.message(18, 6)), F.frame(1, 1, V.message(18, 6, True)),
              F.frame(1, 2, V.message(18, 5, commit=4, commit_term=5)), F.frame(1, 2, V.message(18, 5, True, commit=3, commit_term=5))]
    st, outs, _ = V.run_batch(c, vt, frames, [True, True], [True, True])
    assert (st >> 4).tolist() == [B.WIRE_OK, B.WIRE_TERM, B.WIRE_COMMIT_VOTE, B.WIRE_OK]
    assert outs.tolist() == [(0, B.VOTE_WON | 2 << 8)] and c.term[:2].tolist() == [5, 5]
    assert vt[2, 1] == 1


# --------------------------------------------------------------------------- 3. batch form against the literal form


@pytest.mark.parametrize("seed", range(6))
def test_batch_equals_literal_first_results_in_any_order(seed):
    rng = np.random.default_rng(0x707E + seed)
    e = V.Election(rng, 300, 40)
    frames = e.frames(rng)
    for perm in range(8):
        order = rng.permutation(len(frames))
        blob, off = F.batch([frames[i] for i in order])
        c, vt = V.state_of(e)
        st, outs, tallied = VW.batch(c, vt, blob, off, e.select(), e.pre())
        c2, vt2 = V.state_of(e)
        role = e.role.copy()
        first = VW.literal(c2, vt2, role, blob, off)
        assert same_decisions(outs, first), (seed, perm)
        assert len(outs) > 20 and tallied > len(outs)
        kinds = np.bincount(st >> 4, minlength=16)
        assert all(kinds[k] > 0 for k in (B.WIRE_OK, B.WIRE_DUP, B.WIRE_ROLE, B.WIRE_TERM, B.WIRE_SKIP_TYPE,
                                          B.WIRE_MALFORMED)), kinds


@pytest.mark.parametrize("seed", range(4))
def test_caller_recipe_equals_literal_transitions(seed):
    """The batch form, then the transition lists of the outcomes, leaves the arena -- every column, the votes and the
    terms -- where the reference's one-frame-at-a-time transitions leave it."""
    rng = np.random.default_rng(0x7E57 + seed)
    e = V.Election(rng, 250, 30)
    frames = e.frames(rng)
    blob, off = F.batch([frames[i] for i in rng.permutation(len(frames))])
    c, vt = V.state_of(e)
    _, outs, _ = VW.batch(c, vt, blob, off, e.select(), e.pre())
    res = CO.arena_control(c, vt, e.transitions(outs, e.role))
    assert np.all(res["status"] == 0)
    c2, vt2 = V.state_of(e)
    role = e.role.copy()
    VW.literal(c2, vt2, role, blob, off)
    for name in O.PEER_COLUMNS + ("pflags", "meta") + O.GROUP_COLUMNS:
        assert np.array_equal(getattr(c, name), getattr(c2, name)), name
    assert np.array_equal(vt, vt2)
    won = outs["result"] & 0xFF == B.VOTE_WON
    assert won.sum() > 10 and (~won).sum() > 10
