"""The oracle of the responses that reach a follower or a candidate (oracle/follow_resp_oracle.c) and of the
candidate's step-down in raftgpu_follower_term_wire's batch form, on the CPU: the reference's candidate cases on the
literal form and the batch forms, every status in check order, a claimant beside frames left for raftgpu_vote_wire,
and random bursts -- deposed leaders' late responses, lost candidates' late votes, higher-term rejections, wide
pairs -- on the batch form against the literal form in the reference's delivery order."""
import numpy as np
import pytest

from oracle import oracle as O
from oracle import follow_resp_oracle as FR
from oracle import follow_term_oracle as FT
from oracle import vote_request_oracle as VR
from helpers import B
import app_follow as A
import follow_resp as R
import follow_term as T
import hb_frames as F
import vote_request_frames as Q

COLUMNS = ("term", "term_start", "committed", "last_index", "matched", "next_idx", "peer_committed", "pflags")


def _same_arena(c1, c2):
    for name in COLUMNS:
        assert np.array_equal(getattr(c1, name), getattr(c2, name)), name


def _group(role, term, stale_reply=False, vote=1, voters=0b111):
    """One group (slot 0 = self, id 1) in `role` at `term`, with the candidate flags -> (columns, votes, role array,
    leader array, table)."""
    c, vt, r, t = Q.one(role, term, vote, 10, max(1, term - 1), voters=voters)
    t["flags"] |= R.candidate_flags(role) | (FT.STALE_REPLY if stale_reply else 0)
    return c, vt, r, np.zeros(c.cap, np.uint64), t


def _literal(state, frames_):
    c, vt, r, ld, t = state
    c1, v1, r1, l1, t1 = O.copy_columns(c), vt.copy(), r.copy(), ld.copy(), t.copy()
    blob, off = F.batch(frames_)
    outcome, rb, _, _ = FR.literal(c1, None, v1, r1, l1, t1, blob, off)
    return outcome, rb, c1, v1, r1, l1, t1


def _term_batch(state, frames_):
    """raftgpu_follower_term_wire's batch form and its host side on copies of state -> (status, out, replies, c, votes,
    role, leader, table)."""
    c, vt, r, ld, t = state
    c2, v2, r2, l2, t2 = O.copy_columns(c), vt.copy(), r.copy(), ld.copy(), t.copy()
    blob, off = F.batch(frames_)
    st, out, rb, _, _ = FR.term_batch(c2, None, v2, blob, off, t2)
    R.term_host_side(t2, r2, l2, st, out, frames_)
    return st, out, rb, c2, v2, r2, l2, t2


# --------------------------------------------------------------------------- 1. the reference's cases


@pytest.mark.parametrize("m_term", [1, 2, 3])
def test_candidate_fallback(m_term):
    """test_candidate_fallback (test_raft_paper.rs:292-320): a Candidate at term 1 that hears MsgAppend from n2 at term
    2 or 3 becomes a Follower at that term; at its own term 1 step_candidate's arm does the same (:2215-2219)."""
    state = _group(Q.CANDIDATE, 1)
    fr = [F.frame(0, 0, A.message(3, m_term, frm=2))]
    outcome, _, c1, v1, r1, l1, t1 = _literal(state, fr)
    st, out, _, c2, v2, r2, l2, t2 = _term_batch(state, fr)
    _same_arena(c1, c2)
    assert np.array_equal(v1, v2) and (r1[0], l1[0], c1.term[0]) == (r2[0], l2[0], c2.term[0]) == (Q.FOLLOWER, 2, m_term)
    assert np.array_equal(t1, t2) and outcome.tolist() == [FT.PASS]
    assert st.tolist() == [B.WIRE_OK << 4 | (B.FTERM_STEPPED if m_term == 1 else B.FTERM_BUMPED)]
    assert out.tolist() == [[2, m_term]] and t2["vote"][0] == (1 if m_term == 1 else 0)


@pytest.mark.parametrize("typ", [3, 8], ids=["append", "heartbeat"])
@pytest.mark.parametrize("candidate_term", [2, 3], ids=["below", "at"])
def test_candidate_reset_term_msg(typ, candidate_term):
    """test_candidate_reset_term_msg_{heartbeat,append} (test_raft.rs:1784-1848): the isolated n3 campaigns; the leader
    n1 at term 3 sends it a MsgHeartbeat or MsgAppend and n3 is a Follower at term 3.  "below": n3 campaigned to term 2
    (become_follower at the higher term); "at": n3 is a Candidate at the leader's term 3 (step_candidate's arm)."""
    state = _group(Q.CANDIDATE, candidate_term, vote=3, voters=0b111)
    body = A.message(3, 3, frm=1) if typ == 3 else F.message(8, 3, frm=1)
    fr = [F.frame(0, 2, body)]
    outcome, _, c1, v1, r1, l1, t1 = _literal(state, fr)
    st, out, _, c2, v2, r2, l2, t2 = _term_batch(state, fr)
    _same_arena(c1, c2)
    assert np.array_equal(v1, v2) and np.array_equal(t1, t2) and outcome.tolist() == [FT.PASS]
    assert (r1[0], l1[0], c1.term[0]) == (r2[0], l2[0], c2.term[0]) == (Q.FOLLOWER, 1, 3)
    assert st[0] & 0xF == (B.FTERM_STEPPED if candidate_term == 3 else B.FTERM_BUMPED)
    assert c2.term_start[0] == B.NO_TERM_START and not v2[:, 0].any()


def test_candidate_without_the_flag_is_left_as_before():
    """A candidate's row without RAFTGPU_VOTER_CANDIDATE: the frame at its term stays OK with nothing written."""
    state = _group(Q.CANDIDATE, 3)
    state[4]["flags"] &= ~np.uint32(B.VOTER_CANDIDATE)
    st, out, _, c2, _, r2, _, _ = _term_batch(state, [F.frame(0, 2, F.message(8, 3, frm=1))])
    _same_arena(c2, state[0])
    assert st.tolist() == [B.WIRE_OK << 4] and not out.any() and r2[0] == Q.CANDIDATE


def test_disruptive_follower_pre_vote():
    """test_disruptive_follower_pre_vote (test_raft.rs:2162-2227): n3 is a PreCandidate at term 2 -- pre-voting never
    raised its term -- and n1, leader at term 2, sends it a heartbeat: with the flag n3 steps down to a Follower of n1
    at term 2, its vote kept.  The pre-vote rejections of its peers that arrive afterwards, at term 2, are dropped by
    step_follower; a rejection that arrives before the heartbeat polls."""
    state = _group(Q.PRE_CANDIDATE, 2, stale_reply=True, vote=0)
    fr = [F.frame(0, 0, F.message(8, 2, commit=10, frm=1))]
    outcome, _, c1, v1, r1, l1, t1 = _literal(state, fr)
    st, out, _, c2, v2, r2, l2, t2 = _term_batch(state, fr)
    _same_arena(c1, c2)
    assert np.array_equal(v1, v2) and np.array_equal(t1, t2) and outcome.tolist() == [FT.PASS]
    assert (r2[0], l2[0], c2.term[0]) == (Q.FOLLOWER, 1, 2) and st.tolist() == [B.WIRE_OK << 4 | B.FTERM_STEPPED]
    late = [F.frame(0, 1, F.message(18, 2, reject=True, frm=1)), F.frame(0, 2, F.message(18, 2, reject=True, frm=2))]
    blob, off = F.batch(late)
    fst, fout = FR.batch(c2, None, v2, blob, off, t2)
    assert fst.tolist() == [B.WIRE_IGNORED << 4] * 2 and not fout.any()
    fst, _ = FR.batch(O.copy_columns(state[0]), None, state[1].copy(), blob, off, state[4])
    assert fst.tolist() == [B.WIRE_OK << 4] * 2


# --------------------------------------------------------------------------- 2. the statuses


def test_statuses_in_order():
    """Every status, first failing check first, and the verdicts of a Follower, a PreCandidate and a Candidate."""
    c = O.new_columns(16, 10)
    c.term_start[:] = B.NO_TERM_START
    c.meta[:10], c.term[:10], c.last_index[:10], c.committed[:10] = B.make_meta(0b111, 0, 0, 0), 5, 10, 8
    c.term[3] = 0
    c.meta[6], c.meta[7] = c.meta[6] | Q.META_WIDE_LO, c.meta[7] | Q.META_WIDE_HI
    c.term_start[2] = 9
    t = np.zeros(10, VR.VOTER_DTYPE)
    t["id"], t["flags"], t["persisted"] = 1, B.VOTER_SELECT, 10
    t["flags"][1] = 0
    t["flags"][4] |= B.VOTER_CANDIDATE | B.VOTER_PRE_CANDIDATE
    t["flags"][5] |= B.VOTER_CANDIDATE
    t["flags"][6] |= B.VOTER_CANDIDATE
    fr = [F.frame(99, 0, F.message(4, 6)), F.frame(0, 0, b"\x08"), F.frame(0, 0, F.message(3, 6, frm=2)),
          F.frame(1, 0, F.message(4, 6)), F.frame(2, 0, F.message(9, 6)), F.frame(3, 0, F.message(6, 6)),
          F.frame(0, 0, F.message(18, 0)),
          # the Follower 0: the claimant at 7, the other frames at 7, a stale frame
          F.frame(0, 1, F.message(9, 7)), F.frame(0, 2, F.message(6, 7)), F.frame(0, 3, F.message(4, 5)),
          # the PreCandidate 4 at its term: its own responses, a granting one above the term, the others dropped
          F.frame(4, 1, F.message(18, 5, reject=True)), F.frame(4, 2, F.message(18, 9)), F.frame(4, 3, F.message(6, 5)),
          F.frame(4, 4, F.message(4, 5)), F.frame(4, 5, F.message(18, 3)),
          # the Candidate 5: a granting pre-vote above the term is dropped, its own vote responses are left
          F.frame(5, 1, F.message(18, 8)), F.frame(5, 2, F.message(6, 5)), F.frame(5, 3, F.message(6, 5, reject=True)),
          # the Candidate pair 6-7 by its high half: a rejection at a higher term claims
          F.frame(7, 1, F.message(6, 5)), F.frame(7, 2, F.message(6, 6, reject=True)), F.frame(6, 3, F.message(9, 6))]
    blob, off = F.batch(fr)
    st, out = FR.batch(c, None, np.zeros((O.SLOTS, c.cap), np.uint8), blob, off, t)
    K, OK, IG, ST = B.WIRE_OK << 4 | B.FTERM_BUMPED, B.WIRE_OK << 4, B.WIRE_IGNORED << 4, B.WIRE_STALE << 4
    assert st.tolist() == [B.WIRE_MALFORMED << 4, B.WIRE_MALFORMED << 4, B.WIRE_SKIP_TYPE << 4, B.WIRE_ROLE << 4,
                           B.WIRE_ROLE << 4, B.WIRE_TERM << 4, B.WIRE_TERM << 4,
                           K, IG, ST,
                           OK, OK, IG, IG, ST,
                           IG, OK, OK,
                           ST, K, IG]
    assert out.tolist() == [0] * 7 + [7] + [0] * 11 + [6, 0]
    assert c.term[:8].tolist() == [7, 5, 5, 0, 5, 5, 6, 6]
    assert c.term_start[6] == c.term_start[7] == B.NO_TERM_START


def test_a_claimant_beside_frames_left_for_vote_wire():
    """In one batch a PreCandidate that hears a rejection at a higher term is claimed, and its granting pre-votes at
    or above the new term are then dropped, while a second PreCandidate's grants are left OK for raftgpu_vote_wire."""
    c = O.new_columns(8, 2)
    c.term_start[:] = B.NO_TERM_START
    c.meta[:2], c.term[:2], c.last_index[:2], c.committed[:2] = B.make_meta(0b11111, 0, 0, 0), 4, 10, 10
    t = np.zeros(2, VR.VOTER_DTYPE)
    t["flags"] = B.VOTER_SELECT | B.VOTER_CANDIDATE | B.VOTER_PRE_CANDIDATE
    fr = [F.frame(0, 1, F.message(18, 5)), F.frame(0, 2, F.message(18, 6, reject=True)), F.frame(0, 3, F.message(18, 7)),
          F.frame(1, 1, F.message(18, 5)), F.frame(1, 2, F.message(18, 4, reject=True)), F.frame(1, 3, F.message(18, 5))]
    blob, off = F.batch(fr)
    st, out = FR.batch(c, None, np.zeros((O.SLOTS, c.cap), np.uint8), blob, off, t)
    assert st.tolist() == [B.WIRE_STALE << 4, B.WIRE_OK << 4 | B.FTERM_BUMPED, B.WIRE_IGNORED << 4] + [B.WIRE_OK << 4] * 3
    assert out.tolist() == [0, 6, 0, 0, 0, 0] and c.term[:2].tolist() == [6, 4]


# --------------------------------------------------------------------------- 3. batch form vs literal form


def _state(s):
    c, vt = Q.state_of(s)
    return c, vt, s.role.copy(), s.leader.copy(), s.table.copy()


@pytest.mark.parametrize("seed", range(6))
def test_random_bursts_batch_equals_the_literal_form(seed):
    rng = np.random.default_rng(0x7600 + seed)
    s = R.scenario(rng, 300, 40)
    frames_, meta = R.frames(rng, s)
    perm = rng.permutation(len(frames_))
    frames_, meta = [frames_[i] for i in perm], [meta[i] for i in perm]
    blob, off = F.batch(frames_)
    c, vt, role, leader, table = _state(s)
    st, out = FR.batch(c, None, vt, blob, off, table)
    groups = [m[0] for m in meta]
    R.host_side(table, role, leader, st, out, groups)
    passing = [i for i in range(len(frames_)) if st[i] >> 4 in (B.WIRE_OK, B.WIRE_IGNORED, B.WIRE_STALE)]
    host = [i for i in range(len(frames_)) if i not in set(passing)]
    assert all(st[i] >> 4 == B.WIRE_ROLE for i in host)
    assert all(s.role[meta[i][0]] == Q.LEADER or not s.table["flags"][meta[i][0]] & B.VOTER_SELECT for i in host)
    # the reference: the passing frames one at a time in the delivery order
    c1, vt1, role1, leader1, table1 = _state(s)
    sub = [meta[i] for i in passing]
    verdict = {}
    for k in R.delivery_order(s, sub):
        i = passing[k]
        b1, o1 = F.batch([frames_[i]])
        outcome, _, _, _ = FR.literal(c1, None, vt1, role1, leader1, table1, b1, o1)
        verdict[i] = int(outcome[0])
    table1["flags"][role1 != s.role] |= B.VOTER_SELECT   # the caller's select bits for the groups it made Followers
    _same_arena(c, c1)
    assert np.array_equal(vt, vt1) and np.array_equal(role, role1) and np.array_equal(leader, leader1)
    assert np.array_equal(table, table1)
    for i in passing:
        assert verdict[i] == R.outcome_of(st[i]), (i, int(st[i]), meta[i])
        assert out[i] == (c.term[meta[i][0]] if st[i] & B.FTERM_BUMPED else 0)
    kinds = np.bincount(st >> 4, minlength=16)
    assert kinds[B.WIRE_OK] > 30 and kinds[B.WIRE_STALE] > 100 and kinds[B.WIRE_IGNORED] > 100
    assert np.count_nonzero(st & B.FTERM_BUMPED) > 50


@pytest.mark.parametrize("seed", range(4))
def test_random_step_downs_batch_equals_the_literal_form(seed):
    """raftgpu_follower_term_wire's batch form with the candidate flags against the literal form: the claimant first
    (a bump or a step-down), then the other frames at T, then the stale ones; the frames left OK reach the follower's
    handler in both."""
    rng = np.random.default_rng(0x7610 + seed)
    s = R.scenario(rng, 300, 40, p_role=(0.3, 0.3, 0.4, 0.0))
    frames_ = T.frames(rng, s, deltas=(-1, 0, 0, 0, 1))
    frames_ = [frames_[i] for i in rng.permutation(len(frames_))]
    c, vt, role, leader, table = _state(s)
    state = (c, vt, role, leader, table)
    st, out, rb, c2, v2, r2, l2, t2 = _term_batch(state, frames_)
    groups = [int(np.frombuffer(f[:4], "<u4")[0]) >> 4 for f in frames_]
    assert np.count_nonzero(st & B.FTERM_STEPPED) > 50 and np.count_nonzero(st & B.FTERM_BUMPED) > 20
    # the literal form in the delivery order: each group's claimant, its other frames at T, then its stale frames
    claim = [i for i in range(len(frames_)) if st[i] & (B.FTERM_BUMPED | B.FTERM_STEPPED)]
    rest = [i for i in range(len(frames_)) if st[i] == B.WIRE_OK << 4]
    stale = [i for i in range(len(frames_)) if st[i] >> 4 == B.WIRE_STALE]
    c1, v1, r1, l1, t1 = _state(s)
    replies = {}
    for i in claim + rest + stale:
        b1, o1 = F.batch([frames_[i]])
        outcome, r, _, _ = FR.literal(c1, None, v1, r1, l1, t1, b1, o1)
        want = {B.WIRE_OK: FT.PASS, B.WIRE_STALE: FT.ANSWERED if st[i] & B.RES_OK else FT.DROPPED}[st[i] >> 4]
        assert outcome[0] == want, (i, int(st[i]), groups[i])
        replies[i] = r.tobytes()
    t1["flags"][r1 != s.role] |= B.VOTER_SELECT   # the caller's select bits for the groups it made Followers
    _same_arena(c1, c2)
    assert np.array_equal(v1, v2) and np.array_equal(r1, r2) and np.array_equal(l1, l2) and np.array_equal(t1, t2)
    assert rb.tobytes() == b"".join(replies[i] for i in sorted(replies))
