"""The follower term-prefix oracle (oracle/follow_term_oracle.c) on the CPU: the stale reply's encoder and the frames'
decoder against python-protobuf, the reference's term-rule cases restated on the literal form and through the batch
form, and the batch form followed by the follower passes against the literal form on random batches."""
import json
import os

import numpy as np
import pytest

from oracle import oracle as O
from oracle import follow_term_oracle as FT
from oracle import hb_wire_oracle as H
from oracle import vote_request_oracle as VR
from helpers import B
import app_follow as A
import follow_term as T
import hb_frames as F
import vote_request_frames as Q

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "wire", "follower_terms.json")


def _golden():
    with open(GOLDEN, encoding="utf-8") as f:
        return json.load(f)


# --------------------------------------------------------------------------- 1. the encoder and the decoder


def test_stale_reply_encoder_matches_python_protobuf():
    vs = _golden()["replies"]
    assert len(vs) == 7 ** 3
    for v in vs:
        assert FT.encode_reply(v["to"], v["from"], v["term"]).hex() == v["hex"], v
        assert 4 + 2 + 33 >= 4 + len(bytes.fromhex(v["hex"]))   # FRAME_MAX covers every reply
    assert max(4 + len(bytes.fromhex(v["hex"])) for v in vs) == FT.FRAME_MAX


def test_frames_decode_as_python_protobuf_wrote_them():
    for v in _golden()["frames"]:
        m = H.decode_message(bytes.fromhex(v["hex"]))
        assert m is not None and m["msg_type"] == v["msg_type"], v
        assert (m["from"], m["term"], m["commit"]) == (v["from"], v["term"], v["commit"]), v


# --------------------------------------------------------------------------- 2. the reference's cases


def _one(role, term, stale_reply=False, last_index=10, voters=0b111, pid=1):
    """One group (slot 0 = self, id pid) in `role` at `term` -> (columns, votes, role array, leader array, table)."""
    c, vt, r, t = Q.one(role, term, pid if role != Q.FOLLOWER else 0, last_index, max(1, term - 1), voters=voters)
    t["id"] = pid
    if stale_reply:
        t["flags"] |= FT.STALE_REPLY
    return c, vt, r, np.zeros(c.cap, np.uint64), t


def _both(state, frames_):
    """The literal form and the batch form on copies of state -> ((outcome, replies, c), (status, out, replies, c))."""
    c, vt, r, ld, t = state
    c1, v1, r1, l1, t1 = O.copy_columns(c), vt.copy(), r.copy(), ld.copy(), t.copy()
    blob, off = F.batch(frames_)
    outcome, rb, ro, _ = FT.literal(c1, None, v1, r1, l1, t1, blob, off)
    c2, v2 = O.copy_columns(c), vt.copy()
    st, out, rb2, ro2, _ = FT.batch(c2, None, v2, blob, off, t)
    return (outcome, rb, c1, r1, l1, t1), (st, out, rb2, c2)


@pytest.mark.parametrize("msg_type", [T.APPEND, T.HEARTBEAT])
@pytest.mark.parametrize("role", [Q.FOLLOWER, Q.PRE_CANDIDATE, Q.CANDIDATE, Q.LEADER])
def test_update_term_from_message(role, msg_type):
    """test_raft_paper.rs:57-100: a message at term 2 makes a node at term 1 a Follower at term 2, whatever its role."""
    state = _one(role, 1)
    body = A.message(3, 2, frm=2) if msg_type == T.APPEND else F.message(8, 2, frm=2)
    (outcome, _, c1, r1, l1, _), (st, out, _, c2) = _both(state, [F.frame(0, 0, body)])
    assert outcome.tolist() == [FT.PASS] and c1.term[0] == 2 and r1[0] == Q.FOLLOWER and l1[0] == 2
    assert c1.term_start[0] == B.NO_TERM_START
    if role == Q.LEADER:   # a leader's step-down stays with the host
        assert st.tolist() == [B.WIRE_ROLE << 4] and c2.term[0] == 1
    else:
        assert st.tolist() == [B.WIRE_OK << 4 | B.FTERM_BUMPED] and out.tolist() == [[2, 2]]
        for name in ("term", "term_start", "committed", "last_index", "matched", "next_idx", "pflags"):
            assert np.array_equal(getattr(c1, name), getattr(c2, name)), name


@pytest.mark.parametrize("msg_type", [T.APPEND, T.HEARTBEAT])
def test_candidate_reset_term(msg_type):
    """The higher-term part of test_candidate_reset_term_msg_{heartbeat,append} (test_raft.rs:1784-1848): a Candidate
    at term 2 that hears the leader (id 1) at term 3 becomes its Follower at term 3."""
    state = _one(Q.CANDIDATE, 2, pid=3)
    body = A.message(3, 3, 2, 10, frm=1) if msg_type == T.APPEND else F.message(8, 3, frm=1)
    (outcome, _, c1, r1, l1, t1), (st, out, _, c2) = _both(state, [F.frame(0, 5, body)])
    assert outcome.tolist() == [FT.PASS] and (c1.term[0], r1[0], l1[0], t1["vote"][0]) == (3, Q.FOLLOWER, 1, 0)
    assert st.tolist() == [B.WIRE_OK << 4 | B.FTERM_BUMPED] and out.tolist() == [[1, 3]] and c2.term[0] == 3


@pytest.mark.parametrize("pre_vote", [False, True])
@pytest.mark.parametrize("stale_reply", [False, True])
def test_disruptive_follower(stale_reply, pre_vote):
    """test_disruptive_follower (test_raft.rs:2088-2160): n3, a Candidate at term 3, hears n1's heartbeat at term 2 and
    answers with a MsgAppendResponse at term 3 -- only when check_quorum or pre_vote is on.  _pre_vote (:2162-2227):
    n3, a PreCandidate at n1's term 2, lets the heartbeat through at that term."""
    if pre_vote:
        state = _one(Q.PRE_CANDIDATE, 2, stale_reply, pid=3)
        (outcome, rb, c1, _, _, _), (st, _, rb2, c2) = _both(state, [F.frame(0, 1, F.message(8, 2, 7, frm=1))])
        assert outcome.tolist() == [FT.PASS] and st.tolist() == [B.WIRE_OK << 4] and len(rb) == len(rb2) == 0
        assert c1.term[0] == c2.term[0] == 2
        return
    state = _one(Q.CANDIDATE, 3, stale_reply, pid=3)
    (outcome, rb, c1, _, _, _), (st, out, rb2, c2) = _both(state, [F.frame(0, 1, F.message(8, 2, 7, frm=1))])
    assert c1.term[0] == c2.term[0] == 3 and out.tolist() == [[0, 0]]
    if stale_reply:
        want = np.array([0 << 4 | 1], "<u4").tobytes() + FT.encode_reply(1, 3, 3)
        assert outcome.tolist() == [FT.ANSWERED] and st.tolist() == [B.WIRE_STALE << 4 | B.RES_OK]
        assert rb.tobytes() == rb2.tobytes() == want
    else:
        assert outcome.tolist() == [FT.DROPPED] and st.tolist() == [B.WIRE_STALE << 4]
        assert len(rb) == len(rb2) == 0


def test_free_stuck_candidate_with_check_quorum():
    """test_free_stuck_candidate_with_check_quorum (test_raft.rs:1989-2040): c (id 3), stuck as a Candidate at term 2,
    answers a's heartbeat at term 1 with an empty MsgAppendResponse at term 2, which frees it once a steps down."""
    state = _one(Q.CANDIDATE, 2, True, pid=3)
    (outcome, rb, _, _, _, _), (st, _, rb2, c2) = _both(state, [F.frame(0, 9, F.message(8, 1, frm=1))])
    assert outcome.tolist() == [FT.ANSWERED] and st.tolist() == [B.WIRE_STALE << 4 | B.RES_OK] and c2.term[0] == 2
    msg = H.decode_message(rb2.tobytes()[4:])
    assert rb.tobytes() == rb2.tobytes() and (msg["msg_type"], msg["to"], msg["from"], msg["term"]) == (4, 1, 3, 2)
    assert msg["index"] == msg["commit"] == msg["log_term"] == 0 and not msg["reject"]


def test_statuses_in_order():
    """Every status, first failing check first, and a group's claimant at the lowest frame of the highest term."""
    c = O.new_columns(16, 6)
    c.term_start[:] = B.NO_TERM_START
    c.meta[:6], c.term[:6], c.last_index[:6], c.committed[:6] = B.make_meta(0b111, 0, 0, 0), [5, 5, 5, 0, 5, 5], 10, 8
    c.term_start[2] = 9
    t = np.zeros(6, VR.VOTER_DTYPE)
    t["id"], t["flags"], t["persisted"] = 1, VR.SELECT | FT.STALE_REPLY, 10
    t["flags"][1] = 0
    hb = lambda g, term, frm=2: F.frame(g, 0, F.message(8, term, frm=frm))
    frames_ = [hb(99, 6), F.frame(0, 0, b"\x08"), F.frame(0, 0, F.message(9, 6)), hb(1, 6), hb(2, 6), hb(3, 6), hb(0, 0),
               hb(0, 4), hb(0, 6), hb(0, 7, 3), hb(0, 7, 3), hb(0, 6), hb(4, 5), hb(4, 4)]
    blob, off = F.batch(frames_)
    st, out, rb, ro, tot = FT.batch(c, None, np.zeros((O.SLOTS, c.cap), np.uint8), blob, off, t)
    assert (st >> 4).tolist() == [B.WIRE_MALFORMED, B.WIRE_MALFORMED, B.WIRE_SKIP_TYPE, B.WIRE_ROLE, B.WIRE_ROLE,
                                  B.WIRE_TERM, B.WIRE_TERM, B.WIRE_STALE, B.WIRE_STALE, B.WIRE_OK, B.WIRE_OK,
                                  B.WIRE_STALE, B.WIRE_OK, B.WIRE_STALE]
    assert st[9] & 0xF == B.FTERM_BUMPED and st[10] & 0xF == 0 and out[9].tolist() == [3, 7] and out[10].tolist() == [0, 0]
    assert c.term[0] == 7 and c.term[4] == 5 and tot.tolist() == [4, ro[-1]]
    for k, i in enumerate((7, 8, 11, 13)):
        want = frames_[i][:4] + FT.encode_reply(2, 1, 7 if i != 13 else 5)
        assert rb[ro[k]:ro[k + 1]].tobytes() == want


# --------------------------------------------------------------------------- 3. batch form vs literal form


def _literal_sequence(s, frames_, order):
    """The literal form over frames_ in `order`, each frame it passes then through the follower passes' batch forms
    alone -> (columns, votes, role, leader, table, {frame: verdict}, sorted responses, stale replies)."""
    c, vt = Q.state_of(s)
    role, leader, table = s.role.copy(), s.leader.copy(), s.table.copy()
    verdict, resps, stale = {}, [], []
    for i in order:
        blob, off = F.batch([frames_[i]])
        outcome, rb, _, _ = FT.literal(c, None, vt, role, leader, table, blob, off)
        if outcome[0] == FT.PASS:
            final, r = T.follower_passes(c, s, role, table, frames_, [i])
            verdict[i] = ("pass", final[i])
            resps += r
        else:
            verdict[i] = ("stale", outcome[0] == FT.ANSWERED)
            stale.append(rb.tobytes())
    return c, vt, role, leader, table, verdict, sorted(resps), stale


@pytest.mark.parametrize("seed", range(6))
def test_batch_then_follower_passes_equal_the_literal_form(seed):
    rng = np.random.default_rng(0x7300 + seed)
    s = T.scenario(rng, 200, 30, p_role=(0.5, 0.2, 0.3, 0.0), p_select=1.0)
    frames_ = T.frames(rng, s, per_group=(1, 5))
    frames_ = [frames_[i] for i in rng.permutation(len(frames_))]
    # the pass, the host side of its bumps, the follower passes
    c, vt = Q.state_of(s)
    role, leader, table = s.role.copy(), s.leader.copy(), s.table.copy()
    blob, off = F.batch(frames_)
    st, out, rb, ro, _ = FT.batch(c, None, vt, blob, off, table)
    T.host_side(table, role, leader, st, out, frames_)
    ok = [i for i in range(len(frames_)) if st[i] >> 4 == B.WIRE_OK]
    final, resps = T.follower_passes(c, s, role, table, frames_, ok)
    # the literal form on the delivery order: heartbeats at T, appends at T, the stale frames, each in batch order
    typ = T.types_of(frames_)
    order = [i for i in ok if typ[i] == T.HEARTBEAT] + [i for i in ok if typ[i] == T.APPEND]
    order += [i for i in range(len(frames_)) if st[i] >> 4 == B.WIRE_STALE]
    assert len(order) == len(frames_)   # every frame passed the checks
    c1, vt1, role1, leader1, table1, verdict, resps1, stale1 = _literal_sequence(s, frames_, order)
    for name in ("term", "term_start", "committed", "last_index", "matched", "next_idx", "peer_committed", "pflags"):
        assert np.array_equal(getattr(c, name), getattr(c1, name)), name
    assert np.array_equal(vt, vt1) and np.array_equal(role, role1) and np.array_equal(leader, leader1)
    assert np.array_equal(table, table1)
    for i in range(len(frames_)):
        if st[i] >> 4 == B.WIRE_OK:
            assert verdict[i] == ("pass", final[i]), i
        else:
            assert verdict[i] == ("stale", bool(st[i] & B.RES_OK)), i
    assert sorted(resps) == resps1
    assert [rb[a:b].tobytes() for a, b in zip(ro[:-1], ro[1:])] == [x for x in stale1 if x]
    kinds = np.bincount(st >> 4, minlength=16)
    assert kinds[B.WIRE_OK] > 50 and kinds[B.WIRE_STALE] > 50 and np.count_nonzero(st & B.FTERM_BUMPED) > 20


def test_leaders_and_unselected_groups_are_the_hosts():
    rng = np.random.default_rng(0x7310)
    s = T.scenario(rng, 300, 20, p_role=(0.4, 0.1, 0.1, 0.4), p_select=0.7)
    frames_ = T.frames(rng, s)
    c, vt = Q.state_of(s)
    c0 = O.copy_columns(c)
    blob, off = F.batch(frames_)
    st, _, _, _, _ = FT.batch(c, None, vt, blob, off, s.table)
    g = np.array([int(np.frombuffer(f[:4], "<u4")[0]) >> 4 for f in frames_])
    host = (s.role[g] == Q.LEADER) | ((s.table["flags"][g] & B.VOTER_SELECT) == 0)
    assert host.sum() > 100 and np.all(st[host] == B.WIRE_ROLE << 4) and np.all(st[~host] >> 4 != B.WIRE_ROLE)
    hg = np.unique(g[host])
    for name in ("term", "term_start", "committed", "matched"):
        assert np.array_equal(getattr(c, name)[..., hg], getattr(c0, name)[..., hg]), name
