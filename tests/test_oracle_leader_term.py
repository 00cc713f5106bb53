"""The leader term-prefix oracle (oracle/leader_term_oracle.c) on the CPU: the decoder on the golden frames of the six
types, the reference's term-rule cases at a leader on the literal form and the batch form, granting pre-vote responses
above the term, and on random batches the leader passes, the batch form and the follower passes against the literal
form in the reference's delivery order."""
import json
import os

import numpy as np
import pytest

from oracle import oracle as O
from oracle import follow_term_oracle as FT
from oracle import hb_wire_oracle as H
from oracle import leader_term_oracle as LT
from oracle import vote_request_oracle as VR
from helpers import B
import app_follow as A
import follow_term as T
import hb_frames as F
import leader_term as L
import vote_request_frames as Q

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "wire")


# --------------------------------------------------------------------------- 1. the decoder


def _golden_vectors():
    """(file, fields, hex) of every well-formed Message in the golden wire files: the fields as python-protobuf wrote
    them (a vector's own keys, or its "fields"), msg_type from the canonical first field where a file leaves it out."""
    for name in sorted(os.listdir(GOLDEN)):
        with open(os.path.join(GOLDEN, name), encoding="utf-8") as f:
            doc = json.load(f)
        for vs in doc.values():
            if not isinstance(vs, list):
                continue
            for v in vs:
                if not isinstance(v, dict) or "hex" not in v or v.get("ok") is False or v.get("parses") is False:
                    continue
                fields = dict(v.get("fields") or v)
                raw = bytes.fromhex(v["hex"])
                if "msg_type" not in fields and len(raw) >= 2 and raw[0] == 0x08 and raw[1] < 0x80:
                    fields["msg_type"] = raw[1]
                yield name, fields, raw


def test_golden_frames_of_the_six_types_decode():
    """Every frame of the six types in the golden wire files decodes to the fields python-protobuf wrote."""
    seen = set()
    for name, fields, raw in _golden_vectors():
        if fields.get("msg_type") not in L.TYPES:
            continue
        m = H.decode_message(raw)
        assert m is not None and m["msg_type"] == fields["msg_type"], (name, fields)
        for k in ("term", "from", "reject", "commit"):
            if k in fields and k in m:
                assert int(m[k]) == int(fields[k]), (name, k, fields)
        seen.add(fields["msg_type"])
    assert seen == set(L.TYPES), seen


# --------------------------------------------------------------------------- 2. the reference's cases


def _leader(term, stale_reply=False, last_index=10, voters=0b111, pid=1):
    """One Leader group (slot 0 = self, id pid) at `term` -> (columns, votes, role array, leader array, table)."""
    c, vt, r, t = Q.one(Q.LEADER, term, pid, last_index, max(1, term - 1), voters=voters)
    t["id"] = pid
    if stale_reply:
        t["flags"] |= FT.STALE_REPLY
    return c, vt, r, np.full(c.cap, pid, np.uint64), t


def _both(state, frames_):
    """The literal form and the batch form on copies of state -> ((outcome, replies, c, role, leader, table),
    (status, out, replies, c))."""
    c, vt, r, ld, t = state
    c1, v1, r1, l1, t1 = O.copy_columns(c), vt.copy(), r.copy(), ld.copy(), t.copy()
    blob, off = F.batch(frames_)
    outcome, rb, _, _ = LT.literal(c1, None, v1, r1, l1, t1, blob, off)
    c2, v2 = O.copy_columns(c), vt.copy()
    st, out, rb2, _, _ = LT.batch(c2, None, v2, blob, off, t)
    return (outcome, rb, c1, r1, l1, t1), (st, out, rb2, c2)


def _same_arena(c1, c2):
    for name in ("term", "term_start", "committed", "last_index", "matched", "next_idx", "peer_committed", "pflags"):
        assert np.array_equal(getattr(c1, name), getattr(c2, name)), name


def _body(typ, term, frm=2, reject=False):
    if typ == L.APPEND:
        return A.message(3, term, frm=frm)
    return F.message(typ, term, reject=reject, frm=frm)


@pytest.mark.parametrize("typ", L.TYPES)
def test_leader_update_term_from_message(typ):
    """test_leader_update_term_from_message (test_raft_paper.rs:57-100, the Leader row): a message at term 2 makes a
    leader at term 1 a Follower at term 2; leader_id = m.from for MsgAppend and MsgHeartbeat, none otherwise.  A
    granting pre-vote response is the exception (raft.rs:1319-1320)."""
    state = _leader(1)
    (outcome, _, c1, r1, l1, _), (st, out, _, c2) = _both(state, [F.frame(0, 1, _body(typ, 2, reject=True))])
    _same_arena(c1, c2)
    assert c1.term[0] == c2.term[0] == 2 and r1[0] == Q.FOLLOWER and c2.term_start[0] == B.NO_TERM_START
    lid = 2 if typ in (L.APPEND, L.HEARTBEAT) else 0
    assert l1[0] == lid and st.tolist() == [B.WIRE_OK << 4 | B.FTERM_BUMPED] and out.tolist() == [[lid, 2]]
    assert outcome.tolist() == [FT.PASS if typ in (L.APPEND, L.HEARTBEAT) else LT.IGNORED]


def test_all_server_stepdown_leader_append():
    """test_all_server_stepdown (test_raft.rs:1600-1660), the Leader row's MsgAppend leg: a leader at term 1 that
    receives MsgAppend at term 2 from n2 steps down, term 2, leader n2, vote cleared."""
    state = _leader(1)
    state[4]["vote"] = 1
    (outcome, _, c1, r1, l1, t1), (st, out, _, c2) = _both(state, [F.frame(0, 0, A.message(3, 2, frm=2))])
    _same_arena(c1, c2)
    assert (c1.term[0], r1[0], l1[0], t1["vote"][0]) == (2, Q.FOLLOWER, 2, 0) and outcome.tolist() == [FT.PASS]
    assert st.tolist() == [B.WIRE_OK << 4 | B.FTERM_BUMPED] and out.tolist() == [[2, 2]]


@pytest.mark.parametrize("stale_reply", [False, True])
def test_old_messages(stale_reply):
    """test_old_messages (test_raft.rs:1090-1120): a leader at term 3 drops a MsgAppend at term 2 -- and answers it
    with an empty MsgAppendResponse at term 3 when check_quorum or pre_vote is on."""
    state = _leader(3, stale_reply)
    (outcome, rb, c1, r1, _, _), (st, out, rb2, c2) = _both(state, [F.frame(0, 4, A.message(3, 2, frm=2))])
    _same_arena(c1, c2)
    assert c2.term[0] == 3 and c2.term_start[0] != B.NO_TERM_START and r1[0] == Q.LEADER and out.tolist() == [[0, 0]]
    assert rb.tobytes() == rb2.tobytes()
    if stale_reply:
        assert outcome.tolist() == [FT.ANSWERED] and st.tolist() == [B.WIRE_STALE << 4 | B.RES_OK]
        assert rb2.tobytes() == np.array([0 << 4 | 4], "<u4").tobytes() + FT.encode_reply(2, 1, 3)
    else:
        assert outcome.tolist() == [FT.DROPPED] and st.tolist() == [B.WIRE_STALE << 4] and len(rb2) == 0


@pytest.mark.parametrize("pre_vote", [False, True])
def test_disruptive_follower_steps_the_leader_down(pre_vote):
    """test_disruptive_follower (test_raft.rs:2088-2160): n1, leader at term 2, gets n3's MsgAppendResponse at term 3
    and steps down to a Follower at term 3 with no leader.  _pre_vote (:2162-2227): n3's pre-vote never raised its term,
    so n1 hears nothing above its own term and stays leader."""
    state = _leader(2, True, pid=1)
    body = F.message(4, 2 if pre_vote else 3, frm=3)
    (outcome, _, c1, r1, l1, _), (st, out, _, c2) = _both(state, [F.frame(0, 2, body)])
    _same_arena(c1, c2)
    if pre_vote:
        assert st.tolist() == [B.WIRE_OK << 4] and outcome.tolist() == [FT.PASS] and r1[0] == Q.LEADER
        assert c2.term[0] == 2 and c2.term_start[0] != B.NO_TERM_START
    else:
        assert st.tolist() == [B.WIRE_OK << 4 | B.FTERM_BUMPED] and out.tolist() == [[0, 3]]
        assert (c2.term[0], r1[0], l1[0]) == (3, Q.FOLLOWER, 0) and c2.term_start[0] == B.NO_TERM_START


def test_granted_pre_votes_above_the_term_do_not_raise_it():
    """A MsgRequestPreVoteResponse with reject = false is IGNORED at or above the leader's term and STALE below it;
    it is left out of T, so a rejecting one at the same term still claims."""
    state = _leader(5)
    fr = [F.frame(0, 1, F.message(18, 9, frm=2)), F.frame(0, 2, F.message(18, 5, frm=3)),
          F.frame(0, 3, F.message(18, 4, frm=4))]
    (outcome, _, c1, r1, _, _), (st, out, _, c2) = _both(state, fr)
    _same_arena(c1, c2)
    assert st.tolist() == [LT.WIRE_IGNORED << 4, LT.WIRE_IGNORED << 4, B.WIRE_STALE << 4]
    assert outcome.tolist() == [LT.IGNORED, LT.IGNORED, FT.DROPPED] and c2.term[0] == 5 and r1[0] == Q.LEADER
    fr.append(F.frame(0, 4, F.message(18, 7, reject=True, frm=5)))
    (_, _, c1, _, _, _), (st, out, _, c2) = _both(state, fr)
    _same_arena(c1, c2)
    assert st[:3].tolist() == [LT.WIRE_IGNORED << 4, LT.WIRE_IGNORED << 4, B.WIRE_STALE << 4]
    assert st[3] == B.WIRE_OK << 4 | B.FTERM_BUMPED and out[3].tolist() == [0, 7] and c2.term[0] == 7


def test_statuses_in_order():
    """Every status, first failing check first, the verdicts at the leader's term and at T, and the stale replies."""
    c = O.new_columns(16, 6)
    c.term_start[:] = B.NO_TERM_START
    c.meta[:6], c.term[:6], c.last_index[:6], c.committed[:6] = B.make_meta(0b111, 0, 0, 0), [5, 5, 5, 0, 5, 5], 10, 8
    c.meta[4], c.meta[5] = c.meta[4] | Q.META_WIDE_LO, c.meta[5] | Q.META_WIDE_HI
    c.term_start[[0, 2, 3, 4, 5]] = 9
    t = np.zeros(6, VR.VOTER_DTYPE)
    t["id"], t["flags"], t["persisted"] = 1, FT.STALE_REPLY, 10
    fr = [F.frame(99, 0, F.message(4, 6)), F.frame(0, 0, b"\x08"), F.frame(5, 0, F.message(8, 6, frm=2)),
          F.frame(0, 0, F.message(5, 6)), F.frame(1, 0, F.message(4, 6)), F.frame(3, 0, F.message(4, 6)),
          F.frame(0, 0, F.message(4, 0)),
          # group 0 at term 5: at the term, the claimant at 7, other frames at 7, stale frames
          F.frame(0, 1, F.message(4, 5)), F.frame(0, 2, F.message(8, 5, frm=2)), F.frame(0, 3, F.message(6, 5)),
          F.frame(0, 4, F.message(9, 7)), F.frame(0, 5, F.message(8, 7, frm=3)), F.frame(0, 6, F.message(18, 7, reject=True)),
          F.frame(0, 7, F.message(3, 6, frm=2)), F.frame(0, 8, F.message(9, 4)),
          # the pair 4-5 by its high half, at its term
          F.frame(5, 1, F.message(9, 5)), F.frame(5, 2, F.message(6, 5))]
    blob, off = F.batch(fr)
    st, out, rb, ro, tot = LT.batch(c, None, np.zeros((O.SLOTS, c.cap), np.uint8), blob, off, t)
    assert (st >> 4).tolist() == [B.WIRE_MALFORMED, B.WIRE_MALFORMED, B.WIRE_MALFORMED, B.WIRE_SKIP_TYPE,
                                  B.WIRE_ROLE, B.WIRE_TERM, B.WIRE_TERM,
                                  B.WIRE_OK, LT.WIRE_IGNORED, LT.WIRE_IGNORED, B.WIRE_OK, B.WIRE_OK, LT.WIRE_IGNORED,
                                  B.WIRE_STALE, B.WIRE_STALE, B.WIRE_OK, LT.WIRE_IGNORED]
    assert st[10] & 0xF == B.FTERM_BUMPED and out[10].tolist() == [0, 7] and st[11] & 0xF == 0
    assert st[13] & 0xF == B.RES_OK and st[14] & 0xF == 0 and c.term[0] == 7 and c.term[4] == 5
    assert tot.tolist() == [1, ro[-1]] and rb.tobytes() == fr[13][:4] + FT.encode_reply(2, 1, 7)


# --------------------------------------------------------------------------- 3. batch form vs literal form


def _state(s):
    c, vt = Q.state_of(s)
    return c, vt, s.role.copy(), s.leader.copy(), s.table.copy()


@pytest.mark.parametrize("seed", range(6))
def test_leader_passes_batch_then_follower_passes_equal_the_literal_form(seed):
    rng = np.random.default_rng(0x7400 + seed)
    s = L.scenario(rng, 200, 30)
    s.leader[:] = s.table["id"]
    frames_, meta = L.frames(rng, s)
    perm = rng.permutation(len(frames_))
    frames_, meta = [frames_[i] for i in perm], [meta[i] for i in perm]
    blob, off = F.batch(frames_)
    # the leader passes, this pass, the host side of its bumps, the follower passes
    c, vt, role, leader, table = _state(s)
    lst = L.leader_passes(c, frames_)
    st, out, rb, ro, _ = LT.batch(c, None, vt, blob, off, table)
    L.host_side(table, role, leader, st, out, meta)
    typ = T.types_of(frames_)
    follow = (typ == L.APPEND) | (typ == L.HEARTBEAT)
    ok = [i for i in range(len(frames_)) if st[i] >> 4 == B.WIRE_OK and follow[i]]
    final, resps = T.follower_passes(c, s, role, table, frames_, ok)
    # the reference: the leader passes take the frames at the term; then the literal form in the delivery order, the
    # MsgAppend / MsgHeartbeat it passes through the follower passes
    c1, vt1, role1, leader1, table1 = _state(s)
    lst1 = L.leader_passes(c1, frames_)
    assert np.array_equal(lst, lst1)
    order, _ = L.delivery_order(s, meta)
    assert sorted(order) == list(range(len(frames_)))
    verdict, replies, passed = {}, [], []
    for i in order:
        b1, o1 = F.batch([frames_[i]])
        outcome, r1, _, _ = LT.literal(c1, None, vt1, role1, leader1, table1, b1, o1)
        verdict[i] = int(outcome[0])
        replies.append((i, r1.tobytes()))
        if outcome[0] == FT.PASS and follow[i]:
            passed.append(i)
    table1["flags"][role1 == Q.FOLLOWER] |= B.VOTER_SELECT
    final1, resps1 = T.follower_passes(c1, s, role1, table1, frames_, passed)
    for name in ("term", "term_start", "committed", "last_index", "matched", "next_idx", "peer_committed", "pflags"):
        assert np.array_equal(getattr(c, name), getattr(c1, name)), name
    assert np.array_equal(vt, vt1) and np.array_equal(role, role1) and np.array_equal(leader, leader1)
    assert np.array_equal(table, table1)
    want = {B.WIRE_STALE << 4 | B.RES_OK: FT.ANSWERED, B.WIRE_STALE << 4: FT.DROPPED, LT.WIRE_IGNORED << 4: LT.IGNORED}
    for i in range(len(frames_)):
        k = int(st[i])
        if k >> 4 == B.WIRE_OK:
            exp = LT.IGNORED if (k & B.FTERM_BUMPED and not follow[i]) else FT.PASS
        else:
            exp = want[k]
        assert verdict[i] == exp, (i, k, meta[i])
    assert final == final1 and sorted(resps) == sorted(resps1)
    assert [rb[a:b].tobytes() for a, b in zip(ro[:-1], ro[1:])] == [r for _, r in sorted(replies) if r]
    kinds = np.bincount(st >> 4, minlength=16)
    assert kinds[B.WIRE_OK] > 50 and kinds[B.WIRE_STALE] > 50 and kinds[LT.WIRE_IGNORED] > 50
    assert np.count_nonzero(st & B.FTERM_BUMPED) > 20


def test_followers_are_the_hosts():
    """Frames to groups that are not leaders are ROLE and change nothing."""
    rng = np.random.default_rng(0x7410)
    s = T.scenario(rng, 300, 20, p_role=(0.4, 0.1, 0.1, 0.4))
    frames_, meta = L.frames(rng, s)
    c, vt = Q.state_of(s)
    c0 = O.copy_columns(c)
    blob, off = F.batch(frames_)
    st, _, _, _, _ = LT.batch(c, None, vt, blob, off, s.table)
    host = np.array([s.role[m[0]] != Q.LEADER for m in meta])
    assert host.sum() > 100 and np.all(st[host] == B.WIRE_ROLE << 4) and np.all(st[~host] >> 4 != B.WIRE_ROLE)
    hg = np.unique([m[0] for m, h in zip(meta, host) if h])
    for name in ("term", "term_start", "committed", "matched"):
        assert np.array_equal(getattr(c, name)[..., hg], getattr(c0, name)[..., hg]), name
