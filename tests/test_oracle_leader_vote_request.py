"""The leader vote-request oracle (oracle/leader_vote_request_oracle.c) on the CPU: the reference's cases at a leader
on the batch form against the literal form (vro_literal), every status in check order, the claimant rule, random
bursts through the resubmission loop against the literal form, and one received buffer through the leader's term pass
and then this pass against the literal forms in the documented order."""
import numpy as np
import pytest

from oracle import oracle as O
from oracle import hb_wire_oracle as H
from oracle import leader_term_oracle as LT
from oracle import leader_vote_request_oracle as LV
from oracle import vote_request_oracle as VR
from helpers import B
import follow_term as T
import hb_frames as F
import leader_term as L
import leader_vote_request as LQ
import vote_request_frames as Q

ARENA = ("term", "term_start", "committed", "last_index", "matched", "next_idx", "peer_committed", "pflags")


def _copy(state):
    c, vt, r, t = state
    return O.copy_columns(c), vt.copy(), r.copy(), t.copy()


def _decoded(blob, off):
    return [H.decode_message(blob[off[k] + 4:off[k + 1]].tobytes()) for k in range(len(off) - 1)]


def _both(state, frames_):
    """The literal form and the batch form with its host side on copies of state -> ((responses, c, role, table),
    (status, out, responses, c, role, table)); responses as raw bytes."""
    blob, off = F.batch(frames_)
    c1, v1, r1, t1 = _copy(state)
    rb1, ro1, _ = VR.literal(c1, None, v1, r1, t1, blob, off)
    t1["flags"][r1 == Q.FOLLOWER] |= B.VOTER_SELECT   # the caller's selection of a deposed leader
    c2, v2, r2, t2 = _copy(state)
    st, out, rb2, ro2, _ = LV.batch(c2, None, v2, blob, off, t2)
    LQ.host_side(t2, r2, st, out, frames_)
    return (_split(rb1, ro1), c1, r1, t1, v1), (st, out, _split(rb2, ro2), c2, r2, t2, v2)


def _split(blob, off):
    return [blob[a:b].tobytes() for a, b in zip(off[:-1].tolist(), off[1:].tolist())]


def _same(c1, c2):
    for name in ARENA:
        assert np.array_equal(getattr(c1, name), getattr(c2, name)), name


# --------------------------------------------------------------------------- 1. the reference's cases at a leader


@pytest.mark.parametrize("typ", [Q.VOTE, Q.PRE_VOTE], ids=["vote", "prevote"])
def test_vote_from_any_state_leader_row(typ):
    """test_vote_from_any_state / test_prevote_from_any_state (test_raft.rs:655-760), the Leader row: a leader at term
    2 gets n2's request at term 3.  A vote deposes it -- a Follower at term 3 that voted for 2; a pre-vote is granted
    with nothing changed."""
    state, frames_ = Q.any_state_case(Q.LEADER, typ)
    (r1, c1, role1, t1, v1), (st, out, r2, c2, role2, t2, v2) = _both(state, frames_)
    assert r1 == r2 and len(r2) == 1 and not H.decode_message(r2[0][4:])["reject"]
    _same(c1, c2)
    assert np.array_equal(role1, role2) and np.array_equal(t1, t2) and np.array_equal(v1, v2)
    if typ == Q.VOTE:
        assert st.tolist() == [B.WIRE_OK << 4 | B.VREQ_GRANTED | B.VREQ_VOTED | B.VREQ_BUMPED]
        assert (role2[0], c2.term[0], t2["vote"][0], c2.term_start[0]) == (Q.FOLLOWER, 3, 2, B.NO_TERM_START)
        assert out.tolist() == [[2, 3]]
    else:
        assert st.tolist() == [B.WIRE_OK << 4 | B.VREQ_GRANTED] and out.tolist() == [[2, 2]]
        assert (role2[0], c2.term[0], t2["vote"][0]) == (Q.LEADER, 2, 1) and c2.term_start[0] != B.NO_TERM_START
        assert H.decode_message(r2[0][4:])["term"] == 3   # a grant answers at m.term


@pytest.mark.parametrize("row", [k for k, r in enumerate(Q.RECV_VOTE) if r[0] == Q.LEADER])
def test_recv_msg_request_vote_leader_rows(row):
    """test_recv_msg_request_vote (test_raft.rs:1537-1605), the Leader rows: a request at the leader's term is
    rejected with its commit info, and nothing changes."""
    state, frames_ = Q.recv_vote_case(Q.RECV_VOTE[row])
    (r1, c1, role1, t1, _), (st, out, r2, c2, role2, t2, _) = _both(state, frames_)
    assert r1 == r2 and len(r2) == 1 and H.decode_message(r2[0][4:])["reject"] == Q.RECV_VOTE[row][4]
    assert st.tolist() == [B.WIRE_OK << 4] and out.tolist() == [[2, int(c2.term[0])]]
    _same(c1, c2)
    assert np.array_equal(role1, role2) and np.array_equal(t1, t2) and role2[0] == Q.LEADER


@pytest.mark.parametrize("typ", [Q.VOTE, Q.PRE_VOTE], ids=["vote", "prevote"])
@pytest.mark.parametrize("ctx", [b"", Q.ELECTION, Q.TRANSFER], ids=["none", "election", "transfer"])
def test_lease_at_a_leader(typ, ctx):
    """test_leader_election_with_check_quorum / test_leader_superseding_with_check_quorum (test_raft.rs:1886-2000): a
    leader in lease drops a higher-term request; test_leader_transfer_receive_higher_term_vote (:3568): a
    CampaignTransfer request goes through the lease, and a vote deposes the leader."""
    state = Q.one(Q.LEADER, 2, 1, 1, 2, leader=True, lease=True, check_quorum=True, voters=0b111)
    frames_ = [F.frame(0, 0, Q.request(typ, 3, 2, 1, context=ctx, frm=3))]
    (r1, c1, role1, t1, _), (st, out, r2, c2, role2, t2, _) = _both(state, frames_)
    assert r1 == r2
    _same(c1, c2)
    assert np.array_equal(role1, role2) and np.array_equal(t1, t2)
    if ctx != Q.TRANSFER:
        assert st.tolist() == [VR.WIRE_IGNORED << 4] and r2 == [] and c2.term[0] == 2 and role2[0] == Q.LEADER
    elif typ == Q.VOTE:
        assert st.tolist() == [B.WIRE_OK << 4 | B.VREQ_GRANTED | B.VREQ_VOTED | B.VREQ_BUMPED]
        assert (role2[0], c2.term[0], t2["vote"][0]) == (Q.FOLLOWER, 3, 3)
        assert t2["flags"][0] & (VR.LEADER | VR.LEASE) == 0
    else:
        assert st.tolist() == [B.WIRE_OK << 4 | B.VREQ_GRANTED] and role2[0] == Q.LEADER and c2.term[0] == 2


def test_statuses_in_order():
    """Every status at the first check that fails, the decisions before a claimant, the claimant and what follows it."""
    c = O.new_columns(16, 8)
    c.term_start[:] = B.NO_TERM_START
    c.meta[:8], c.term[:8], c.last_index[:8], c.committed[:8] = B.make_meta(0b111, 0, 0, 0), 5, 10, 8
    c.term[3] = 0
    c.term_start[[0, 2, 3, 4, 5]] = 9
    c.meta[6], c.meta[7] = c.meta[6] | Q.META_WIDE_LO, c.meta[7] | Q.META_WIDE_HI
    c.term_start[6] = 9
    t = np.zeros(8, VR.VOTER_DTYPE)
    t["id"], t["vote"], t["last_term"], t["commit_term"], t["persisted"] = 1, 1, 4, 3, 10
    t["flags"] = VR.LEADER
    t["flags"][1] = VR.SELECT | VR.LEADER   # a follower, selected: ROLE here all the same
    t["flags"][5] = VR.LEADER | VR.LEASE
    fr = [F.frame(99, 0, Q.request(Q.VOTE, 6)),                              # MALFORMED: past the arena
          F.frame(0, 0, b"\x08"),                                           # MALFORMED: truncated
          F.frame(7, 0, Q.request(Q.VOTE, 6)),                              # MALFORMED: a pair's high half
          F.frame(0, 0, Q.request(6, 6)),                                   # SKIP_TYPE
          F.frame(1, 0, Q.request(Q.VOTE, 6)),                              # ROLE: not a leader
          F.frame(3, 0, Q.request(Q.VOTE, 6)),                              # TERM: unknown term
          F.frame(0, 0, Q.request(Q.VOTE, 0)),                              # TERM: a local message
          # group 0 at term 5: before its claimant, the claimant, after it
          F.frame(0, 1, Q.request(Q.VOTE, 4, frm=2)),                       # IGNORED: lower-term vote
          F.frame(0, 2, Q.request(Q.PRE_VOTE, 4, frm=2)),                   # OK: rejected at 5, no commit fields
          F.frame(0, 3, Q.request(Q.VOTE, 5, 4, 10, 9, 4, frm=2)),          # OK: at the term, rejected (no COMMIT_VOTE)
          F.frame(0, 4, Q.request(Q.PRE_VOTE, 6, 4, 10, frm=3)),            # OK: granted at 6, the term stays
          F.frame(0, 5, Q.request(Q.PRE_VOTE, 6, 3, 10, 9, 4, frm=3)),      # OK: rejected at 5 (no COMMIT_VOTE)
          F.frame(0, 6, Q.request(Q.VOTE, 7, 4, 10, frm=4)),                # OK: the claimant, bumped and granted
          F.frame(0, 7, Q.request(Q.PRE_VOTE, 4, frm=2)),                   # DUP
          # group 2: a claimant rejected with the commit ahead; group 4: a grant at the term; group 5: in lease
          F.frame(2, 0, Q.request(Q.VOTE, 6, 3, 10, 9, 4, frm=2)),          # COMMIT_VOTE
          F.frame(2, 1, Q.request(Q.VOTE, 4, frm=2)),                       # DUP
          F.frame(4, 0, Q.request(Q.VOTE, 5, 4, 10, frm=1)),                # OK: granted at the term, VOTED
          F.frame(4, 1, Q.request(Q.VOTE, 6, 4, 10, frm=2)),                # DUP
          F.frame(5, 0, Q.request(Q.VOTE, 6, 4, 10, frm=2)),                # IGNORED: lease
          F.frame(5, 1, Q.request(Q.VOTE, 6, 4, 10, context=Q.TRANSFER, frm=2)),  # OK: forced, bumped
          # the pair 6-7 by its low half: a bump resets both halves
          F.frame(6, 0, Q.request(Q.VOTE, 8, 4, 10, frm=2))]
    blob, off = F.batch(fr)
    st, out, rb, ro, tot = LV.batch(c, None, np.zeros((O.SLOTS, c.cap), np.uint8), blob, off, t)
    W = B
    assert (st >> 4).tolist() == [W.WIRE_MALFORMED] * 3 + [W.WIRE_SKIP_TYPE, W.WIRE_ROLE, W.WIRE_TERM, W.WIRE_TERM,
                                                           VR.WIRE_IGNORED, W.WIRE_OK, W.WIRE_OK, W.WIRE_OK, W.WIRE_OK,
                                                           W.WIRE_OK, W.WIRE_DUP, VR.WIRE_COMMIT_VOTE, W.WIRE_DUP,
                                                           W.WIRE_OK, W.WIRE_DUP, VR.WIRE_IGNORED, W.WIRE_OK, W.WIRE_OK]
    low = (st & 0xF).tolist()
    assert low[8:13] == [0, 0, B.VREQ_GRANTED, 0, B.VREQ_GRANTED | B.VREQ_VOTED | B.VREQ_BUMPED]
    assert low[16] == B.VREQ_GRANTED | B.VREQ_VOTED and low[19] & B.VREQ_BUMPED and low[20] & B.VREQ_BUMPED
    assert out[8:13].tolist() == [[2, 5], [2, 5], [3, 5], [3, 5], [4, 7]] and out[16].tolist() == [1, 5]
    assert not out[13:16].any() and not out[17:19].any()
    assert c.term[:8].tolist() == [7, 5, 5, 0, 5, 6, 8, 8] and c.term_start[6] == c.term_start[7] == B.NO_TERM_START
    assert c.term_start[[2, 4]].tolist() == [9, 9] and tot[0] == 8
    r = _decoded(rb, ro)
    assert [(m["msg_type"], m["term"], bool(m["reject"]), m["commit"]) for m in r[:5]] == \
        [(18, 5, True, 0), (6, 5, True, 8), (18, 6, False, 0), (18, 5, True, 8), (6, 7, False, 0)]


# --------------------------------------------------------------------------- 2. the resubmission loop is exact


@pytest.mark.parametrize("seed", range(8))
def test_resubmission_loop_equals_the_literal_form(seed):
    """Random bursts of 1-4 vote requests per leader (both types; terms below, at and above; in and out of lease;
    transfer contexts; commit ahead; m.from the leader's own vote; wide pairs): this pass, its host side, the host's
    step of COMMIT_VOTE frames and raftgpu_vote_request_wire on the frames of deposed groups, until no frame is left,
    reach the literal form's state and per-group responses."""
    rng = np.random.default_rng(0x7500 + seed)
    s = LQ.scenario(rng, 300, 40)
    frames_ = s.frames(rng, per_group=(1, 4), noise=False)
    frames_ = [frames_[i] for i in rng.permutation(len(frames_))]
    c1, v1 = Q.state_of(s)
    t1, r1 = s.table.copy(), s.role.copy()
    want = LQ.literal(c1, None, v1, r1, t1, frames_)
    c2, v2 = Q.state_of(s)
    t2, r2 = s.table.copy(), s.role.copy()
    got, rounds, kinds = LQ.settle(c2, None, v2, r2, t2, frames_, *LQ.oracle_passes(c2, None, v2))
    assert rounds > 1 and got == want
    _same(c1, c2)
    assert np.array_equal(v1, v2) and np.array_equal(r1, r2) and np.array_equal(t1["vote"], t2["vote"])
    t1["flags"][r1 == Q.FOLLOWER] |= B.VOTER_SELECT    # the host side's selection of a deposed leader
    assert np.array_equal(t1["flags"], t2["flags"])
    lead = kinds[0]
    for k in (B.WIRE_OK, B.WIRE_DUP, B.WIRE_ROLE, B.WIRE_COMMIT_VOTE, VR.WIRE_IGNORED):
        assert lead[k] > 0, (k, lead)
    assert kinds[1][B.WIRE_ROLE] == 0


def test_claimants_are_the_only_frames_that_change_state():
    """Per group, the frames before the claimant read the state the batch started from: deciding each of them alone
    on a fresh copy gives the same status and response."""
    rng = np.random.default_rng(0x7510)
    s = LQ.scenario(rng, 400, 0)
    frames_ = s.frames(rng, per_group=(2, 4), noise=False)
    c, v = Q.state_of(s)
    blob, off = F.batch(frames_)
    st, out, rb, ro, _ = LV.batch(c, None, v, blob, off, s.table)
    resp = iter(_split(rb, ro))
    checked = 0
    for i, fr in enumerate(frames_):
        k = int(st[i]) >> 4
        if k == B.WIRE_DUP:
            continue
        c1, v1 = Q.state_of(s)
        st1, out1, rb1, _, _ = LV.batch(c1, None, v1, *F.batch([fr]), s.table)
        assert st1[0] == st[i] and np.array_equal(out1[0], out[i]), i
        assert rb1.tobytes() == (next(resp) if k == B.WIRE_OK else b""), i
        checked += 1
    assert checked > 400 and np.count_nonzero(st >> 4 == B.WIRE_DUP) > 50


# --------------------------------------------------------------------------- 3. one buffer after the leader's term pass


@pytest.mark.parametrize("seed", range(4))
def test_after_the_leader_term_pass_equals_the_literal_forms(seed):
    """One received buffer of the six types raftgpu_leader_term_wire takes and of vote requests, at leaders: the
    leader passes, raftgpu_leader_term_wire and its host side, the follower passes, then this pass's resubmission
    loop -- against the reference's order: the literal leader-term form in its delivery order with the follower
    passes, then the literal vote-request form over the vote requests in frame order."""
    rng = np.random.default_rng(0x7520 + seed)
    s = L.scenario(rng, 200, 30)
    s.leader[:] = s.table["id"]
    lt_frames, meta = L.frames(rng, s, per_group=(0, 4))
    vr_frames = s.frames(rng, per_group=(1, 3), noise=False)
    tag = [("lt", k) for k in range(len(lt_frames))] + [("vr", k) for k in range(len(vr_frames))]
    tag = [tag[i] for i in rng.permutation(len(tag))]
    frames_ = [lt_frames[k] if w == "lt" else vr_frames[k] for w, k in tag]
    lt_at = [i for i, (w, _) in enumerate(tag) if w == "lt"]
    vr_at = [i for i, (w, _) in enumerate(tag) if w == "vr"]
    lt_meta = [meta[tag[i][1]] for i in lt_at]
    # the passes in the documented order, on one buffer
    c, vt = Q.state_of(s)
    role, leader, table = s.role.copy(), s.leader.copy(), s.table.copy()
    L.leader_passes(c, frames_)
    blob, off = F.batch(frames_)
    st, out, _, _, _ = LT.batch(c, None, vt, blob, off, table)
    assert np.all(st[vr_at] == B.WIRE_SKIP_TYPE << 4)
    L.host_side(table, role, leader, st[lt_at], out[lt_at], lt_meta)
    typ = T.types_of(frames_)
    ok = [i for i in lt_at if st[i] >> 4 == B.WIRE_OK and typ[i] in (L.APPEND, L.HEARTBEAT)]
    final, _ = T.follower_passes(c, s, role, table, frames_, ok)
    got, _, kinds = LQ.settle(c, None, vt, role, table, [frames_[i] for i in vr_at], *LQ.oracle_passes(c, None, vt))
    # the reference
    c1, vt1 = Q.state_of(s)
    role1, leader1, table1 = s.role.copy(), s.leader.copy(), s.table.copy()
    L.leader_passes(c1, frames_)
    sub = [frames_[i] for i in lt_at]
    order, _ = L.delivery_order(s, lt_meta)
    passed = []
    for j in order:
        outcome, _, _, _ = LT.literal(c1, None, vt1, role1, leader1, table1, *F.batch([sub[j]]))
        if outcome[0] == LT.FT.PASS and sub[j][5] in (L.APPEND, L.HEARTBEAT):
            passed.append(j)
    table1["flags"][role1 == Q.FOLLOWER] |= B.VOTER_SELECT
    final1, _ = T.follower_passes(c1, s, role1, table1, sub, passed)
    want = LQ.literal(c1, None, vt1, role1, table1, [frames_[i] for i in vr_at])
    assert got == want
    _same(c, c1)
    assert np.array_equal(vt, vt1) and np.array_equal(role, role1)
    table1["flags"][role1 == Q.FOLLOWER] |= B.VOTER_SELECT
    assert np.array_equal(table, table1)
    assert kinds[0][B.WIRE_ROLE] > 20 and kinds[0][B.WIRE_OK] > 20 and np.count_nonzero(role == Q.FOLLOWER) > 20
