"""Followers and candidates for the tests of the responses that reach them (raftgpu_follower_response_wire,
oracle/follow_resp_oracle.c) and of the candidate's step-down in raftgpu_follower_term_wire: random groups in every
role with the caller's voter table and its candidate flags, the bursts that follow a deposition or an election, the
caller's host side of a bump or a step-down, and the reference's delivery order."""
import numpy as np

from helpers import B
from oracle import follow_term_oracle as FT
from oracle import leader_term_oracle as LT
from oracle import vote_request_oracle as VR
import follow_term as T
import hb_frames as F
import pass_forms as PF
import vote_request_frames as Q

APP_RESP, VOTE_RESP, HB_RESP, PRE_VOTE_RESP = 4, 6, 9, 18
TYPES = (APP_RESP, VOTE_RESP, HB_RESP, PRE_VOTE_RESP)
FOLLOWER_TYPES = (3, 8)

# the device form in pass_forms' table: the voter table in, status u8[n] and out u64[n] back, no replies
PF.PASSES.setdefault("follower_response_wire", PF._frame_pass(PF.VOTERS, PF.ST + (("out", np.uint64, ()),)))


def candidate_flags(role):
    """RAFTGPU_VOTER_CANDIDATE / _PRE_CANDIDATE for a role."""
    return {Q.PRE_CANDIDATE: B.VOTER_CANDIDATE | B.VOTER_PRE_CANDIDATE, Q.CANDIDATE: B.VOTER_CANDIDATE}.get(int(role), 0)


def scenario(rng, n_narrow, n_wide, p_role=(0.4, 0.2, 0.3, 0.1), p_select=0.95, p_reply=0.5):
    """T.scenario's groups, table and setup, with the candidate flags of every (Pre)Candidate set."""
    s = T.scenario(rng, n_narrow, n_wide, p_role=p_role, p_select=p_select, p_reply=p_reply)
    for g in s.lows:
        s.table["flags"][g] |= candidate_flags(s.role[g])
    return s


def frames(rng, s, per_group=(1, 5), deltas=(-2, -1, 0, 0, 0, 1, 1, 3), types=TYPES):
    """Responses of the four types to every group at its term + one of deltas (at least 1) -- a deposed leader's late
    append and heartbeat responses, late votes, rejections at a higher term -- addressed to a cell (a pair's high half
    for a share of them) -> (frames, meta), meta per frame = (low half, type, m.term, reject)."""
    out, meta = [], []
    for g in s.lows:
        term, last, com = int(s.term[g]), int(s.last[g]), int(s.committed[g])
        for _ in range(int(rng.integers(per_group[0], per_group[1] + 1))):
            t = max(1, term + int(rng.choice(deltas)))
            typ = int(rng.choice(types))
            h = g + 1 if s.wide[g] and rng.random() < 0.3 else g
            slot = int(rng.integers(1, 8))
            reject = bool(rng.random() < 0.5) if typ in (VOTE_RESP, PRE_VOTE_RESP) else False
            body = F.message(typ, t, reject=reject, commit=int(rng.integers(0, com + 1)) if typ == HB_RESP else 0,
                             index=int(rng.integers(0, last + 1)) if typ == APP_RESP else 0, frm=slot + 1)
            out.append(F.frame(h, slot, body))
            meta.append((g, typ, t, reject))
    return out, meta


def host_side(table, role, leader, status, out_t, groups):
    """become_follower(T, INVALID_ID)'s host side for every RAFTGPU_FTERM_BUMPED frame of this pass: a Follower with no
    leader, no vote, no candidacy, selected for the follower passes."""
    for i in np.flatnonzero((status >> 4 == B.WIRE_OK) & ((status & B.FTERM_BUMPED) != 0)):
        g = groups[i]
        role[g], leader[g], table["vote"][g] = Q.FOLLOWER, 0, 0
        table["flags"][g] &= ~np.uint32(VR.LEADER | VR.LEASE | B.VOTER_CANDIDATE | B.VOTER_PRE_CANDIDATE)
        table["flags"][g] |= B.VOTER_SELECT


def term_host_side(table, role, leader, status, out, frames_):
    """raftgpu_follower_term_wire's host side: become_follower(T, m.from) for a BUMPED frame (vote 0), and
    become_follower(term, m.from) for a STEPPED one (the vote kept); either way no candidacy and the follower select."""
    for i in np.flatnonzero((status >> 4 == B.WIRE_OK) & ((status & (B.FTERM_BUMPED | B.FTERM_STEPPED)) != 0)):
        g = int(np.frombuffer(frames_[i][:4], "<u4")[0]) >> 4
        role[g], leader[g] = Q.FOLLOWER, out[i][0]
        if status[i] & B.FTERM_BUMPED:
            table["vote"][g] = 0
        table["flags"][g] &= ~np.uint32(VR.LEADER | VR.LEASE | B.VOTER_CANDIDATE | B.VOTER_PRE_CANDIDATE)
        table["flags"][g] |= B.VOTER_SELECT | (VR.LEADER if out[i][0] else 0)


def delivery_order(s, meta):
    """The reference's order for the batch: each group's claimant, the other frames at T, then the stale frames, each
    in batch order -> order.  T leaves the granting pre-vote responses out."""
    top = {}
    for g, typ, t, rej in meta:
        top[g] = max(top.get(g, int(s.term[g])), int(s.term[g]) if typ == PRE_VOTE_RESP and not rej else t)
    grant = {i for i, (g, typ, t, rej) in enumerate(meta) if typ == PRE_VOTE_RESP and not rej}
    claim = {}
    for i, (g, typ, t, rej) in enumerate(meta):
        if i not in grant and t == top[g] and t > int(s.term[g]):
            claim.setdefault(g, i)
    claimants = sorted(claim.values())
    at_top = [i for i, (g, typ, t, rej) in enumerate(meta) if t >= top[g] and i not in claimants]
    stale = [i for i, (g, typ, t, rej) in enumerate(meta) if t < top[g]]
    return claimants + at_top + stale


def outcome_of(status):
    """The literal form's outcome a batch status stands for: the claimant is bumped and then dropped by step_follower,
    OK reaches step_candidate's poll, IGNORED and STALE are dropped."""
    k = int(status)
    if k >> 4 == B.WIRE_OK:
        return LT.IGNORED if k & B.FTERM_BUMPED else FT.PASS
    return {B.WIRE_IGNORED: LT.IGNORED, B.WIRE_STALE: FT.DROPPED}[k >> 4]
