"""Vote requests for the voter-pass tests: the test encoder of MsgRequestVote / MsgRequestPreVote (proto3, fields in
number order, zero scalars and an empty context not written), the caller's voter table, and random voter scenarios --
configurations, roles, tables and batches of frames -- that run the same on the device arena and on the oracle."""
import numpy as np

from oracle import oracle as O
from oracle import control_oracle as CO
from oracle import vote_request_oracle as VR
from helpers import B
from control_cmds import cmds, META_WIDE_LO, META_WIDE_HI
import hb_frames as F

VOTE, PRE_VOTE = 5, 17
FOLLOWER, PRE_CANDIDATE, CANDIDATE, LEADER = range(4)
TRANSFER, ELECTION, PRE_ELECTION = b"CampaignTransfer", b"CampaignElection", b"CampaignPreElection"
NO_TERM_START = B.NO_TERM_START


def request(msg_type, term=0, log_term=0, index=0, commit=0, commit_term=0, priority=0, context=b"", to=0, frm=0) -> bytes:
    out = b""
    for no, v in ((1, msg_type), (2, to), (3, frm), (4, term), (5, log_term), (6, index), (8, commit)):
        if v:
            out += F.varint(no << 3) + F.varint(v)
    if context:
        out += F.varint(12 << 3 | 2) + F.varint(len(context)) + context
    for no, v in ((14, priority), (15, commit_term)):
        if v:
            out += F.varint(no << 3) + F.varint(v)
    return out


def voters(n) -> np.ndarray:
    return np.zeros(n, B.VOTER_DTYPE)


class Scenario:
    """n_narrow narrow groups [0, n_narrow) and n_wide wide pairs (low halves n_narrow, n_narrow + 2, ...), each a
    Follower, PreCandidate, Candidate or Leader at a random term, with joint configurations and learners.  setup is the
    control list that builds the arena; table is the caller's voter table (flags 0 on high halves); role, term, last and
    committed are per group slot (a pair's on both halves)."""

    def __init__(self, rng, n_narrow, n_wide, p_role=(0.5, 0.15, 0.2, 0.15), p_select=0.97):
        self.n_narrow, self.n_wide = n_narrow, n_wide
        self.n = n_narrow + 2 * n_wide
        self.lows = list(range(n_narrow)) + list(range(n_narrow, self.n, 2))
        self.wide = np.zeros(self.n, bool)
        self.wide[n_narrow:] = True
        self.role = np.zeros(self.n, np.uint8)
        self.term = np.zeros(self.n, np.uint64)
        self.last = np.zeros(self.n, np.uint64)
        self.committed = np.zeros(self.n, np.uint64)
        self.table = voters(self.n)
        setup = []
        for g in self.lows:
            wide = bool(self.wide[g])
            peers = 16 if wide else 8
            inc = int(rng.integers(1, 1 << peers)) if rng.random() < 0.5 else (0x1F if not wide else 0x1F01)
            out = int(rng.integers(0, 1 << peers)) if rng.random() < 0.25 else 0
            learn = int(rng.integers(0, 1 << peers)) & ~(inc | out) if rng.random() < 0.3 else 0
            s = int(rng.choice([p for p in range(peers) if inc >> p & 1]))
            li = int(rng.integers(5, 1 << 20))
            com = int(rng.integers(0, li + 1))
            term = int(rng.integers(2, 1 << 40)) if rng.random() < 0.9 else int(rng.integers(2, 200))
            role = int(rng.choice(4, p=p_role))
            halves = [g, g + 1] if wide else [g]
            self.role[halves], self.term[halves], self.last[halves], self.committed[halves] = role, term, li, com
            sid = s + 1
            setup.append((B.CTL_SET_CONF, g, s, 0, (inc, out, learn, li + 1)))
            setup.append((B.CTL_RESET, g, 0, 0, (NO_TERM_START, li, com, li)))
            setup.append((B.CTL_SET_TERM, g, 0, 0, (term,)))
            if role == LEADER:
                setup.append((B.CTL_RESET, g, 0, 0, (li + 1, li, com, li)))
                setup.append((B.CTL_BECOME_LEADER, g))
            t = self.table[g]
            t["id"], t["last_term"] = sid, max(1, term - int(rng.integers(0, 3)))
            t["commit_term"] = int(rng.integers(1, int(t["last_term"]) + 1)) if com else 0
            t["persisted"] = li - int(rng.integers(0, 3)) if li > 3 else li
            t["priority"] = int(rng.choice([0, 0, 1, 5]))
            if role in (PRE_CANDIDATE, CANDIDATE, LEADER):
                t["vote"] = sid if role != PRE_CANDIDATE or rng.random() < 0.5 else 0
            else:
                t["vote"] = int(rng.choice([0, 0, sid % 9 + 1, int(rng.integers(1, 10))]))
            leader = role == LEADER or (role == FOLLOWER and rng.random() < 0.5)
            flags = (B.VOTER_SELECT if role != LEADER and rng.random() < p_select else 0) | (B.VOTER_LEADER if leader else 0)
            if leader and rng.random() < 0.5:
                flags |= B.VOTER_LEASE
            t["flags"] = flags
        self.setup = cmds(*setup)

    def frames(self, rng, per_group=(1, 3), noise=True, commit_vote=True, only_decided=False):
        """Vote requests to every group: per_group[0]..per_group[1] each, at terms around the group's, logs around its
        log, from random candidates, some pre-votes, some in lease, some forced by CampaignTransfer.  With noise also
        other types, malformed and truncated frames, high halves and unallocated groups.  commit_vote: some carry
        commit > committed with commit_term.  only_decided: every frame reaches the term rules (selected, non-leader
        groups; m.term > 0; no COMMIT_VOTE)."""
        out = []
        for g in self.lows:
            if only_decided and (self.role[g] == LEADER or not (self.table[g]["flags"] & B.VOTER_SELECT)):
                continue
            term, li = int(self.term[g]), int(self.last[g])
            lt = int(self.table[g]["last_term"])
            for _ in range(int(rng.integers(per_group[0], per_group[1] + 1))):
                typ = PRE_VOTE if rng.random() < 0.4 else VOTE
                mt = max(1, term + int(rng.choice([-1, 0, 0, 1, 1, 2])))
                lg = max(0, lt + int(rng.choice([-1, 0, 0, 1])))
                ix = max(0, li + int(rng.choice([-1, 0, 0, 1])))
                c = ct = 0
                if rng.random() < 0.3:
                    c, ct = int(rng.integers(0, int(self.committed[g]) + 1)), int(rng.integers(0, 4))
                if commit_vote and not only_decided and rng.random() < 0.08:
                    c, ct = int(self.committed[g]) + 1 + int(rng.integers(0, 50)), int(rng.integers(1, 100))
                ctx = TRANSFER if rng.random() < 0.15 else (ELECTION if rng.random() < 0.3 else b"")
                body = request(typ, mt, lg, ix, c, ct, int(rng.choice([0, 0, 1, 5, 9])), ctx, to=int(self.table[g]["id"]),
                               frm=int(rng.integers(1, 10)))
                out.append(F.frame(g, int(rng.integers(16)), body))
            if not noise or rng.random() > 0.15:
                continue
            k = int(rng.integers(5))
            if k == 0:    # another message type
                out.append(F.frame(g, 0, request(int(rng.choice([6, 18, 8, 3])), term)))
            elif k == 1:  # garbage bytes
                out.append(F.frame(g, 0, rng.integers(0, 256, int(rng.integers(1, 12)), dtype=np.uint8).tobytes()))
            elif k == 2:  # a truncated frame
                out.append(F.frame(g, 0, request(VOTE, term + 1, 1, 1 << 40, context=TRANSFER))[:-3])
            elif k == 3:  # a wide pair's high half, or m.term 0
                h = g + 1 if self.wide[g] else g
                out.append(F.frame(h, 0, request(VOTE, 0 if h == g else term + 1, lt, li)))
            else:         # a group past the arena's highest slot
                out.append(F.frame(self.n + int(rng.integers(1, 100)), 0, request(VOTE, term + 1)))
        return out


def one(role, term, vote, last_index, last_term, leader=False, lease=False, check_quorum=False, voters=0b1,
         committed=None, commit_term=0, priority=0):
    """One group (slot 0 = self, id 1) in `role` at `term` with the given log -> (columns, votes, role, table)."""
    c = O.new_columns(8, 1)
    c.meta[0] = B.make_meta(voters, 0, 0, 0)
    c.term[0], c.last_index[0] = term, last_index
    c.committed[0] = last_index if committed is None else committed
    c.term_start[0] = last_index if role == LEADER else B.NO_TERM_START
    t = np.zeros(1, VR.VOTER_DTYPE)
    t["id"], t["vote"], t["last_term"], t["commit_term"], t["persisted"], t["priority"] = \
        1, vote, last_term, commit_term, last_index, priority
    t["flags"] = (VR.SELECT if role != LEADER else 0) | (VR.LEADER if leader else 0) | (VR.LEASE if lease else 0) | \
        (VR.CHECK_QUORUM if check_quorum else 0)
    return c, np.zeros((O.SLOTS, c.cap), np.uint8), np.array([role], np.uint8), t


# test_raft.rs:1537-1605: (role, index, log_term, vote, want reject) against a log of two entries at term 2
RECV_VOTE = [
    (FOLLOWER, 0, 0, 0, True), (FOLLOWER, 0, 1, 0, True), (FOLLOWER, 0, 2, 0, True), (FOLLOWER, 0, 3, 0, False),
    (FOLLOWER, 1, 0, 0, True), (FOLLOWER, 1, 1, 0, True), (FOLLOWER, 1, 2, 0, True), (FOLLOWER, 1, 3, 0, False),
    (FOLLOWER, 2, 0, 0, True), (FOLLOWER, 2, 1, 0, True), (FOLLOWER, 2, 2, 0, False), (FOLLOWER, 2, 3, 0, False),
    (FOLLOWER, 3, 0, 0, True), (FOLLOWER, 3, 1, 0, True), (FOLLOWER, 3, 2, 0, False), (FOLLOWER, 3, 3, 0, False),
    (FOLLOWER, 3, 2, 2, False), (FOLLOWER, 3, 2, 1, True), (LEADER, 3, 3, 1, True), (PRE_CANDIDATE, 3, 3, 1, True),
    (CANDIDATE, 3, 3, 1, True),
]


def recv_vote_case(row):
    role, index, log_term, vote, _ = row
    term = max(2, log_term)
    return one(role, term, vote, 2, 2), [F.frame(0, 0, request(VOTE, term, log_term, index, frm=2))]


# test_raft_paper.rs:962-1006: (log as (term, index) entries, m.log_term, m.index, want reject) at m.term 3
VOTER = [([(1, 1)], 1, 1, False), ([(1, 1)], 1, 2, False), ([(1, 1), (1, 2)], 1, 1, True),
         ([(1, 1)], 2, 1, False), ([(1, 1)], 2, 2, False), ([(1, 1), (1, 2)], 2, 1, False),
         ([(2, 1)], 1, 1, True), ([(2, 1)], 1, 2, True), ([(2, 1), (1, 2)], 1, 1, True)]


def voter_case(row):
    ents, log_term, index, _ = row
    # a new Raft at term 0 over that log (term 0 is the host's: the pass needs a known term, so the group sits at 1)
    state = one(FOLLOWER, 1, 0, len(ents), ents[-1][0], voters=0b11)
    return state, [F.frame(0, 0, request(VOTE, 3, log_term, index, frm=2))]


def any_state_case(role, typ):
    """test_raft.rs:655-760: three voters, term 1 (a Follower whose leader is 3, a PreCandidate), 2 (a Candidate or a
    Leader, who voted for themselves; the leader appended its empty entry); a request from 2 at term + 1."""
    term = 2 if role in (CANDIDATE, LEADER) else 1
    vote = 1 if role in (CANDIDATE, LEADER) else 0
    last = 1 if role == LEADER else 0
    state = one(role, term, vote, last, term if last else 0, leader=role in (FOLLOWER, LEADER), voters=0b111)
    return state, [F.frame(0, 0, request(typ, term + 1, term + 1, 42, frm=2))]


def state_of(s):
    c = O.new_columns(s.n + 8, s.n)
    c.term_start[:] = B.NO_TERM_START
    c.meta[s.n_narrow:s.n:2], c.meta[s.n_narrow + 1:s.n:2] = META_WIDE_LO, META_WIDE_HI   # the allocated pairs
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
            role[g] = FOLLOWER
        if status[i] & B.VREQ_VOTED:    # vote = m.from, election_elapsed = 0
            table["vote"][g] = out[i][0]
            if table["flags"][g] & VR.LEADER and table["flags"][g] & VR.CHECK_QUORUM:
                table["flags"][g] |= VR.LEASE
