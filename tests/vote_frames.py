"""Vote responses for the vote-pass tests: the test encoder of MsgRequestVoteResponse / MsgRequestPreVoteResponse
(proto3, fields in number order, zero scalars not written), and random elections -- configurations, the campaign lists
of INTEGRATION.md section 6, and batches of frames -- that run the same on the device arena and on the oracle."""
import numpy as np

from oracle import oracle as O
from oracle import control_oracle as CO
from oracle import vote_wire_oracle as VW
from helpers import B
from control_cmds import cmds, META_WIDE_LO, META_WIDE_HI  # noqa: F401
import hb_frames as F

VOTE_RESPONSE, PRE_VOTE_RESPONSE = 6, 18
FOLLOWER, PRE_CANDIDATE, CANDIDATE, LEADER = range(4)
NO_TERM_START = B.NO_TERM_START


def message(msg_type, term=0, reject=False, commit=0, commit_term=0, to=0, frm=0) -> bytes:
    out = b""
    for no, v in ((1, msg_type), (2, to), (3, frm), (4, term), (8, commit), (10, int(reject)), (15, commit_term)):
        if v:
            out += F.varint(no << 3) + F.varint(v)
    return out


def bitmap(bits) -> np.ndarray:
    """u32 words from group 0 of a bool per group slot (padded to whole words, at least one)."""
    bits = np.asarray(bits, dtype=bool)
    pad = np.zeros((-len(bits)) % 32 or (32 if len(bits) == 0 else 0), dtype=bool)
    return np.packbits(np.concatenate([bits, pad]), bitorder="little").view(np.uint32).copy()


class Election:
    """n_narrow narrow groups [0, n_narrow) and n_wide wide pairs (low halves n_narrow, n_narrow + 2, ...), each a
    Follower, a Leader, a PreCandidate or a Candidate at a random term.  Every group's self slot is an incoming voter and
    its configuration has at least two voters in each half of a joint configuration, so the self vote alone decides
    nothing.  setup (SET_CONF, RESET, SET_TERM, BECOME_LEADER) and campaign (section 6 step 1) are control lists; role
    and term are per group slot (a pair's on both halves)."""

    def __init__(self, rng, n_narrow, n_wide, p_role=(0.1, 0.1, 0.4, 0.4)):
        self.n_narrow, self.n_wide = n_narrow, n_wide
        self.n = n_narrow + 2 * n_wide
        self.lows = list(range(n_narrow)) + list(range(n_narrow, self.n, 2))
        self.wide = np.zeros(self.n, bool)
        self.wide[n_narrow:] = True
        self.role = np.zeros(self.n, np.uint8)
        self.term = np.zeros(self.n, np.uint64)
        self.last = np.zeros(self.n, np.uint64)
        self.committed = np.zeros(self.n, np.uint64)
        self.self_slot = np.zeros(self.n, np.int64)
        self.present = np.zeros(self.n, np.uint32)
        setup, camp = [], []
        for g in self.lows:
            wide = bool(self.wide[g])
            peers = 16 if wide else 8
            while True:
                inc = int(rng.integers(0, 1 << peers)) if rng.random() < 0.5 else (0x1F if not wide else 0x1F01)
                out = int(rng.integers(0, 1 << peers)) if rng.random() < 0.25 else 0
                if bin(inc).count("1") >= 2 and (out == 0 or bin(out).count("1") >= 2):
                    break
            learn = int(rng.integers(0, 1 << peers)) & ~(inc | out) if rng.random() < 0.3 else 0
            s = int(rng.choice([p for p in range(peers) if inc >> p & 1]))
            li = int(rng.integers(5, 1 << 20))
            com = int(rng.integers(0, li + 1))
            term = int(rng.integers(1, 1 << 40)) if rng.random() < 0.9 else int(rng.integers(1, 200))
            role = int(rng.choice(4, p=p_role))
            halves = [g, g + 1] if wide else [g]
            self.role[halves], self.term[halves], self.last[halves] = role, term, li
            self.committed[halves], self.self_slot[halves], self.present[halves] = com, s, inc | out | learn
            setup.append((B.CTL_SET_CONF, g, s, 0, (inc, out, learn, li + 1)))
            setup.append((B.CTL_RESET, g, 0, 0, (NO_TERM_START, li, com, li)))
            setup.append((B.CTL_SET_TERM, g, 0, 0, (term,)))
            if role == LEADER:
                setup.append((B.CTL_RESET, g, 0, 0, (li + 1, li, com, li)))
                setup.append((B.CTL_BECOME_LEADER, g))
            elif role == CANDIDATE:  # become_candidate: reset(term + 1) (raft.rs:1101-1122)
                self.term[halves] = term + 1
                camp.append((B.CTL_RESET, g, 0, 0, (NO_TERM_START, li, com, li)))
                camp.append((B.CTL_SET_TERM, g, 0, 0, (term + 1,)))
            if role in (PRE_CANDIDATE, CANDIDATE):  # reset_votes, then poll(self.id, true) (raft.rs:1124-1138, 1233-1278)
                camp.append((B.CTL_RESET_VOTES, g))
                camp.append((B.CTL_RECORD_VOTE, g, s, 1))
                camp.append((B.CTL_VOTE_RESULT, g))
        self.setup, self.campaign = cmds(*setup), cmds(*camp)

    def select(self):
        return bitmap(np.isin(self.role, (PRE_CANDIDATE, CANDIDATE)))

    def pre(self):
        return bitmap(self.role == PRE_CANDIDATE)

    def frames(self, rng, noise=True, commit_vote=False):
        """One response per present non-self peer of every candidate (some missing), in the candidate's own type at a
        term it polls at; with noise also repeats of a cell, the other response type, stale terms, frames to
        followers and leaders, other message types, peers past the group's slots and malformed frames -- none of which
        changes anything in either form.  commit_vote: a few responses carry commit > committed with commit_term."""
        out = []
        for g in self.lows:
            role, term, com = int(self.role[g]), int(self.term[g]), int(self.committed[g])
            peers = 16 if self.wide[g] else 8
            cand = role in (PRE_CANDIDATE, CANDIDATE)
            mine = PRE_VOTE_RESPONSE if role == PRE_CANDIDATE else VOTE_RESPONSE
            for p in range(peers):
                if p == self.self_slot[g] or not (int(self.present[g]) >> p & 1):
                    continue
                h, s = (g + 1, p - 8) if p >= 8 else (g, p)
                if cand and rng.random() < 0.85:
                    rej = rng.random() < 0.4
                    t = term + 1 if role == PRE_CANDIDATE and not rej and rng.random() < 0.7 else term
                    c = int(rng.integers(0, com + 1)) if rng.random() < 0.3 else 0
                    ct = int(rng.integers(1, 1 << 20)) if c and rng.random() < 0.5 else 0
                    if commit_vote and rng.random() < 0.1:
                        c, ct = com + 1 + int(rng.integers(0, 100)), int(rng.integers(1, 100))
                    out.append(F.frame(h, s, message(mine, t, rej, c, ct, to=1, frm=p + 1)))
                    if noise and rng.random() < 0.1:   # the same cell again, maybe with the other vote: DUP
                        rej2 = rng.random() < 0.5 and t == term   # (a rejection from a higher term is become_follower)
                        out.append(F.frame(h, s, message(mine, t, rej2, to=1, frm=p + 1)))
                if not noise or rng.random() > 0.15:
                    continue
                k = int(rng.integers(6))
                if k == 0:    # the other response type, at the group's own term
                    other = VOTE_RESPONSE if mine == PRE_VOTE_RESPONSE else PRE_VOTE_RESPONSE
                    out.append(F.frame(h, s, message(other, term, rng.random() < 0.5)))
                elif k == 1:  # a stale term
                    out.append(F.frame(h, s, message(mine, max(1, term - 1 - int(rng.integers(0, 3))), rng.random() < 0.5)))
                elif k == 2:  # another message type
                    out.append(F.frame(h, s, message(int(rng.choice([4, 9, 5, 17])), term)))
                elif k == 3:  # a peer slot past the group's 8
                    out.append(F.frame(h, 8 + int(rng.integers(8)), message(mine, term, rng.random() < 0.5)))
                elif k == 4:  # garbage bytes
                    out.append(F.frame(h, s, rng.integers(0, 256, int(rng.integers(1, 12)), dtype=np.uint8).tobytes()))
                else:         # a group past the arena, or a truncated frame
                    out.append(F.frame(self.n + 8 + int(rng.integers(100)), s, message(mine, term)) if rng.random() < 0.5
                               else F.frame(h, s, message(mine, term, True, 1 << 40, 7))[:-1])
        return out

    def transitions(self, outcomes, pre_role):
        """The caller's lists for the pass's outcomes (section 6): a Candidate that won becomes leader (step 3), a
        PreCandidate that won campaigns (step 1), a loser becomes follower (RESET at its term).  pre_role: the role of
        each group slot when the batch ran."""
        rows = []
        for g, w in zip(outcomes["group"].tolist(), outcomes["result"].tolist()):
            li, com = int(self.last[g]), int(self.committed[g])
            if w & 0xFF == B.VOTE_WON and pre_role[g] == PRE_CANDIDATE:
                rows.append((B.CTL_RESET, g, 0, 0, (NO_TERM_START, li, com, li)))
                rows.append((B.CTL_SET_TERM, g, 0, 0, (int(self.term[g]) + 1,)))
                rows.append((B.CTL_RESET_VOTES, g))
                rows.append((B.CTL_RECORD_VOTE, g, int(self.self_slot[g]), 1))
                rows.append((B.CTL_VOTE_RESULT, g))
            elif w & 0xFF == B.VOTE_WON:
                rows.append((B.CTL_RESET, g, 0, 0, (li + 1, li, com, li)))
                rows.append((B.CTL_BECOME_LEADER, g))
            else:
                rows.append((B.CTL_RESET, g, 0, 0, (NO_TERM_START, li, com, li)))
        return cmds(*rows)


def candidates(metas, terms, committed=None):
    """Oracle columns for the given group metas (one candidate each), last_index 10, committed 5 unless given."""
    n = len(metas)
    c = O.new_columns(n + 8, n)
    c.term_start[:] = B.NO_TERM_START
    c.meta[:n] = metas
    c.term[:n] = terms
    c.last_index[:n] = 10
    c.committed[:n] = 5 if committed is None else committed
    return c, np.zeros((O.SLOTS, c.cap), np.uint8)


def run_batch(c, votes, frames, select, pre=None):
    blob, off = F.batch(frames)
    return VW.batch(c, votes, blob, off, bitmap(select), None if pre is None else bitmap(pre))


# test_raft_paper.rs:199-250: (size, {id: vote}, the state after) for a candidate at term 1 whose self vote is in
ONE_ROUND = [
    (1, {}, "Leader"), (3, {2: True, 3: True}, "Leader"), (3, {2: True}, "Leader"),
    (5, {2: True, 3: True, 4: True, 5: True}, "Leader"), (5, {2: True, 3: True, 4: True}, "Leader"),
    (5, {2: True, 3: True}, "Leader"),
    (3, {2: False, 3: False}, "Follower"), (5, {2: False, 3: False, 4: False, 5: False}, "Follower"),
    (5, {2: True, 3: False, 4: False, 5: False}, "Follower"),
    (3, {}, "Candidate"), (5, {2: True}, "Candidate"), (5, {2: False, 3: False}, "Candidate"), (5, {}, "Candidate"),
]


def expected_state(first, outcomes):
    w = first if first & 0xFF != B.VOTE_PENDING else (int(outcomes["result"][0]) if len(outcomes) else B.VOTE_PENDING)
    return {B.VOTE_WON: "Leader", B.VOTE_LOST: "Follower", B.VOTE_PENDING: "Candidate"}[w & 0xFF]


def state_of(e):
    c = O.new_columns(e.n + 8, e.n)
    c.term_start[:] = B.NO_TERM_START
    c.meta[e.n_narrow:e.n:2], c.meta[e.n_narrow + 1:e.n:2] = META_WIDE_LO, META_WIDE_HI   # the allocated pairs
    vt = np.zeros((O.SLOTS, c.cap), np.uint8)
    assert np.all(CO.arena_control(c, vt, e.setup)["status"] == 0)
    CO.arena_control(c, vt, e.campaign)
    return c, vt
