"""Followers for the term-prefix tests (raftgpu_follower_term_wire, oracle/follow_term_oracle.c): random groups in every
role with the caller's voter table, MsgAppend / MsgHeartbeat batches at lower, equal and higher terms with one `from`
per term, the caller's host side of a bump, and the sequence "this pass, raftgpu_follower_heartbeat,
raftgpu_follower_append" run on the batch oracles, with its DUP frames resubmitted until none is left."""
import numpy as np

from helpers import B
from control_cmds import cmds
from oracle import app_follow_oracle as AL
from oracle import follow_term_oracle as FT
from oracle import hb_follow_oracle as HF
from oracle import vote_request_oracle as VR
import app_follow as A
import hb_follow as HB
import hb_frames as F
import vote_request_frames as Q

APPEND, HEARTBEAT = 3, 8


def leader_of(term: int) -> int:
    """One `from` per term, as a real leader's frames carry."""
    return 2 + term % 5


def scenario(rng, n_narrow, n_wide, p_role=(0.55, 0.15, 0.2, 0.1), p_select=0.95, p_reply=0.5):
    """Q.Scenario's groups, table and setup, with RAFTGPU_VOTER_STALE_REPLY on a share of the groups."""
    s = Q.Scenario(rng, n_narrow, n_wide, p_role=p_role, p_select=p_select)
    for g in s.lows:
        if rng.random() < p_reply:
            s.table["flags"][g] |= FT.STALE_REPLY
    s.leader = np.zeros(s.n, np.uint64)
    return s


def frames(rng, s, per_group=(1, 4), deltas=(-2, -1, 0, 0, 1, 1, 3), p_append=0.5):
    """MsgAppend / MsgHeartbeat frames to every group at its term + one of deltas (at least 1), from leader_of(term),
    entry-less appends near the group's log."""
    out = []
    for g in s.lows:
        term, last, com = int(s.term[g]), int(s.last[g]), int(s.committed[g])
        lt = int(s.table[g]["last_term"])
        for _ in range(int(rng.integers(per_group[0], per_group[1] + 1))):
            t = max(1, term + int(rng.choice(deltas)))
            frm = leader_of(t)
            if rng.random() < p_append:
                ix = max(0, last + int(rng.choice([-1, 0, 0, 1])))
                body = A.message(APPEND, t, lt if rng.random() < 0.8 else lt + 1, ix,
                                 int(rng.integers(0, com + 2)), frm=frm, to=int(s.table[g]["id"]))
            else:
                body = F.message(HEARTBEAT, t, int(rng.integers(0, com + 1)), frm=frm)
            out.append(F.frame(g, int(rng.integers(16)), body))
    return out


def types_of(frames_):
    """msg_type of each frame (the second byte of the Message: every frame here starts with field 1)."""
    return np.array([f[5] for f in frames_], np.uint8)


def log_table(s):
    """The follower passes' log table: a run of the last term over the group's last five indexes."""
    lt = np.zeros(s.n, AL.LOG_DTYPE)
    lt["id"] = s.table["id"]
    lt["run_term"] = s.table["last_term"]
    lt["run_start"] = np.maximum(1, s.last.astype(np.int64) - 5).astype(np.uint64)
    return lt


def selected(s, role, table):
    """The follower passes' selection: a Follower that the caller's table selects."""
    return (role == Q.FOLLOWER) & ((table["flags"] & B.VOTER_SELECT) != 0)


def host_side(table, role, leader, status, out, frames_):
    """become_follower(T, m.from)'s host side for every RAFTGPU_FTERM_BUMPED frame."""
    for i in np.flatnonzero((status >> 4 == B.WIRE_OK) & ((status & B.FTERM_BUMPED) != 0)):
        g = int(np.frombuffer(frames_[i][:4], "<u4")[0]) >> 4
        role[g], leader[g], table["vote"][g] = Q.FOLLOWER, out[i][0], 0
        table["flags"][g] &= ~np.uint32(VR.LEADER | VR.LEASE)
        if out[i][0]:
            table["flags"][g] |= VR.LEADER


def follower_passes(c, s, role, table, frames_, idx):
    """raftgpu_follower_heartbeat's then raftgpu_follower_append's batch forms over frames_[idx], each resubmitting
    its DUP frames until none is left -> ({frame: final status}, [responses])."""
    sel = selected(s, role, table)
    logs = log_table(s)
    logs["flags"] = np.where(sel, AL.SELECT, 0)
    final, resps = {}, []
    for typ in (HEARTBEAT, APPEND):
        pend = [i for i in idx if frames_[i][5] == typ]
        while pend:
            blob, off = F.batch([frames_[i] for i in pend])
            if typ == HEARTBEAT:
                st, _, rb, ro, _ = HF.follower_heartbeats(c, None, blob, off, HB.bitmap(sel), s.table["id"])
            else:
                st, _, rb, ro, _ = AL.batch(c, None, logs, blob, off)
            resps += [rb[a:b].tobytes() for a, b in zip(ro[:-1], ro[1:])]
            nxt = []
            for k, i in enumerate(pend):
                final[i] = int(st[k])
                if st[k] >> 4 == B.WIRE_DUP:
                    nxt.append(i)
            pend = nxt
    return final, resps


def noise(rng, s, k):
    """Frames the checks before the verdict settle: other types, garbage, truncated frames, high halves, m.term 0 and
    groups past the arena's highest slot."""
    out = []
    for _ in range(k):
        g = int(rng.choice(s.lows))
        term = int(s.term[g])
        kind = int(rng.integers(6))
        if kind == 0:
            out.append(F.frame(g, 0, F.message(int(rng.choice([4, 9, 5, 7, 10])), term + 1, frm=2)))
        elif kind == 1:
            out.append(F.frame(g, 0, rng.integers(0, 256, int(rng.integers(1, 12)), dtype=np.uint8).tobytes()))
        elif kind == 2:
            out.append(F.frame(g, 0, F.message(8, term + 1, 1 << 40, frm=2)[:-3]))
        elif kind == 3:
            out.append(F.frame(g + 1 if s.wide[g] else g, 0, F.message(8, term + 1 if s.wide[g] else 0, frm=2)))
        elif kind == 4:
            out.append(F.frame(g, 0, F.message(3, 0, frm=2)))
        else:
            out.append(F.frame(s.n + int(rng.integers(1, 100)), 0, F.message(8, term + 1, frm=2)))
    return out


def leaders(n, P, term, li):
    """n narrow leader groups of P voters (self slot 0) at `term`: the empty entry at li + 1 = term_start, committed li,
    every peer a Replicate peer matched at li that was sent the empty entry (next li + 2), and the earlier run [1, li]
    at term - 1 stated."""
    a = B.Arena(n + 64)
    a.enable_leader_runs()
    assert a.group_alloc_range(n) == 0
    ops = []
    for g in range(n):
        ops += [(B.CTL_SET_CONF, g, 0, 0, ((1 << P) - 1, 0, 0, li + 1)), (B.CTL_RESET, g, 0, 0, (li + 1, li, li, li)),
                (B.CTL_SET_TERM, g, 0, 0, (term,)), (B.CTL_BECOME_LEADER, g)]
        for s in range(1, P):
            ops += [(B.CTL_PROGRESS_OP, g, s, B.POP_MAYBE_UPDATE, (li,)), (B.CTL_PROGRESS_OP, g, s, B.POP_BECOME_REPLICATE),
                    (B.CTL_PROGRESS_OP, g, s, B.POP_OPTIMISTIC_UPDATE, (li + 1,))]
    assert np.all(a.control(cmds(*ops))["status"] == 0)
    rows = np.zeros(n, B.LEADER_RUNS_DTYPE)
    rows["group"], rows["term"], rows["term_start"] = np.arange(n), term, li + 1
    rows["run_start"][:, 0], rows["run_term"][:, 0] = 1, term - 1
    assert np.all(a.leader_runs_set(rows) == 0)
    return a


def to_followers(blob, off, P):
    """The transport: leader cell (g, s) -> follower group g * (P - 1) + s - 1, x = s."""
    h = HB.headers(blob, off)
    return HB.with_headers(blob, off, (((h >> 4) * (P - 1) + (h & 15) - 1) << 4 | (h & 15)).astype(np.uint32))


def to_leaders(blob, off, P):
    h = HB.headers(blob, off)
    return HB.with_headers(blob, off, (((h >> 4) // (P - 1)) << 4 | (h & 15)).astype(np.uint32))


def followers(nf, term, li, P, rng):
    fa = B.Arena(nf + 64)
    assert fa.group_alloc_range(nf) == 0
    fcom = (li - rng.integers(0, 4, nf)).astype(np.uint64)
    for col, arr in ((B.COL_TERM, np.full(nf, term, np.uint64)), (B.COL_LAST_INDEX, np.full(nf, li, np.uint64)),
                     (B.COL_COMMITTED, fcom), (B.COL_TERM_START, np.full(nf, B.NO_TERM_START, np.uint64))):
        fa.column_write(col, 0, 0, arr)
    table = Q.voters(nf)
    table["id"] = np.arange(nf) % (P - 1) + 2
    table["persisted"], table["last_term"] = li, term
    table["flags"] = B.VOTER_SELECT | B.VOTER_STALE_REPLY
    return fa, table
