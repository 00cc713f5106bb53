"""Followers for the term-prefix tests (raftgpu_follower_term_wire, oracle/follow_term_oracle.c): random groups in every
role with the caller's voter table, MsgAppend / MsgHeartbeat batches at lower, equal and higher terms with one `from`
per term, the caller's host side of a bump, and the sequence "this pass, raftgpu_follower_heartbeat,
raftgpu_follower_append" run on the batch oracles, with its DUP frames resubmitted until none is left."""
import numpy as np

from helpers import B
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
