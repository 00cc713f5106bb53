"""Leaders for the term-prefix tests at a leader (raftgpu_leader_term_wire, oracle/leader_term_oracle.c): random leader
groups with the caller's voter table, batches of the six types a leader receives at lower, equal and higher terms, the
leader passes' batch oracles, the caller's host side of a bump, and the reference's delivery order."""
import numpy as np

from helpers import B
from oracle import hb_wire_oracle as H
from oracle import oracle as O
from oracle import vote_request_oracle as VR
import app_follow as A
import follow_term as T
import hb_frames as F
import vote_request_frames as Q

APPEND, APP_RESP, VOTE_RESP, HEARTBEAT, HB_RESP, PRE_VOTE_RESP = 3, 4, 6, 8, 9, 18
TYPES = (APPEND, APP_RESP, VOTE_RESP, HEARTBEAT, HB_RESP, PRE_VOTE_RESP)


def scenario(rng, n_narrow, n_wide, p_reply=0.5):
    """Leaders only: T.scenario's groups, table and setup with every group a Leader."""
    return T.scenario(rng, n_narrow, n_wide, p_role=(0.0, 0.0, 0.0, 1.0), p_reply=p_reply)


def frames(rng, s, per_group=(1, 6), deltas=(-2, -1, 0, 0, 0, 1, 1, 3)):
    """Frames of the six types to every leader at its term + one of deltas (at least 1): MsgAppend / MsgHeartbeat to
    the group's own slot from T.leader_of(term), responses to a cell (a pair's high half for a share of them), at
    most one MsgAppendResponse and one MsgHeartbeatResponse per cell -> (frames, meta), meta per frame = (low half,
    type, m.term, reject)."""
    out, meta = [], []
    for g in s.lows:
        term, last, com = int(s.term[g]), int(s.last[g]), int(s.committed[g])
        lt = int(s.table[g]["last_term"])
        used = set()
        for _ in range(int(rng.integers(per_group[0], per_group[1] + 1))):
            t = max(1, term + int(rng.choice(deltas)))
            typ = int(rng.choice(TYPES))
            reject = False
            if typ in (APPEND, HEARTBEAT):
                frm = T.leader_of(t)
                if typ == APPEND:
                    body = A.message(APPEND, t, lt, max(0, last + int(rng.choice([-1, 0, 1]))),
                                     int(rng.integers(0, com + 2)), frm=frm, to=int(s.table[g]["id"]))
                else:
                    body = F.message(HEARTBEAT, t, int(rng.integers(0, com + 1)), frm=frm)
                out.append(F.frame(g, int(rng.integers(16)), body))
            else:
                h = g + 1 if s.wide[g] and rng.random() < 0.3 else g
                slot = int(rng.integers(1, 8))
                if typ in (APP_RESP, HB_RESP):
                    if (h, slot, typ) in used:
                        continue
                    used.add((h, slot, typ))
                    body = F.message(typ, t, commit=int(rng.integers(0, com + 1)) if typ == HB_RESP else 0,
                                     index=int(rng.integers(0, last + 1)) if typ == APP_RESP else 0, frm=slot + 1)
                else:
                    reject = bool(rng.random() < 0.5)
                    body = F.message(typ, t, reject=reject, frm=slot + 1)
                out.append(F.frame(h, slot, body))
            meta.append((g, typ, t, reject))
    return out, meta


def leader_passes(c, frames_):
    """The wire step's and raftgpu_heartbeat_wire's batch oracles over the whole batch (each takes its own type at the
    group's term) -> their status bytes, WIRE_SKIP_TYPE for the other's frames."""
    blob, off = F.batch(frames_)
    st, recs, _, _ = O.wire_decode_batch(blob, off, c.n_groups, c.term)
    ok = np.flatnonzero(st == O.WIRE_OK)
    O.arena_apply(c, np.array([tuple(recs[i]) for i in ok], dtype=B.APPEND_RESP_DTYPE), mode=0)
    hst, _ = H.apply(c, None, blob, off, c.term)
    return np.where(st == O.WIRE_SKIP_TYPE, hst >> 4, st)


def host_side(table, role, leader, status, out, meta):
    """become_follower(T, leader_id)'s host side for every RAFTGPU_FTERM_BUMPED frame, and the follower passes'
    selection for the Follower it makes."""
    for i in np.flatnonzero((status >> 4 == B.WIRE_OK) & ((status & B.FTERM_BUMPED) != 0)):
        g = meta[i][0]
        role[g], leader[g], table["vote"][g] = Q.FOLLOWER, out[i][0], 0
        table["flags"][g] &= ~np.uint32(VR.LEADER | VR.LEASE)
        if out[i][0]:
            table["flags"][g] |= VR.LEADER
        table["flags"][g] |= B.VOTER_SELECT


def delivery_order(s, meta):
    """The reference's order for the batch: granting pre-vote responses, the frames at the leader's term, each group's
    claimant, the other frames at T, then the stale frames, each in batch order -> (order, the frames at T > term)."""
    top = {}
    grant = [i for i, (g, typ, t, rej) in enumerate(meta) if typ == PRE_VOTE_RESP and not rej]
    for i, (g, typ, t, rej) in enumerate(meta):
        if i not in grant:
            top[g] = max(top.get(g, int(s.term[g])), t)
    at_term = [i for i, (g, typ, t, rej) in enumerate(meta) if i not in grant and t == int(s.term[g])]
    at_top = [i for i, (g, typ, t, rej) in enumerate(meta) if i not in grant and t == top[g] and t > int(s.term[g])]
    claim = {}
    for i in at_top:
        claim.setdefault(meta[i][0], i)
    claimants = sorted(claim.values())
    rest = [i for i in at_top if i not in claimants]
    taken = set(grant) | set(at_term) | set(at_top)
    stale = [i for i in range(len(meta)) if i not in taken]
    return grant + at_term + claimants + rest + stale, at_top


def noise(rng, s, k):
    """Frames the checks before the verdict settle: other types, garbage, truncated frames, a pair's high half on types
    3 and 8, m.term 0 and groups past the arena's highest slot."""
    out = []
    for _ in range(k):
        g = int(rng.choice(s.lows))
        term = int(s.term[g])
        kind = int(rng.integers(6))
        if kind == 0:
            out.append(F.frame(g, 0, F.message(int(rng.choice([5, 7, 10, 17])), term + 1, frm=2)))
        elif kind == 1:
            out.append(F.frame(g, 0, rng.integers(0, 256, int(rng.integers(1, 12)), dtype=np.uint8).tobytes()))
        elif kind == 2:
            out.append(F.frame(g, 0, F.message(4, term + 1, 1 << 40, frm=2)[:-3]))
        elif kind == 3:
            out.append(F.frame(g + 1 if s.wide[g] else g, 0, F.message(8, term + 1 if s.wide[g] else 0, frm=2)))
        elif kind == 4:
            out.append(F.frame(g, 1, F.message(9, 0, frm=2)))
        else:
            out.append(F.frame(s.n + int(rng.integers(1, 100)), 0, F.message(4, term + 1, frm=2)))
    return out
