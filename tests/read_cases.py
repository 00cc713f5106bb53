"""ReadIndex (ReadOnlyOption::Safe) scenarios for the read-index tests, written once against a driver: the oracle's
(oracle/read_oracle.c with the control oracle) or an arena's (the C-ABI).  The reference's read-only tests are
restated at the tracker level: what the leader's ReadOnly and ProgressTracker see of each message."""
import numpy as np

from oracle import oracle as O
from oracle import read_oracle as RO
from helpers import B
import hb_frames as F
from control_cmds import NO_TERM_START, META_WIDE_LO, META_WIDE_HI, cmds

HB_CTX = B.REC_HEARTBEAT | B.REC_READ_CTX


def reqs(*pairs) -> np.ndarray:
    out = np.zeros(len(pairs), dtype=B.READ_REQ_DTYPE)
    for i, (g, ctx) in enumerate(pairs):
        out[i]["group"], out[i]["ctx"] = g, ctx
    return out


def acks(*rows) -> np.ndarray:
    """rows of (group, peer_slot, ctx[, flags]) -> heartbeat response records carrying the ctx in `index`."""
    out = np.zeros(len(rows), dtype=B.APPEND_RESP_DTYPE)
    for i, r in enumerate(rows):
        g, s, ctx = r[:3]
        out[i] = (g, s, r[3] if len(r) > 3 else HB_CTX, 0, ctx, 0)
    return out


def pairs(released) -> list:
    return [(int(r["group"]), int(r["ctx"]), int(r["index"])) for r in released]


class OracleDriver:
    """n groups of an oracle arena, all allocated, with their ReadOnly queues."""

    def __init__(self, n, max_pending=8):
        self.c = O.new_columns(n + 8, n)
        self.c.term_start[:] = NO_TERM_START
        self.votes = np.zeros((O.SLOTS, self.c.cap), dtype=np.uint8)
        self.q = RO.ReadQueues(self.c.cap, max_pending)
        self.q.allocated[:n] = 1

    def control(self, *rows):
        return self.q.control(self.c, self.votes, cmds(*rows))["status"].tolist()

    def request(self, r):
        return self.q.request(self.c, r)

    def ack(self, recs):
        return self.q.ack_seq(self.c, recs)

    def recheck(self, groups):
        return self.q.recheck(self.c, groups)

    def queue(self, g):
        return [tuple(map(int, x)) for x in zip(*self.q.pending(g))]

    def last_ctx(self, g):
        return self.q.last_ctx(g)


class ArenaDriver:
    """n groups of a GPU arena with read queues."""

    def __init__(self, n, max_pending=8):
        self.a = B.Arena(n + 8)
        self.a.enable_read_index(max_pending)
        assert self.a.group_alloc_range(n) == 0

    def control(self, *rows):
        return self.a.control(cmds(*rows))["status"].tolist()

    def request(self, r):
        return self.a.read_index_request(r)

    def ack(self, recs):
        return self.a.read_index_ack(recs)

    def recheck(self, groups):
        return self.a.read_index_recheck(groups)

    def queue(self, g):
        return [tuple(map(int, x)) for x in zip(*self.a.read_index_get(g))]

    def last_ctx(self, g):
        d = self.a.device_alloc(8)
        self.a.read_index_last_ctx_device(g, 1, d)
        out = np.zeros(1, np.uint64)
        self.a.d2h(out, d)
        self.a.device_free(d)
        return int(out[0])


def leader(d, g, voters, learners=0, self_slot=0, committed=1, last_index=None):
    """Group g becomes leader (Raft::reset + become_leader, raft.rs:942-971, 1162-1203) over the given slot masks, then
    commits up to `committed` within its term (the leader's log ends at last_index)."""
    li = committed if last_index is None else last_index
    st = d.control((B.CTL_SET_CONF, g, self_slot, 0, (voters, 0, learners, 1)),
                   (B.CTL_RESET, g, 0, 0, (NO_TERM_START, 0, 0, 0)),
                   (B.CTL_BECOME_LEADER, g),                                  # term_start = last_index = 1
                   (B.CTL_SET_LOG_BOUNDS, g, 0, 0, (1, li)),
                   (B.CTL_COMMIT_TO, g, 0, 0, (committed,)))
    assert st == [B.OK] * 5, st


# --------------------------------------------------------------------------- the reference's tests, restated

def raft_frees_read_only_mem(d):
    """test_raft.rs:1442-1479: peers {1, 2}; the read is queued, the heartbeat carries its ctx, peer 2's response
    releases it and the queue is empty again."""
    leader(d, 0, 0b11)
    res, rel = d.request(reqs((0, 7)))
    assert res.tolist() == [B.READ_QUEUED] and len(rel) == 0
    assert d.queue(0) == [(7, 1, 0b01)] and d.last_ctx(0) == 7
    assert pairs(d.ack(acks((0, 1, 7)))) == [(0, 7, 1)]
    assert d.queue(0) == [] and d.last_ctx(0) == 0


def read_only_option_safe(d):
    """test_raft.rs:2230-2318: three voters.  Each row sends ctx1, ctx1, ctx11 (the second ctx1 is pending: nothing
    changes); without the pending flag both peers' responses arrive, with it they are dropped until ctx11 is sent
    again and its heartbeat's responses release both reads, in queue order, with the row's commit index."""
    leader(d, 0, 0b111)
    for row, (wri, pending) in enumerate([(11, False), (21, False), (31, False), (41, True), (51, True), (61, True)]):
        c1, c11 = 10 * row + 1, 10 * row + 2
        assert d.control((B.CTL_SET_LOG_BOUNDS, 0, 0, 0, (1, wri)), (B.CTL_COMMIT_TO, 0, 0, 0, (wri,))) == [B.OK, B.OK]
        res, rel = d.request(reqs((0, c1), (0, c1), (0, c11)))
        assert res.tolist() == [B.READ_QUEUED, B.READ_DUP, B.READ_QUEUED] and len(rel) == 0
        if pending:   # the responses are dropped; ctx11 is requested again and its heartbeat answered
            res, rel = d.request(reqs((0, c11)))
            assert res.tolist() == [B.READ_DUP]
            assert d.last_ctx(0) == c11
            got = pairs(d.ack(acks((0, 1, c11), (0, 2, c11))))
        else:         # the heartbeats of ctx1, then of ctx11, answered by both peers
            got = pairs(d.ack(acks((0, 1, c1)))) + pairs(d.ack(acks((0, 2, c1)))) + \
                pairs(d.ack(acks((0, 1, c11)))) + pairs(d.ack(acks((0, 2, c11))))
        assert got == [(0, c1, wri), (0, c11, wri)], (row, got)
        assert d.queue(0) == []


def read_only_with_learner(d):
    """test_raft.rs:2321-2391: one voter and one learner is a singleton, so every read is ready at once with the
    commit index; and (group 1: voters {1, 2}, learner 3) a learner's ack does not make a quorum."""
    leader(d, 0, 0b01, learners=0b10)
    for wri, ctx in [(11, 1), (21, 2), (31, 3), (41, 4)]:
        assert d.control((B.CTL_SET_LOG_BOUNDS, 0, 0, 0, (1, wri)), (B.CTL_COMMIT_TO, 0, 0, 0, (wri,))) == [B.OK, B.OK]
        res, rel = d.request(reqs((0, ctx)))
        assert res.tolist() == [B.READ_READY] and pairs(rel) == [(0, ctx, wri)]
        assert d.queue(0) == []
    leader(d, 1, 0b011, learners=0b100, committed=5)
    res, _ = d.request(reqs((1, 9)))
    assert res.tolist() == [B.READ_QUEUED]
    assert pairs(d.ack(acks((1, 2, 9)))) == []
    assert d.queue(1) == [(9, 5, 0b101)]
    assert pairs(d.ack(acks((1, 1, 9)))) == [(1, 9, 5)]


def read_only_for_new_leader(d):
    """test_raft.rs:2503-2578: the new leader's log holds entries 1-2 of the old term, its own noop is 3 and it has
    committed only 1: the read is dropped.  Once entry 4 of its term commits, the read is queued with index 4 and
    released by the peers' acks."""
    assert d.control((B.CTL_SET_CONF, 0, 0, 0, (0b111, 0, 0, 3)),
                     (B.CTL_RESET, 0, 0, 0, (NO_TERM_START, 2, 1, 2)),
                     (B.CTL_BECOME_LEADER, 0)) == [B.OK] * 3                  # term_start = last_index = 3
    res, rel = d.request(reqs((0, 5)))
    assert res.tolist() == [B.READ_DROPPED] and len(rel) == 0 and d.queue(0) == []
    assert d.control((B.CTL_SET_LOG_BOUNDS, 0, 0, 0, (3, 4)), (B.CTL_COMMIT_TO, 0, 0, 0, (4,))) == [B.OK, B.OK]
    res, _ = d.request(reqs((0, 5)))
    assert res.tolist() == [B.READ_QUEUED]
    assert pairs(d.ack(acks((0, 1, 5), (0, 2, 5)))) == [(0, 5, 4)]
    # a non-leader (term_start = NO_TERM_START) drops every request
    assert d.control((B.CTL_RESET, 0, 0, 0, (NO_TERM_START, 4, 4, 4))) == [B.OK]
    assert d.request(reqs((0, 6)))[0].tolist() == [B.READ_DROPPED]


def read_when_quorum_becomes_less(d):
    """test_raft.rs:5380-5415: two voters, peer 2's heartbeat response is lost; removing peer 2 leaves a one-voter
    quorum, and post_conf_change's recheck releases the read."""
    leader(d, 0, 0b11)
    assert d.request(reqs((0, 3)))[0].tolist() == [B.READ_QUEUED]
    assert pairs(d.recheck([0])) == []                     # the configuration has not changed: no quorum yet
    assert d.control((B.CTL_SET_CONF, 0, 0, 0, (0b01, 0, 0, 2))) == [B.OK]
    assert pairs(d.recheck([0])) == [(0, 3, 1)]
    assert d.queue(0) == []


REFERENCE_CASES = [raft_frees_read_only_mem, read_only_option_safe, read_only_with_learner, read_only_for_new_leader,
                   read_when_quorum_becomes_less]


def edge_cases(d, n_groups):
    """What the device form adds, on an arena of n_groups groups with max_pending = 4: FULL, NO_CTX, NO_GROUP (an
    unallocated group), acks that find nothing, the removed-peer and reset hooks."""
    leader(d, 0, 0b111, learners=0b1000)
    res, _ = d.request(reqs(*[(0, 100 + k) for k in range(5)], (0, 0), (n_groups + 1, 1)))
    assert res.tolist() == [B.READ_QUEUED] * 4 + [B.READ_FULL, B.READ_NO_CTX, B.READ_NO_GROUP]
    # an unknown ctx, ctx 0, an absent peer, a record without READ_CTX, an unallocated group: nothing
    assert pairs(d.ack(acks((0, 1, 999), (0, 1, 0), (0, 5, 101), (0, 1, 101, B.REC_HEARTBEAT), (n_groups + 1, 0, 1)))) == []
    # peer 2 acks the second read: it and the one in front of it are released
    assert pairs(d.ack(acks((0, 2, 101)))) == [(0, 100, 1), (0, 101, 1)]
    assert pairs(d.ack(acks((0, 1, 103), (0, 1, 103)))) == [(0, 102, 1), (0, 103, 1)]
    # the learner's ack stays in the mask without making a quorum; removing the learner clears its bit
    assert d.request(reqs((0, 105)))[0].tolist() == [B.READ_QUEUED]
    assert pairs(d.ack(acks((0, 3, 105)))) == [] and d.queue(0) == [(105, 1, 0b1001)]
    assert d.control((B.CTL_SET_CONF, 0, 0, 0, (0b111, 0, 0, 2))) == [B.OK]
    assert d.queue(0) == [(105, 1, 0b0001)] and d.last_ctx(0) == 105
    # Raft::reset (raft.rs:957) empties the queue
    assert d.control((B.CTL_RESET, 0, 0, 0, (1, 1, 1, 1))) == [B.OK]
    assert d.queue(0) == [] and d.last_ctx(0) == 0


# --------------------------------------------------------------------------- random workloads

def random_setup(rng, n_narrow, n_wide):
    """A control list that configures n_narrow narrow groups [0, n_narrow) and n_wide wide groups (low halves
    n_narrow, n_narrow + 2, ...): plain, joint and learner configurations; leaders that have or have not committed
    in their term, followers; some one-voter singletons."""
    rows = []
    for k in range(n_narrow + n_wide):
        wide = k >= n_narrow
        g = k if not wide else n_narrow + 2 * (k - n_narrow)
        peers, lim = (16, 0xFFFF) if wide else (8, 0xFF)
        r = rng.random()
        if r < 0.1:
            inc = 1 << int(rng.integers(peers))                                 # a singleton
        elif wide:
            inc = int(rng.integers(1, lim + 1)) | (1 << (8 + int(rng.integers(8))))
        else:
            inc = 0x1F if rng.random() < 0.5 else int(rng.integers(1, lim + 1))
        out = int(rng.integers(0, lim + 1)) if rng.random() < 0.2 else 0
        learn = int(rng.integers(0, lim + 1)) & ~(inc | out) & lim if rng.random() < 0.3 else 0
        present = [p for p in range(peers) if (inc | out | learn) >> p & 1]
        self_slot = int(rng.choice(present)) if rng.random() < 0.95 else B.CTL_NO_SELF
        li = int(rng.integers(5, 60))
        rows.append((B.CTL_SET_CONF, g, self_slot, 0, (inc, out, learn, li + 1)))
        rows.append((B.CTL_RESET, g, 0, 0, (NO_TERM_START, li, int(rng.integers(0, li + 1)), li)))
        if rng.random() < 0.85:                                                  # a leader
            rows.append((B.CTL_BECOME_LEADER, g))
            top = li + 1 + int(rng.integers(0, 20))
            rows.append((B.CTL_SET_LOG_BOUNDS, g, 0, 0, (li + 1, top)))
            if rng.random() < 0.85:                                              # that has committed in its term
                rows.append((B.CTL_COMMIT_TO, g, 0, 0, (int(rng.integers(li + 1, top + 1)),)))
    return cmds(*rows)


def random_requests(rng, n_groups_total, per_group, ctx_space, bad_groups=()):
    """Requests for a random subset of group slots [0, n_groups_total) (high halves and unallocated ones included
    via bad_groups), in group order, several per group, ctx ids drawn from a small space so that duplicates occur;
    a few ctx 0."""
    gs = np.concatenate([rng.integers(0, n_groups_total, int(n_groups_total * per_group)), np.asarray(bad_groups, dtype=np.int64)])
    gs.sort()
    out = np.zeros(len(gs), dtype=B.READ_REQ_DTYPE)
    out["group"] = gs
    out["ctx"] = rng.integers(1, ctx_space + 1, len(gs))
    out["ctx"][rng.random(len(gs)) < 0.002] = 0
    return out


def random_acks(rng, q, meta, n_groups_total, n, wide_hi):
    """Heartbeat responses: mostly for pending contexts from random peer slots (absent peers and learners included),
    some repeated, some for unknown contexts or ctx 0, some without READ_CTX; shuffled.  q: oracle queues (for the
    pending contexts), meta: the group metas, wide_hi: bool per group slot."""
    gs = rng.integers(0, n_groups_total, n)
    slots = rng.integers(0, 8, n)
    recs = np.zeros(n, dtype=B.APPEND_RESP_DTYPE)
    recs["group"], recs["peer_slot"] = gs, slots
    recs["flags"] = HB_CTX
    qg = np.where(wide_hi[gs], gs - 1, gs)
    cnt = q.count[qg].astype(np.int64)
    pick = rng.integers(0, np.maximum(cnt, 1))
    ctx = np.where(cnt > 0, q.ctx[qg, np.minimum(pick, q.max_pending - 1)], rng.integers(1, 50, n).astype(np.uint64))
    r = rng.random(n)
    ctx = np.where(r < 0.05, rng.integers(1, 1 << 40, n).astype(np.uint64), ctx)
    ctx = np.where(r > 0.99, np.uint64(0), ctx)
    recs["index"] = ctx
    recs["commit"] = rng.integers(0, 60, n)
    recs["flags"][rng.random(n) < 0.03] = B.REC_HEARTBEAT
    recs["flags"][rng.random(n) < 0.01] = 0
    dup = rng.random(n) < 0.1                                   # repeated cells
    recs[dup] = recs[rng.integers(0, n, int(dup.sum()))]
    return recs[rng.permutation(n)]


def by_group(released) -> np.ndarray:
    """Released reads in a canonical order that keeps each group's own order: a stable sort by group."""
    r = np.asarray(released)
    return r[np.argsort(r["group"], kind="stable")]


def oracle_queue_view(q, n):
    """(counts, ctx, index, acks) of the oracle's first n queues, entries past the count zeroed (raftgpu_read_index_read's
    layout)."""
    k = np.arange(q.max_pending)[None, :] < q.count[:n, None]
    return (q.count[:n].copy(), np.where(k, q.ctx[:n], 0).astype(np.uint64), np.where(k, q.index[:n], 0).astype(np.uint64),
            np.where(k, q.acks[:n], 0).astype(np.uint16))


def queues_equal(a, q, n, what):
    got, want = a.read_index_read(0, n), oracle_queue_view(q, n)
    for name, x, y in zip(("count", "ctx", "index", "acks"), got, want):
        if not np.array_equal(x, y):
            g = int(np.argwhere(x != y)[0][0])
            raise AssertionError(f"{what}: queue {name} of group {g}: got {x[g]} want {y[g]}")


def mixed_batch(rng, d, n, terms, reads, k):
    """k frames, shuffled: append responses (accepts near matched, rejects without log_term), heartbeat responses
    (contexts of length 0, 8 and others; ids pending, released earlier or never queued), other message types;
    stale terms; several frames per cell (a wide group's peers 8..15 are named through its high half)."""
    gs = rng.integers(0, n, k)
    hi_half = (d.c.meta[gs] & META_WIDE_HI) != 0
    slots = rng.integers(0, 8, k)
    kind = rng.random(k)
    stale = rng.random(k) < 0.05
    qg = np.where(hi_half, gs - 1, gs)
    frames = []
    for i in range(k):
        g, s = int(gs[i]), int(slots[i])
        t = int(terms[g]) + (1 if stale[i] else 0)
        if kind[i] < 0.35:     # MsgAppendResponse
            m = int(d.c.matched[s, g])
            if rng.random() < 0.1:
                body = F.message(4, term=t, index=m + 1, reject=True, reject_hint=max(0, m - 1))
            else:
                body = F.message(4, term=t, index=m + int(rng.integers(0, 4)), commit=m)
        elif kind[i] < 0.93:   # MsgHeartbeatResponse
            r = rng.random()
            ctx = None
            if r < 0.55:
                cnt = int(d.q.count[qg[i]])
                x = int(d.q.ctx[qg[i], int(rng.integers(0, cnt))]) if cnt else int(rng.integers(1, 60))
                ctx = F.ctx_bytes(x)
            elif r < 0.65:
                ctx = F.ctx_bytes(int(rng.integers(1, 1 << 62)))                 # never queued
            elif r < 0.72:
                ctx = bytes(rng.integers(0, 256, int(rng.choice([1, 7, 9, 16]))).astype(np.uint8))
            body = F.message(9, term=t, commit=int(rng.integers(0, 80)), context=ctx)
        else:                  # other types, some with a context
            body = F.message(int(rng.choice([3, 6, 8, 15, 16])), term=t, index=5,
                             context=F.ctx_bytes(7) if rng.random() < 0.5 else None)
        frames.append(F.frame(g, s, body))
    dup = rng.random(k) < 0.1                       # more frames for cells already in the batch
    frames += [frames[j] for j in rng.integers(0, k, int(dup.sum()))]
    order = rng.permutation(len(frames))
    return F.batch([frames[j] for j in order])
