"""The heartbeat-frame oracle (oracle/hb_frames_oracle.c): its encoder against python-protobuf's bytes
(tests/golden/wire/heartbeats.json, scripts/gen_wire_heartbeat_golden.py), its frames decoded back to the fields they
were built from, test_bcast_beat and the read-only cases restated, and the one-broadcast-per-round form of ReadIndex's
heartbeats against the reference's one broadcast per request."""
import json
import os

import numpy as np
import pytest

from oracle import hb_frames_oracle as HF
from oracle import hb_wire_oracle as H
from helpers import B, O
import hb_frames as F
import read_cases as R

HERE = os.path.dirname(os.path.abspath(__file__))
U64 = (1 << 64) - 1


def vectors():
    with open(os.path.join(HERE, "golden", "wire", "heartbeats.json")) as f:
        return json.load(f)["vectors"]


def frames_of(blob, offsets):
    """[(group, slot, decoded message)] of a frame blob."""
    out = []
    for lo, hi in zip(offsets[:-1].tolist(), offsets[1:].tolist()):
        hdr = int.from_bytes(bytes(blob[lo:lo + 4]), "little")
        m = H.decode_message(bytes(blob[lo + 4:hi]))
        assert m is not None
        out.append((hdr >> 4, hdr & 15, m))
    return out


def test_golden_vectors_encode_byte_for_byte():
    vs = vectors()
    for v in vs:
        got = HF.encode_heartbeat(v["to"], v["from"], v["term"], v["commit"], v["ctx"] or 0)
        assert got.hex() == v["hex"], v
        assert len(got) <= 56
    # the coverage the vectors promise
    for name in ("to", "from", "term"):
        vals = {v[name] for v in vs}
        assert {0, 1, 127, 128, 1 << 32, 1 << 63, U64} <= vals, name
    assert {0, U64} <= {v["commit"] for v in vs}
    assert {None, 0, 1, U64} <= {v["ctx"] for v in vs}


def _leader_columns(n, cap=None):
    c = O.new_columns(cap or n + 8, n)
    c.term_start[:] = R.NO_TERM_START
    return c


def test_frames_decode_to_their_fields():
    """Random leaders of every configuration (narrow, joint, learners, no self slot, wide pairs): each frame decodes
    through hwo_decode_message to exactly the fields send_heartbeat + send give it, in (group, slot) order."""
    rng = np.random.default_rng(0xB0A7)
    n = 600
    c = _leader_columns(n)
    for g in range(0, n - 100):
        inc = int(rng.integers(1, 256))
        out = int(rng.integers(0, 256)) if rng.random() < 0.2 else 0
        learn = int(rng.integers(0, 256)) & ~(inc | out) if rng.random() < 0.3 else 0
        c.meta[g] = B.make_meta(inc, out, learn, None if rng.random() < 0.1 else int(rng.integers(8)))
    for lo in range(n - 100, n, 2):
        c.meta[lo] = B.make_meta(int(rng.integers(1, 256)), 0, 0, int(rng.integers(8))) | R.META_WIDE_LO
        c.meta[lo + 1] = B.make_meta(int(rng.integers(1, 256)), 0, 0, None) | R.META_WIDE_HI
    c.term_start[:n] = np.where(rng.random(n) < 0.8, 5, R.NO_TERM_START)
    c.term[:n] = rng.choice(np.array([0, 1, 127, 128, 1 << 40, U64], np.uint64), n, p=[0.05, 0.35, 0.15, 0.15, 0.15, 0.15])
    c.committed[:n] = rng.integers(0, 1 << 40, n)
    c.matched[:, :n] = rng.integers(0, 1 << 40, (8, n))
    q = R.RO.ReadQueues(c.cap, 4)
    q.allocated[:n] = 1
    q.count[:n] = rng.integers(0, 3, n)
    q.ctx[:n] = rng.integers(1, 1 << 63, (n, 4), dtype=np.uint64)
    ids = rng.integers(0, 1 << 63, (9, n), dtype=np.uint64)
    ids[:, ::7] = rng.choice(np.array([0, 1, 128, U64], np.uint64), (9, len(range(0, n, 7))))
    blob, offsets, totals = HF.bcast_heartbeats(c, q, 0, n, ids)
    assert totals[0] > 2 * n and offsets[0] == 0 and offsets[-1] == len(blob)
    got = frames_of(blob, offsets)
    want = []
    no_term = 0
    for g in range(n):
        lo = g - 1 if c.meta[g] & R.META_WIDE_HI else g
        if c.term_start[lo] == R.NO_TERM_START:
            continue
        if c.term[lo] == 0:
            no_term += lo == g
            continue
        meta = int(c.meta[g])
        peers = (meta | meta >> 8 | meta >> 16) & 0xFF
        if meta & B.META_HAS_SELF:
            peers &= ~(1 << (meta >> 24 & 7))
        wide = c.meta[lo] & R.META_WIDE_LO
        committed = int(max(c.committed[lo], c.committed[lo + 1])) if wide else int(c.committed[g])
        ctx = int(q.ctx[lo, q.count[lo] - 1]) if q.count[lo] else 0
        for s in range(8):
            if peers >> s & 1:
                want.append((g, s, int(ids[s, g]), int(ids[8, lo]), int(c.term[lo]), min(int(c.matched[s, g]), committed), ctx))
    assert int(totals[2]) == no_term > 0
    assert len(got) == len(want) == int(totals[0])
    for (g, s, m), (wg, ws, to, frm, term, commit, ctx) in zip(got, want):
        assert (g, s) == (wg, ws)
        assert m == {"msg_type": 8, "reject": 0, "to": to, "from": frm, "term": term, "log_term": 0, "index": 0,
                     "commit": commit, "commit_term": 0, "request_snapshot": 0, "reject_hint": 0, "priority": 0,
                     "context": F.ctx_bytes(ctx) if ctx else b""}, (g, s)


def test_bcast_beat():
    """test_raft.rs:2680-2735: a leader of {1, 2, 3} (term 2, log offset 1000, ten entries after its noop, committed
    1000), peer 2 a slow follower (matched 1005), peer 3 up to date: MsgBeat sends two MsgHeartbeats, each with
    commit = min(committed, matched), no index and no log_term.  Then again with committed 1008, where the min bites."""
    offset = 1000
    c = _leader_columns(1)
    c.meta[0] = B.make_meta(0b111, self_slot=0)
    c.term[0], c.term_start[0], c.last_index[0], c.committed[0] = 2, offset + 1, offset + 11, offset
    c.matched[0, 0], c.matched[1, 0], c.matched[2, 0] = offset + 11, offset + 5, offset + 11
    ids = np.array([[1], [2], [3], [0], [0], [0], [0], [0], [1]], np.uint64)
    for committed in (offset, offset + 8):
        c.committed[0] = committed
        blob, offsets, totals = HF.bcast_heartbeats(c, None, 0, 1, ids)
        msgs = frames_of(blob, offsets)
        assert totals.tolist() == [2, len(blob), 0]
        want_commit = {2: min(committed, offset + 5), 3: min(committed, offset + 11)}
        assert [(g, s) for g, s, _ in msgs] == [(0, 1), (0, 2)]
        for _, _, m in msgs:
            assert m["msg_type"] == 8 and m["index"] == 0 and m["log_term"] == 0
            assert m["from"] == 1 and m["term"] == 2 and m["context"] == b""
            assert m["commit"] == want_commit[m["to"]]
    # a follower (no term range) sends nothing; a leader without a term sends nothing and is counted
    c.term_start[0] = R.NO_TERM_START
    assert HF.bcast_heartbeats(c, None, 0, 1, ids)[2].tolist() == [0, 0, 0]
    c.term_start[0], c.term[0] = offset + 1, 0
    assert HF.bcast_heartbeats(c, None, 0, 1, ids)[2].tolist() == [0, 0, 1]


class FramesDriver(R.OracleDriver):
    """The oracle driver, whose last_ctx also checks the heartbeat a MsgBeat would send: every frame of the group
    carries the 8 bytes of the last pending read id, or no context when nothing is pending."""

    def __init__(self, n, max_pending=8):
        super().__init__(n, max_pending)
        self.c.term[:] = 3
        self.ids = np.arange(1, 9 * n + 1, dtype=np.uint64).reshape(9, n)
        self.beats = 0

    def beat(self, g):
        """MsgBeat at group g through the oracle: the frames' contexts against ReadOnly::last_pending_request_ctx."""
        want = super().last_ctx(g)
        blob, offsets, totals = HF.bcast_heartbeats(self.c, self.q, g, 1, self.ids[:, g:g + 1])
        msgs = frames_of(blob, offsets)
        if self.c.term_start[g] != R.NO_TERM_START:
            meta = int(self.c.meta[g])
            peers = (meta | meta >> 8 | meta >> 16) & 0xFF
            if meta & B.META_HAS_SELF:
                peers &= ~(1 << (meta >> 24 & 7))
            assert len(msgs) == bin(peers).count("1")
        for grp, s, m in msgs:
            assert grp == g and m["context"] == (F.ctx_bytes(want) if want else b"")
            assert m["to"] == self.ids[s, g] and m["from"] == self.ids[8, g] and m["term"] == 3
        self.beats += len(msgs)
        return want

    def last_ctx(self, g):
        return self.beat(g)

    def request(self, r):
        out = super().request(r)
        for g in np.unique(r["group"]).tolist():
            if g < self.c.n_groups:
                self.beat(g)
        return out

    def ack(self, recs):
        out = super().ack(recs)
        for g in np.unique(recs["group"]).tolist():
            if g < self.c.n_groups:
                self.beat(g)
        return out


@pytest.mark.parametrize("case", R.REFERENCE_CASES, ids=lambda f: f.__name__)
def test_read_cases_heartbeat_context(case):
    d = FramesDriver(4)
    case(d)
    assert d.beats > 0


def test_one_broadcast_per_round_releases_what_one_per_request_does():
    """The reference broadcasts a heartbeat with each MsgReadIndex's ctx (raft.rs:2079).  Selecting the groups whose
    requests were QUEUED or DUP and sending one broadcast with the last pending ctx, answered by the same followers
    (each answers all or none of a round's heartbeats), releases exactly what the per-request heartbeats release for a
    group that had no read pending before the round.  With reads left from earlier rounds it releases a subset of what
    the per-request heartbeats followed by the reference's next MsgBeat (which carries the last pending ctx,
    raft.rs:876) release: an older entry's earlier acks are not combined with this round's."""
    rng = np.random.default_rng(0x5E1)
    n = 3000
    d = R.OracleDriver(n)
    d.q.control(d.c, d.votes, R.random_setup(rng, n, 0))
    d.c.term[:] = 2
    ids = np.arange(1, 9 * n + 1, dtype=np.uint64).reshape(9, n)

    def peers(g):
        meta = int(d.c.meta[g])
        p = (meta | meta >> 8 | meta >> 16) & 0xFF
        return p & ~(1 << (meta >> 24 & 7)) if meta & B.META_HAS_SELF else p

    released = fresh_checked = 0
    for rnd in range(4):
        reqs = R.random_requests(rng, n, 1.5, 30)
        fresh = d.q.count[:n] == 0
        q1 = d.q.copy()
        res, _ = d.q.request(d.c, reqs)
        q1.request(d.c, reqs)
        answering = rng.random((n, 8)) < 0.6
        sel_groups = np.unique(reqs["group"][np.isin(res, (B.READ_QUEUED, B.READ_DUP))]).astype(np.int64)
        # the reference: one heartbeat per QUEUED / DUP request, then a MsgBeat with the last pending ctx
        per_req = [(int(r["group"]), s, int(r["ctx"])) for r, x in zip(reqs, res) if x in (B.READ_QUEUED, B.READ_DUP)
                   for s in range(8) if peers(int(r["group"])) >> s & 1 and answering[r["group"], s]]
        want_a = q1.ack_seq(d.c, R.acks(*per_req)) if per_req else np.zeros(0, R.RO.READ_STATE_DTYPE)
        beat = [(int(g), s, q1.last_ctx(int(g))) for g in sel_groups for s in range(8)
                if peers(int(g)) >> s & 1 and answering[g, s] and q1.count[g]]
        want_b = q1.ack_seq(d.c, R.acks(*beat)) if beat else np.zeros(0, R.RO.READ_STATE_DTYPE)
        want = np.concatenate([np.asarray(want_a, R.RO.READ_STATE_DTYPE), np.asarray(want_b, R.RO.READ_STATE_DTYPE)])
        # one broadcast per round: the frames of the selected groups, answered by the same peers
        select = np.zeros((n + 31) // 32, np.uint32)
        np.bitwise_or.at(select, sel_groups // 32, np.left_shift(np.uint32(1), (sel_groups % 32).astype(np.uint32)))
        blob, offsets, _ = HF.bcast_heartbeats(d.c, d.q, 0, n, ids, select)
        rows = [(g, s, int.from_bytes(m["context"], "little")) for g, s, m in frames_of(blob, offsets) if answering[g, s]]
        assert {g for g, _, _ in rows} <= set(sel_groups.tolist())
        got = d.q.ack_seq(d.c, R.acks(*rows)) if rows else np.zeros(0, R.RO.READ_STATE_DTYPE)
        assert set(R.pairs(got)) <= set(R.pairs(want)), rnd
        assert len(R.pairs(got)) == len(set(R.pairs(got))), rnd
        a_fresh = [p for p in R.pairs(want_a) if fresh[p[0]]]
        got_fresh = [p for p in R.pairs(R.by_group(got)) if fresh[p[0]]]
        assert a_fresh == got_fresh, rnd
        released += len(got)
        fresh_checked += len(got_fresh)
    assert released > 500 and fresh_checked > 300
