"""The follower heartbeat oracle (oracle/hb_follow_oracle.c): its encoder against python-protobuf's bytes
(tests/golden/wire/heartbeat_follow.json, scripts/gen_wire_hb_follow_golden.py), test_handle_heartbeat restated, every
status reached by a crafted frame that changes nothing, and the round trip leader -> followers -> leader on the
oracles alone."""
import json
import os

import numpy as np

from oracle import hb_follow_oracle as HL
from oracle import hb_frames_oracle as HF
from oracle import hb_wire_oracle as H
from helpers import B, O
import hb_follow as FL
import hb_frames as F
import read_cases as R

HERE = os.path.dirname(os.path.abspath(__file__))
U64 = (1 << 64) - 1
OK_RESP = B.WIRE_OK << 4 | B.RES_OK


def vectors():
    with open(os.path.join(HERE, "golden", "wire", "heartbeat_follow.json")) as f:
        return json.load(f)["vectors"]


def test_golden_vectors_encode_byte_for_byte():
    vs = vectors()
    for v in vs:
        ctx = None if v["ctx"] is None else bytes.fromhex(v["ctx"])
        got = HL.encode_response(v["to"], v["from"], v["term"], v["commit"], ctx)
        assert got.hex() == v["hex"], v
        assert len(got) <= 56
    for name in ("to", "from", "term", "commit"):  # the coverage the vectors promise
        assert {0, 1, 127, 128, 1 << 32, 1 << 63, U64} <= {v[name] for v in vs}, name
    ctxs = {v["ctx"] for v in vs}
    assert {None, "00" * 8, "01" + "00" * 7, "ff" * 8} <= ctxs


def _followers(n, cap=None):
    """n follower groups: term 2, log [1, 3], committed 2, ids 1..n, all selected."""
    c = O.new_columns(cap or n + 8, n)
    c.term_start[:] = R.NO_TERM_START
    c.term[:n], c.last_index[:n], c.committed[:n] = 2, 3, 2
    return c, np.arange(1, c.cap + 1, dtype=np.uint64), FL.bitmap(np.ones(c.cap, bool))


def _run(c, frames, ids, select, q=None):
    blob, off = F.batch(frames)
    return HL.follower_heartbeats(c, q, blob, off, select, ids)


def test_handle_heartbeat():
    """test_raft.rs:1350-1394: a follower at committed 2 (log up to 3) commits up to m.commit and never down, and sends
    exactly one MsgHeartbeatResponse."""
    for m_commit, w_commit in ((3, 3), (1, 2)):
        c, ids, sel = _followers(1)
        st, frm, blob, off, tot = _run(c, [F.frame(0, 5, F.message(8, term=2, commit=m_commit, frm=2))], ids, sel)
        assert st.tolist() == [OK_RESP] and frm.tolist() == [2]
        assert int(c.committed[0]) == w_commit
        assert tot.tolist() == [1, len(blob)]
        (hdr, body), = FL.frames_of(blob, off)
        assert hdr == 0 << 4 | 5
        m = H.decode_message(body)
        assert (m["msg_type"], m["to"], m["from"], m["term"], m["commit"], m["context"]) == (9, 2, 1, 2, w_commit, b"")


def _crafted(c):
    """(frame, status) pairs, each frame failing exactly one check; groups 0-5 follow, 6 leads, 7 has no term, 8-9 are
    a wide pair, 10 is not selected."""
    hb = lambda g, **k: F.frame(g, 3, F.message(8, **{"term": 2, "commit": 2, "frm": 9, **k}))
    return [
        (b"\x01\x00", B.WIRE_MALFORMED),                                      # shorter than the header
        (F.frame(1, 0, b"\x08"), B.WIRE_MALFORMED),                           # a truncated varint
        (hb(c.n_groups), B.WIRE_MALFORMED),                                   # no such group
        (hb(9), B.WIRE_MALFORMED),                                            # a wide pair's high half
        (F.frame(1, 0, F.message(9, term=2, commit=2)), B.WIRE_SKIP_TYPE),    # a MsgHeartbeatResponse
        (F.frame(1, 0, F.message(3, term=2, index=1)), B.WIRE_SKIP_TYPE),     # a MsgAppend
        (hb(6), B.WIRE_ROLE),                                                 # a leader
        (hb(10), B.WIRE_ROLE),                                                # not selected
        (hb(7), B.WIRE_TERM),                                                 # the group has no term
        (hb(2, term=3), B.WIRE_TERM),                                         # a higher term: become_follower
        (hb(2, term=1), B.WIRE_TERM),                                         # a lower one
        (hb(2, term=0), B.WIRE_TERM),                                         # a local message
        (hb(3, context=b"abcd"), B.WIRE_CONTEXT),                             # not 8 bytes
        (hb(4, commit=4), B.WIRE_COMMIT_RANGE),                               # past last_index 3: fatal!
        (hb(8, commit=6), B.WIRE_COMMIT_RANGE),                               # past both halves of the pair
    ]


def _crafted_arena():
    c, ids, sel = _followers(12)
    c.term_start[6] = 1
    c.term[7] = 0
    c.meta[8], c.meta[9] = R.META_WIDE_LO, R.META_WIDE_HI
    c.last_index[9], c.committed[9] = 5, 4                                    # the pair's top is 5
    sel = FL.bitmap(np.arange(c.cap) != 10)
    return c, ids, sel


def test_every_status_changes_nothing():
    c, ids, sel = _crafted_arena()
    cases = _crafted(c)
    before = FL.state(c, c.cap)
    for frame, want in cases:
        st, frm, blob, off, tot = _run(c, [frame], ids, sel)
        assert st.tolist() == [want << 4] and frm.tolist() == [0], (frame, st)
        assert tot.tolist() == [0, 0] and len(blob) == 0 and off.tolist() == [0]
        assert FL.same_state(FL.state(c, c.cap), before), frame
    st, _, _, _, tot = _run(c, [f for f, _ in cases], ids, sel)                # all at once
    assert st.tolist() == [w << 4 for _, w in cases] and tot.tolist() == [0, 0]
    assert FL.same_state(FL.state(c, c.cap), before)
    # an unallocated group is malformed where read queues say which groups exist
    q = R.RO.ReadQueues(c.cap, 4)
    q.allocated[:12] = 1
    q.allocated[5] = 0
    st, _, _, _, _ = _run(c, [F.frame(5, 0, F.message(8, term=2, commit=2))], ids, sel, q)
    assert st.tolist() == [B.WIRE_MALFORMED << 4]
    assert FL.same_state(FL.state(c, c.cap), before)


def test_dup_and_wide_pairs():
    """The first passing frame of a group is applied, a later one is DUP and changes nothing -- even one that would
    have moved committed further; a frame that fails an earlier check does not count as the first.  A wide pair
    commits on both halves."""
    c, ids, sel = _crafted_arena()
    frames = [F.frame(2, 1, F.message(8, term=3, commit=3)),                   # TERM: not the group's first
              F.frame(2, 2, F.message(8, term=2, commit=2, frm=4)),           # applied: committed stays 2
              F.frame(2, 3, F.message(8, term=2, commit=3, frm=5)),           # DUP
              F.frame(8, 4, F.message(8, term=2, commit=5, frm=6, context=F.ctx_bytes(0)))]
    st, frm, blob, off, tot = _run(c, frames, ids, sel)
    assert st.tolist() == [B.WIRE_TERM << 4, OK_RESP, B.WIRE_DUP << 4, OK_RESP]
    assert frm.tolist() == [0, 4, 0, 6]
    assert int(c.committed[2]) == 2 and c.committed[8:10].tolist() == [5, 5] and c.last_index[8:10].tolist() == [5, 5]
    got = [(h, H.decode_message(b)) for h, b in FL.frames_of(blob, off)]
    assert [h for h, _ in got] == [2 << 4 | 2, 8 << 4 | 4]
    assert [(m["to"], m["from"], m["commit"], m["context"]) for _, m in got] == [(4, 3, 2, b""), (6, 9, 5, bytes(8))]


def _leaders(rng, n):
    """n leader groups of the oracle with random configurations, terms, commits and read queues."""
    d = R.OracleDriver(n, max_pending=4)
    setup = R.random_setup(rng, n, 0)
    d.q.control(d.c, d.votes, setup)
    d.c.term[:n] = rng.integers(1, 1 << 20, n)
    d.c.matched[:, :n] = rng.integers(0, 90, (O.SLOTS, n))                    # (the heartbeats' commit is min(matched, committed))
    reqs = R.random_requests(rng, n, 0.8, 1 << 40)
    d.q.request(d.c, reqs)
    return d


def test_round_trip_on_the_oracles():
    """hfo_bcast_heartbeats -> the transport (leader cell (g, s) <-> follower group 8 g + s, x = s) -> the follower
    oracle -> the transport back -> hwo_apply: every response carries the follower's max(committed, m.commit) and the
    heartbeat's context, and the leader applies all of them."""
    rng = np.random.default_rng(0x4EF1)
    n = 400
    d = _leaders(rng, n)
    ids = rng.integers(1, 1 << 63, (9, n), dtype=np.uint64)
    hb, hoff, htot = HF.bcast_heartbeats(d.c, d.q, 0, n, ids)
    assert int(htot[0]) > 500
    lh = FL.headers(hb, hoff)
    fg = (lh >> 4) * 8 + (lh & 15)                                             # the follower of each frame
    fol = O.new_columns(8 * n + 8, 8 * n)
    fol.term_start[:] = R.NO_TERM_START
    fol.term[fg] = d.c.term[lh >> 4]
    fol.last_index[:] = rng.integers(0, 80, fol.cap)
    fol.committed[:] = np.minimum(fol.last_index, rng.integers(0, 80, fol.cap))
    before = fol.committed.copy()
    self_ids = ids[lh & 15, lh >> 4]
    fids = np.zeros(fol.cap, np.uint64)
    fids[fg] = self_ids
    blob = FL.with_headers(hb, hoff, fg.astype(np.uint32) << 4 | (lh & 15))
    st, frm, rb, ro, rt = HL.follower_heartbeats(fol, None, blob, hoff, FL.bitmap(np.ones(fol.cap, bool)), fids)
    bodies = [H.decode_message(b) for _, b in FL.frames_of(hb, hoff)]
    commits = np.array([m["commit"] for m in bodies], np.uint64)
    top = np.maximum(before[fg], fol.last_index[fg])
    want_st = np.where(commits > top, B.WIRE_COMMIT_RANGE << 4, OK_RESP)
    assert np.array_equal(st, want_st) and (st == OK_RESP).sum() > 300 and (st != OK_RESP).sum() > 10
    ok = st == OK_RESP
    assert np.array_equal(frm[ok], ids[8, lh >> 4][ok])                        # m.from = the leader's id
    resp = FL.frames_of(rb, ro)
    assert len(resp) == ok.sum() == int(rt[0])
    for k, (i, (h, body)) in enumerate(zip(np.flatnonzero(ok), resp)):
        m = H.decode_message(body)
        assert h == int(fg[i]) << 4 | int(lh[i] & 15)
        assert m["commit"] == max(int(before[fg[i]]), int(commits[i])) == int(fol.committed[fg[i]])
        assert m["context"] == bodies[i]["context"] and m["to"] == bodies[i]["from"] and m["from"] == int(self_ids[i])
    back = FL.with_headers(rb, ro, FL.headers(rb, ro) // 128 << 4 | (FL.headers(rb, ro) & 15))
    wst, rel = H.apply(d.c, d.q, back, ro, d.c.term)
    assert np.all((wst >> 4) == B.WIRE_OK) and len(rel) > 0
