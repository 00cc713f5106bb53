"""The heartbeat-response wire oracle (oracle/hb_wire_oracle.c): its decode against python-protobuf's verdicts
(tests/golden/wire/heartbeat_responses.json, scripts/gen_wire_hb_golden.py), the status rules, and that frames built
from records and applied give exactly what the record form gives (ro_arena_apply_heartbeat + ro_read_ack_seq)."""
import json
import os

import numpy as np
import pytest

from oracle import hb_wire_oracle as H
from oracle import read_oracle as RO
from helpers import B, O
import hb_frames as F
import read_cases as R

HERE = os.path.dirname(os.path.abspath(__file__))


def vectors():
    with open(os.path.join(HERE, "golden", "wire", "heartbeat_responses.json")) as f:
        return json.load(f)["vectors"]


def test_golden_vectors_decode_to_python_protobufs_fields_and_context():
    kinds, lens = set(), set()
    for v in vectors():
        got = H.decode_message(bytes.fromhex(v["hex"]))
        if not v["ok"]:
            assert got is None, (v["kind"], v["hex"])
            continue
        assert got is not None, (v["kind"], v["hex"])
        want = dict(v["fields"], context=bytes.fromhex(v["context"]))
        assert got == want, (v["kind"], v["hex"], got, want)
        kinds.add(v["kind"])
        lens.add(len(want["context"]))
    assert {"canonical", "repeated_context", "context_varint", "unknown_fields", "other_type", "truncated"} <= kinds
    assert {0, 8} < lens
    ids = {int.from_bytes(bytes.fromhex(v["context"]), "little") for v in vectors() if v["ok"] and len(v["context"]) == 16}
    assert {0, 1, (1 << 64) - 1} <= ids


def _one_group(read_queues=True):
    """Group 0: leader over voters {0, 1, 2} (self 0), term 5, one pending read with id 77."""
    d = R.OracleDriver(4)
    R.leader(d, 0, 0b111)
    assert d.request(R.reqs((0, 77)))[0].tolist() == [B.READ_QUEUED]
    terms = np.zeros(d.c.cap, np.uint64)
    terms[0] = 5
    return d, terms, (d.q if read_queues else None)


CTX77 = F.ctx_bytes(77)


@pytest.mark.parametrize("frames,reads,want", [
    # (group, slot, body) rows -> the status high nibbles
    ([(0, 1, F.message(9, term=5))], True, [B.WIRE_OK]),
    ([(0, 1, F.message(9, term=5, context=CTX77))], True, [B.WIRE_OK]),
    ([(0, 1, F.message(9, term=5, context=CTX77))], False, [B.WIRE_CONTEXT]),
    ([(0, 1, F.message(9, term=5))], False, [B.WIRE_OK]),
    ([(0, 1, F.message(9, term=5, context=b"\x01" * 7))], True, [B.WIRE_CONTEXT]),
    ([(0, 1, F.message(9, term=5, context=b"\x01" * 9))], True, [B.WIRE_CONTEXT]),
    ([(0, 1, F.message(9, term=6, context=b"\x01" * 9))], True, [B.WIRE_TERM]),     # the term rule comes first
    ([(0, 1, F.message(9, term=4, context=CTX77))], True, [B.WIRE_TERM]),
    ([(1, 1, F.message(9, term=9))], True, [B.WIRE_OK]),                               # group 1: term not checked
    ([(0, 1, F.message(4, term=5, index=1))], True, [B.WIRE_SKIP_TYPE]),               # MsgAppendResponse
    ([(0, 1, F.message(8, term=5, context=CTX77))], True, [B.WIRE_SKIP_TYPE]),         # MsgHeartbeat
    ([(0, 1, F.message(9, term=5) + b"\x08")], True, [B.WIRE_MALFORMED]),
    ([(4, 1, F.message(9))], True, [B.WIRE_MALFORMED]),                                # no such group
    ([(0, 1, F.message(9, term=5)), (0, 1, F.message(9, term=5, context=CTX77))], True, [B.WIRE_OK, B.WIRE_DUP]),
    # a frame that is not applied does not take its cell
    ([(0, 1, F.message(9, term=5, context=b"xy")), (0, 1, F.message(9, term=5))], True, [B.WIRE_CONTEXT, B.WIRE_OK]),
    ([(0, 1, F.message(9, term=4)), (0, 1, F.message(9, term=5))], True, [B.WIRE_TERM, B.WIRE_OK]),
    ([(0, 9, F.message(9, term=5)), (0, 9, F.message(9, term=5))], True, [B.WIRE_OK, B.WIRE_OK]),   # no slot 9
])
def test_status_rules(frames, reads, want):
    d, terms, q = _one_group(reads)
    blob, off = F.batch([F.frame(g, s, b) for g, s, b in frames])
    status, _ = H.decode_batch(blob, off, d.c.n_groups, terms, read_queues=reads)
    assert status.tolist() == want
    before = O.copy_columns(d.c)
    st, rel = H.apply(d.c, q, blob, off, terms)
    assert (st >> 4).tolist() == want
    applied = (st >> 4) == B.WIRE_OK
    if not applied.any():                                    # nothing applied: the tracker is untouched
        for name in ("pflags", "peer_committed"):
            assert np.array_equal(getattr(d.c, name), getattr(before, name))


def test_context_acks_and_releases():
    d, terms, q = _one_group()
    blob, off = F.batch([F.frame(0, 1, F.message(9, term=5, commit=1, context=F.ctx_bytes(0))),
                         F.frame(0, 3, F.message(9, term=5, context=CTX77)),        # no Progress: ignored
                         F.frame(0, 2, F.message(9, term=5, commit=1, context=CTX77))])
    st, rel = H.apply(d.c, q, blob, off, terms)
    assert st.tolist() == [B.RES_OK | B.RES_SEND, B.RES_NO_PROGRESS, B.RES_OK | B.RES_SEND]   # matched 0 < last_index 1
    assert R.pairs(rel) == [(0, 77, 1)] and q.count[0] == 0


def test_frames_equal_records():
    """Random heartbeat records (one per cell, shuffled, ids pending or not, some without a context) on groups of
    every configuration: encoded as frames and applied by the oracle, they leave the same columns, results and
    released reads as the records through ro_arena_apply_heartbeat + ro_read_ack_seq."""
    rng = np.random.default_rng(0xF2A)
    n_narrow, n_wide = 3000, 100
    n = n_narrow + 2 * n_wide
    d = R.OracleDriver(n)
    for k in range(n_wide):
        lo = n_narrow + 2 * k
        d.c.meta[lo], d.c.meta[lo + 1] = R.META_WIDE_LO, R.META_WIDE_HI
    d.q.control(d.c, d.votes, R.random_setup(rng, n_narrow, n_wide))
    d.q.request(d.c, R.random_requests(rng, n, 3.0, 40))
    wide_hi = (d.c.meta[: d.c.cap] & R.META_WIDE_HI) != 0
    for rnd in range(3):
        cells = rng.choice(8 * n, 3 * n, replace=False)
        recs = np.zeros(len(cells), B.APPEND_RESP_DTYPE)
        recs["group"], recs["peer_slot"] = cells % n, cells // n
        recs["flags"] = B.REC_HEARTBEAT | B.REC_READ_CTX
        g = recs["group"]
        qg = np.where(wide_hi[g], g - 1, g)
        cnt = d.q.count[qg].astype(np.int64)
        pick = rng.integers(0, np.maximum(cnt, 1))
        recs["index"] = np.where(cnt > 0, d.q.ctx[qg, np.minimum(pick, d.q.max_pending - 1)], rng.integers(1, 50, len(g)))
        recs["index"][rng.random(len(g)) < 0.1] = 0
        recs["commit"] = rng.integers(0, 70, len(g))
        recs = recs[rng.permutation(len(recs))]
        ref, q2 = O.copy_columns(d.c), d.q.copy()
        want_res = O.arena_apply_heartbeat(ref, recs)
        want_rel = q2.ack_seq(ref, recs)
        frames = [F.frame(int(r["group"]), int(r["peer_slot"]),
                          F.message(9, commit=int(r["commit"]), context=F.ctx_bytes(int(r["index"])) if r["index"] else None))
                  for r in recs]
        blob, off = F.batch(frames)
        st, rel = H.apply(d.c, d.q, blob, off, None)
        assert np.array_equal(st, want_res), rnd
        assert np.array_equal(R.by_group(rel), R.by_group(want_rel)), rnd
        assert len(rel) > 100, rnd
        for name in ("pflags", "peer_committed", "matched", "next_idx"):
            assert np.array_equal(getattr(d.c, name), getattr(ref, name)), (rnd, name)
        for name in ("count", "ctx", "index", "acks"):
            assert np.array_equal(getattr(d.q, name), getattr(q2, name)), (rnd, name)
    assert RO.READ_STATE_DTYPE.itemsize == 24
