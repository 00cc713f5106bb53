"""ReadIndex (ReadOnlyOption::Safe) on the CPU oracle (oracle/read_oracle.c): the reference's read-only tests restated
at the tracker level, the device form's edge cases, the claim that a batch of acks can be applied as OR-every-ack-
then-advance (DESIGN.md 3.9), and the C layout of the request and released-read structs."""
import os
import sys

import numpy as np
import pytest

from oracle import read_oracle as RO
from helpers import B
import read_cases as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("case", R.REFERENCE_CASES, ids=lambda f: f.__name__)
def test_reference_read_only_cases(case):
    case(R.OracleDriver(4))


def test_edge_cases():
    R.edge_cases(R.OracleDriver(2, max_pending=4), 2)


def _random_world(rng, n_narrow, n_wide, P):
    d = R.OracleDriver(n_narrow + 2 * n_wide, max_pending=P)
    for k in range(n_wide):
        lo = n_narrow + 2 * k
        d.c.meta[lo], d.c.meta[lo + 1] = R.META_WIDE_LO, R.META_WIDE_HI
    d.q.control(d.c, d.votes, R.random_setup(rng, n_narrow, n_wide))
    n = n_narrow + 2 * n_wide
    for _ in range(3):   # fill the queues: several requests per group, duplicates and full queues among them
        d.q.request(d.c, R.random_requests(rng, n, 2.0, 12))
    return d, n


@pytest.mark.parametrize("seed", range(6))
def test_ack_batches_are_order_independent(seed):
    """Random queues and ack batches: every permutation of a batch applied one response at a time (the reference's
    handle_heartbeat_response) gives the same final queues and the same per-group release lists as OR-every-ack-
    then-advance-to-the-last-quorum, which is what the device computes."""
    rng = np.random.default_rng(1000 + seed)
    d, n = _random_world(rng, 120, 8, 4 + seed % 5)
    wide_hi = (d.c.meta[:d.c.cap] & R.META_WIDE_HI) != 0
    assert d.q.count[:n].sum() > 100
    for _ in range(4):
        recs = R.random_acks(rng, d.q, d.c.meta, n, 600, wide_hi)
        qb = d.q.copy()
        want = R.by_group(qb.ack_batch(d.c, recs))
        want_q = R.oracle_queue_view(qb, n)
        for _ in range(12):
            qs = d.q.copy()
            got = R.by_group(qs.ack_seq(d.c, recs[rng.permutation(len(recs))]))
            assert np.array_equal(got, want)
            for a, b in zip(R.oracle_queue_view(qs, n), want_q):
                assert np.array_equal(a, b)
        d.q = qb
        assert len(want) > 0


def test_read_layouts_match_the_header():
    sys.path.insert(0, os.path.join(ROOT, "scripts"))
    import gen_rust_stub as G
    lay = G.struct_layouts()
    for name, dt in (("raftgpu_read_req", B.READ_REQ_DTYPE), ("raftgpu_read_state", B.READ_STATE_DTYPE)):
        size, offs = lay[name]
        assert size == dt.itemsize, name
        assert [(f, o) for f, o, _ in offs] == [(f, dt.fields[f][1]) for f in dt.names], name
    assert lay["raftgpu_read_req"][0] == 16 and lay["raftgpu_read_state"][0] == 24
    assert RO.READ_REQ_DTYPE == B.READ_REQ_DTYPE and RO.READ_STATE_DTYPE == B.READ_STATE_DTYPE
    consts, _, _, _ = G.parse_header()
    read = {n[len("RAFTGPU_READ_"):]: v for n, v, _ in consts if n.startswith("RAFTGPU_READ_")}
    assert read == {n[len("READ_"):]: getattr(B, n) for n in dir(B) if n.startswith("READ_") and n[5:] in read}
    assert {k: v for k, v in read.items() if k != "MAX_PENDING"} == {
        "QUEUED": RO.QUEUED, "READY": RO.READY, "DUP": RO.DUP, "DROPPED": RO.DROPPED, "FULL": RO.FULL,
        "NO_GROUP": RO.NO_GROUP, "NO_CTX": RO.NO_CTX}
    rec = {n: v for n, v, _ in consts if n.startswith("RAFTGPU_REC_")}
    assert rec["RAFTGPU_REC_READ_CTX"] == B.REC_READ_CTX == RO.REC_READ_CTX
    assert rec["RAFTGPU_REC_HEARTBEAT"] == RO.REC_HEARTBEAT
