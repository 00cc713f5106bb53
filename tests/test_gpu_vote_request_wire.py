"""Vote requests at a voter on the GPU (raftgpu_vote_request_wire[_device]) against the batch oracle
(oracle/vote_request_oracle.c): the reference's voter tables, every status, random 100K-group batches with joint
configurations, learners, wide pairs, leases and hostile frames, a 1M-group election storm through the resubmission
loop, the refusals and the host form's admission rule.  Run with -m gpu."""
import numpy as np
import pytest

from oracle import oracle as O
from oracle import read_oracle as RO
from oracle import vote_request_oracle as VR
from helpers import B, arena_of, votes, ARENA_COLUMNS
from control_cmds import cmds
import hb_frames as F
import pass_forms as PF
import vote_request_frames as Q

pytestmark = pytest.mark.gpu

def _columns(a, n):
    c = a.read_columns(n)
    return {k: getattr(c, k) for k in ARENA_COLUMNS} | {"term": a.column_read(B.COL_TERM, 0, 0, n, np.uint64)}


def _single(state):
    """An arena holding Q.one's group 0."""
    c, _, _, _ = state
    a = B.Arena(64)
    assert a.group_alloc_range(1) == 0
    meta = int(c.meta[0])
    a.control(cmds((B.CTL_SET_CONF, 0, 0, 0, (meta & 0xFF, 0, 0, int(c.last_index[0]) + 1)),
                   (B.CTL_RESET, 0, 0, 0, (int(c.term_start[0]), int(c.last_index[0]), int(c.committed[0]),
                                           int(c.last_index[0]))),
                   (B.CTL_SET_TERM, 0, 0, 0, (int(c.term[0]),))))
    return a


# --------------------------------------------------------------------------- 1. the reference's tables, both forms


def _table_rows():
    rows = [("recv", k) for k in range(len(Q.RECV_VOTE))] + [("voter", k) for k in range(len(Q.VOTER))]
    return rows + [("any", (r, t)) for r in (Q.FOLLOWER, Q.CANDIDATE, Q.PRE_CANDIDATE, Q.LEADER) for t in (Q.VOTE, Q.PRE_VOTE)]


def _table_case(kind, k):
    if kind == "recv":
        return Q.recv_vote_case(Q.RECV_VOTE[k])
    if kind == "voter":
        return Q.voter_case(Q.VOTER[k])
    return Q.any_state_case(*k)


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_reference_tables_match_the_oracle(device):
    for kind, k in _table_rows():
        state, frames = _table_case(kind, k)
        a = _single(state)
        c, vt, _, t = state
        blob, off = F.batch(frames)
        want = VR.batch(c, None, vt, blob, off, t)
        got = PF.run(a, "vote_request_wire", *F.batch(frames), t, device=device)
        for w, g, name in zip(want, got, ("status", "out", "bytes", "offsets", "totals")):
            assert np.array_equal(w, g), (kind, k, name, w, g)
        cols = _columns(a, 1)
        assert cols["term"][0] == c.term[0] and cols["term_start"][0] == c.term_start[0], (kind, k)
        a.close()


def test_statuses_in_order_match_the_oracle():
    for device in (False, True):
        a = B.Arena(64)
        assert a.group_alloc_range(6) == 0
        meta = B.make_meta(0b111, 0, 0, 0)
        a.control(cmds(*[(B.CTL_SET_CONF, g, 0, 0, (0b111, 0, 0, 11)) for g in range(6)],
                       *[(B.CTL_RESET, g, 0, 0, (9 if g == 2 else B.NO_TERM_START, 10, 8, 10)) for g in range(6)],
                       *[(B.CTL_SET_TERM, g, 0, 0, (0 if g == 3 else 5,)) for g in range(6)]))
        c = O.new_columns(16, 6)
        c.term_start[:] = B.NO_TERM_START
        c.meta[:6], c.term[:6], c.last_index[:6], c.committed[:6] = meta, [5, 5, 5, 0, 5, 5], 10, 8
        c.term_start[2] = 9
        t = np.zeros(6, VR.VOTER_DTYPE)
        t["id"], t["last_term"], t["flags"], t["commit_term"] = 1, 4, VR.SELECT, 3
        t["flags"][1], t["flags"][5] = 0, VR.SELECT | VR.LEADER | VR.LEASE
        frames = [F.frame(99, 0, Q.request(Q.VOTE, 6)), F.frame(0, 0, b"\x08"), F.frame(0, 0, Q.request(6, 6)),
                  F.frame(1, 0, Q.request(Q.VOTE, 6)), F.frame(2, 0, Q.request(Q.VOTE, 6)), F.frame(3, 0, Q.request(Q.VOTE, 6)),
                  F.frame(0, 0, Q.request(Q.VOTE, 0)), F.frame(0, 0, Q.request(Q.VOTE, 4)),
                  F.frame(0, 0, Q.request(Q.VOTE, 6, 4, 10, frm=2)), F.frame(4, 0, Q.request(Q.VOTE, 5, 3, 10, 9, 4, frm=2)),
                  F.frame(5, 0, Q.request(Q.PRE_VOTE, 6, 4, 10, frm=2)), F.frame(5, 0, Q.request(Q.PRE_VOTE, 6, 4, 10, frm=2)),
                  F.frame(1, 0, Q.request(Q.PRE_VOTE, 4, 4, 10, frm=3))]
        blob, off = F.batch(frames)
        want = VR.batch(c, None, np.zeros((O.SLOTS, c.cap), np.uint8), blob, off, t)
        got = PF.run(a, "vote_request_wire", *F.batch(frames), t, device=device)
        assert all(np.array_equal(w, g) for w, g in zip(want, got)), (device, want[0], got[0])
        assert (got[0] >> 4).tolist() == [B.WIRE_MALFORMED, B.WIRE_MALFORMED, B.WIRE_SKIP_TYPE, B.WIRE_ROLE, B.WIRE_ROLE,
                                          B.WIRE_TERM, B.WIRE_TERM, B.WIRE_IGNORED, B.WIRE_DUP, B.WIRE_COMMIT_VOTE,
                                          B.WIRE_IGNORED, B.WIRE_DUP, B.WIRE_ROLE]
        assert np.array_equal(_columns(a, 6)["term"], c.term[:6])
        a.close()


# --------------------------------------------------------------------------- 2. random 100K-group batches


@pytest.mark.parametrize("device,read_index", [(False, False), (True, False), (True, True)],
                         ids=["host", "device", "device-read-queues"])
def test_random_batches_vs_oracle(device, read_index):
    rng = np.random.default_rng(0x7200 + 2 * device + read_index)
    s = Q.Scenario(rng, 96_000, 2_000)
    a = arena_of(s, read_index)
    c, vt = Q.state_of(s)
    q = None
    if read_index:
        q = RO.ReadQueues(c.cap, 8)
        q.allocated[: s.n] = 1
    table = s.table.copy()
    kinds = np.zeros(16, np.int64)
    for rnd in range(2):
        frames = s.frames(rng)
        frames = [frames[i] for i in rng.permutation(len(frames))]
        blob, off = F.batch(frames)
        want = VR.batch(c, q, vt, blob, off, table)
        got = PF.run(a, "vote_request_wire", *F.batch(frames), table, device=device)
        for w, g, name in zip(want, got, ("status", "out", "bytes", "offsets", "totals")):
            assert np.array_equal(w, g), (rnd, name, np.flatnonzero(w != g)[:5] if w.shape == g.shape else (w.shape, g.shape))
        cols = _columns(a, s.n)
        for name in ARENA_COLUMNS + ("term",):
            assert np.array_equal(cols[name], getattr(c, name)[..., : s.n]), (rnd, name)
        assert np.array_equal(votes(a, s.n), vt[:, : s.n])
        if read_index:
            assert all(len(a.read_index_get(g)[0]) == q.count[g] for g in range(0, s.n, 997))
        Q.caller_update(table, s.role, got[0], got[1], frames)
        kinds += np.bincount(got[0] >> 4, minlength=16)
    for k in (B.WIRE_OK, B.WIRE_DUP, B.WIRE_ROLE, B.WIRE_TERM, B.WIRE_SKIP_TYPE, B.WIRE_MALFORMED, B.WIRE_COMMIT_VOTE,
              B.WIRE_IGNORED):
        assert kinds[k] > 100, (k, kinds)
    a.close()


# --------------------------------------------------------------------------- 3. the 1M-group storm


def test_1m_storm_pre_vote_then_vote_round():
    """1M five-voter groups at term 7: a pre-vote round (term 8, changes nothing the pass writes), then a vote round
    that bumps every term, with a second candidate's request for one group in eight resubmitted as DUP."""
    rng = np.random.default_rng(0x7201)
    n = 1_000_000
    a = B.Arena(n)
    assert a.group_alloc_range(n) == 0
    g = np.arange(n, dtype=np.uint32)
    last = rng.integers(10, 1 << 30, n).astype(np.uint64)
    com = last - rng.integers(0, 10, n).astype(np.uint64)
    setup = np.zeros(3 * n, B.CTL_CMD_DTYPE)
    setup["group"] = np.tile(g, 3)
    setup["op"][:n], setup["a"][:n, 0], setup["a"][:n, 3] = B.CTL_SET_CONF, 0x1F, last + 1
    setup["op"][n:2 * n] = B.CTL_RESET
    setup["a"][n:2 * n] = np.stack([np.full(n, B.NO_TERM_START, np.uint64), last, com, last], 1)
    setup["op"][2 * n:], setup["a"][2 * n:, 0] = B.CTL_SET_TERM, 7
    assert np.all(a.control(setup)["status"] == 0)
    c = O.new_columns(n, n)
    c.term_start[:] = B.NO_TERM_START
    vt = np.zeros((O.SLOTS, n), np.uint8)
    from oracle import control_oracle as CO
    CO.arena_control(c, vt, setup)
    table = Q.voters(n)
    table["id"], table["last_term"], table["persisted"], table["flags"] = 1, 7, last, B.VOTER_SELECT
    table["commit_term"] = 7
    for typ in (Q.PRE_VOTE, Q.VOTE):
        second = np.flatnonzero(rng.random(n) < 0.125).astype(np.uint32)
        gs = np.concatenate([g, second])
        e = np.zeros(len(gs), B.SYNTH_VOTE_REQUEST_DTYPE)
        e["hdr"], e["msg_type"], e["to"], e["from"] = gs << 4 | 1, typ, 1, rng.integers(2, 6, len(gs))
        e["term"], e["log_term"], e["index"] = 8, 7, last[gs] + rng.integers(0, 2, len(gs)).astype(np.uint64) - 1
        e = e[rng.permutation(len(e))]
        blob, off = B.synth_encode_vote_requests(e)
        pending_blob, pending_off, rounds = blob, off, 0
        while len(pending_off) > 1:
            want = VR.batch(c, None, vt, pending_blob, pending_off, table)
            got = PF.device(a, "vote_request_wire", pending_blob[: pending_off[-1]], pending_off, table)
            for w, gg, name in zip(want, got, ("status", "out", "bytes", "offsets", "totals")):
                assert np.array_equal(w, gg), (typ, rounds, name)
            st, out = got[0], got[1]
            voted = np.flatnonzero(st & B.VREQ_VOTED)
            at = pending_off[voted].astype(np.int64)
            hdr = sum(pending_blob[at + k].astype(np.uint32) << np.uint32(8 * k) for k in range(4))
            table["vote"][hdr >> 4] = out[voted, 0]
            dup = np.flatnonzero(st >> 4 == B.WIRE_DUP)
            frames = [pending_blob[pending_off[i]:pending_off[i + 1]].tobytes() for i in dup]
            pending_blob, pending_off = F.batch(frames) if frames else (np.zeros(0, np.uint8), np.zeros(1, np.uint32))
            rounds += 1
        assert rounds == 2
    assert np.all(_columns(a, n)["term"] == 8) and np.all(c.term[:n] == 8)
    cols = _columns(a, n)
    for name in ARENA_COLUMNS:
        assert np.array_equal(cols[name], getattr(c, name)[..., :n]), name
    a.close()


# --------------------------------------------------------------------------- 4. refusals and admission


def test_refusals_before_any_launch():
    a = B.Arena(64)
    assert a.group_alloc_range(16) == 0
    a.control(cmds(*[(B.CTL_SET_CONF, g, 0, 0, (0x7, 0, 0, 11)) for g in range(16)],
                   *[(B.CTL_SET_TERM, g, 0, 0, (3,)) for g in range(16)]))
    L, h = a._L, a._h
    n = 16
    blob, off = F.batch([F.frame(g, 0, Q.request(Q.VOTE, 4, frm=2)) for g in range(n)])
    blob = np.concatenate([blob, np.zeros(16, np.uint8)])
    t = Q.voters(64)
    t["flags"] = B.VOTER_SELECT
    bound = B.vote_request_wire_bound(n)
    nb = off[-1]
    with PF.refusals(a, "vote_request_wire", blob, off, t, n_bytes=nb) as r:
        dev, d = r.call, r.args
        refused = [dev(cap=bound - 1), dev(b=d["b"] + 4), dev(v=d["v"] + 8), dev(rb=d["rb"] + 4), dev(nb=1 << 32),
                   dev(n=1 << 32, cap=1 << 40), dev(n=(1 << 26) + 1, cap=1 << 40), dev(v=None), dev(st=None), dev(b=None),
                   dev(o=None), dev(rb=None), dev(t=None), dev(ro=None)]
        assert refused == [B.ERR_INVALID] * len(refused), refused
        assert r.untouched()                                                  # nothing was launched
        assert np.all(a.column_read(B.COL_TERM, 0, 0, 16, np.uint64) == 3)
        st, out, rb, ro, tot = np.zeros(n, np.uint8), np.zeros(2 * n, np.uint64), np.zeros(bound, np.uint8), \
            np.zeros(n + 1, np.uint32), np.zeros(2, np.uint64)
        assert L.raftgpu_vote_request_wire(h, blob.ctypes.data, nb, off.ctypes.data, n, t.ctypes.data, st.ctypes.data,
                                           out.ctypes.data, rb.ctypes.data, bound - 1, ro.ctypes.data, tot.ctypes.data) == B.ERR_INVALID
        assert L.raftgpu_vote_request_wire(h, blob.ctypes.data, nb, off.ctypes.data, n, None, st.ctypes.data,
                                           out.ctypes.data, rb.ctypes.data, bound, ro.ctypes.data, tot.ctypes.data) == B.ERR_INVALID
        assert dev() == B.OK                                                      # the same call with every rule kept
        gt = r.read("t", np.zeros(2, np.uint64))
        assert gt.tolist()[0] == n and np.all(a.column_read(B.COL_TERM, 0, 0, 16, np.uint64) == 4)
    a.close()


def test_host_form_refuses_while_records_are_enqueued():
    a = B.Arena(64)
    assert a.group_alloc_range(4) == 0
    a.control(cmds(*[(B.CTL_SET_CONF, g, 0, 0, (0x7, 0, 0, 11)) for g in range(4)],
                   *[(B.CTL_SET_TERM, g, 0, 0, (3,)) for g in range(4)]))
    rec = np.zeros(1, B.APPEND_RESP_DTYPE)
    rec["group"], rec["peer_slot"], rec["index"] = 0, 1, 1
    a.enqueue(rec)
    t = Q.voters(4)
    t["flags"] = B.VOTER_SELECT
    frames = F.Frames([F.frame(g, 0, Q.request(Q.VOTE, 4, frm=2)) for g in range(4)])
    n = frames.n
    st, out = np.full(n, 0xEE, np.uint8), np.full(2 * n, 7, np.uint64)
    rb, ro, tot = np.zeros(64 * n, np.uint8), np.full(n + 1, 9, np.uint32), np.full(2, 9, np.uint64)
    rc = a._L.raftgpu_vote_request_wire(a._h, frames.bytes.ctypes.data, frames.n_bytes, frames.offsets.ctypes.data, n,
                                        t.ctypes.data, st.ctypes.data, out.ctypes.data, rb.ctypes.data, len(rb),
                                        ro.ctypes.data, tot.ctypes.data)
    assert rc == B.ERR_BUSY
    assert np.all(st == 0xEE) and np.all(out == 7) and tot.tolist() == [0, 0] and ro[0] == 0   # written before admission
    assert np.all(a.column_read(B.COL_TERM, 0, 0, 4, np.uint64) == 3)
    a.close()
