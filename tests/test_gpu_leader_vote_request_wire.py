"""Vote requests at a leader on the GPU (raftgpu_leader_vote_request_wire[_device]) against the batch oracle
(oracle/leader_vote_request_oracle.c), byte for byte: the reference's cases at a leader, every status, random
100K-group bursts with wide pairs, read queues and hostile frames through the resubmission loop, 1M leaders in the
three bursts a store sees, the refusals, and one partition-heal buffer through the leader-side passes in the documented
order.  Run with -m gpu."""
import numpy as np
import pytest

from oracle import oracle as O
from oracle import control_oracle as CO
from oracle import leader_term_oracle as LT
from oracle import leader_vote_request_oracle as LV
from oracle import read_oracle as RO
from helpers import B, arena_of, check_columns
from control_cmds import cmds
import hb_frames as F
import leader_term as L
import leader_vote_request as LQ
import pass_forms as PF
import vote_request_frames as Q

pytestmark = pytest.mark.gpu


def _small(state):
    """An arena holding Q.one's group 0."""
    c = state[0]
    a = B.Arena(64)
    assert a.group_alloc_range(1) == 0
    a.control(cmds((B.CTL_SET_CONF, 0, 0, 0, (int(c.meta[0]) & 0xFF, 0, 0, int(c.last_index[0]) + 1)),
                   (B.CTL_RESET, 0, 0, 0, (int(c.term_start[0]), int(c.last_index[0]), int(c.committed[0]),
                                           int(c.last_index[0]))),
                   (B.CTL_SET_TERM, 0, 0, 0, (int(c.term[0]),))))
    return a


# --------------------------------------------------------------------------- 1. the reference's cases, both forms


def _cases():
    out = [Q.any_state_case(Q.LEADER, t) for t in (Q.VOTE, Q.PRE_VOTE)]
    out += [Q.recv_vote_case(r) for r in Q.RECV_VOTE if r[0] == Q.LEADER]
    for typ in (Q.VOTE, Q.PRE_VOTE):
        for ctx in (b"", Q.ELECTION, Q.TRANSFER):
            out.append((Q.one(Q.LEADER, 2, 1, 1, 2, leader=True, lease=True, voters=0b111),
                        [F.frame(0, 0, Q.request(typ, 3, 2, 1, context=ctx, frm=3))]))
    return out


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_reference_cases_match_the_oracle(device):
    for k, (state, frames_) in enumerate(_cases()):
        a = _small(state)
        c, vt, _, t = state
        blob, off = F.batch(frames_)
        want = LV.batch(c, None, vt, blob, off, t)
        got = PF.run(a, "leader_vote_request_wire", blob, off, t, device=device)
        PF.equal(want, got, LQ.NAMES, k)
        assert a.column_read(B.COL_TERM, 0, 0, 1, np.uint64)[0] == c.term[0], k
        assert a.read_columns(1).term_start[0] == c.term_start[0], k
        a.close()


# --------------------------------------------------------------------------- 2. random bursts through the loop


def _device_passes(a, device):
    return (lambda blob, off, t: PF.run(a, "leader_vote_request_wire", blob, off, t, device=device),
            lambda blob, off, t: PF.run(a, "vote_request_wire", blob, off, t, device=device))


def _checked(passes, oracles, state):
    """Each pass call runs the device pass and its oracle on the same batch and compares them byte for byte."""
    a, c, vt, n = state

    def wrap(dev, orc, name):
        def run(blob, off, t):
            want, got = orc(blob, off, t), dev(blob, off, t)
            PF.equal(want, got, LQ.NAMES, name)
            check_columns(a, c, vt, n)
            return got
        return run
    return [wrap(d, o, nm) for d, o, nm in zip(passes, oracles, ("leader", "voter"))]


@pytest.mark.parametrize("device,read_index", [(False, False), (True, False), (True, True)],
                         ids=["host", "device", "device-read-queues"])
def test_random_bursts_vs_oracle(device, read_index):
    """100K leaders (96K narrow, 2K wide pairs) with 1-4 vote requests each and hostile frames: every round of the
    resubmission loop -- this pass, then raftgpu_vote_request_wire on the deposed groups' frames -- byte for byte
    against the batch oracles, with every arena column after each call."""
    rng = np.random.default_rng(0x7600 + 2 * device + read_index)
    s = LQ.scenario(rng, 96_000, 2_000, p_check_quorum=0.0)
    a = arena_of(s, read_index)
    c, vt = Q.state_of(s)
    q = None
    if read_index:
        q = RO.ReadQueues(c.cap, 8)
        q.allocated[: s.n] = 1
    table, role = s.table.copy(), s.role.copy()
    passes = _checked(_device_passes(a, device), LQ.oracle_passes(c, q, vt), (a, c, vt, s.n))
    # one call with requests whose commit is ahead (COMMIT_VOTE: the host would step them), then the loop without
    frames_ = s.frames(rng, per_group=(1, 4))
    frames_ = [frames_[i] for i in rng.permutation(len(frames_))]
    first = passes[0](*F.batch(frames_), table)
    LQ.host_side(table, role, first[0], first[1], frames_)
    frames_ = s.frames(rng, per_group=(1, 4), commit_vote=False)
    frames_ = [frames_[i] for i in rng.permutation(len(frames_))]
    _, rounds, kinds = LQ.settle(c, q, vt, role, table, frames_, *passes)
    kinds[0] += np.bincount(first[0] >> 4, minlength=16)
    assert rounds > 2 and kinds[0][B.WIRE_COMMIT_VOTE] + kinds[1][B.WIRE_COMMIT_VOTE] == np.count_nonzero(
        first[0] >> 4 == B.WIRE_COMMIT_VOTE)
    for k in (B.WIRE_OK, B.WIRE_DUP, B.WIRE_ROLE, B.WIRE_TERM, B.WIRE_SKIP_TYPE, B.WIRE_MALFORMED, B.WIRE_COMMIT_VOTE,
              B.WIRE_IGNORED):
        assert kinds[0][k] > 100, (k, kinds[0])
    assert kinds[1][B.WIRE_OK] > 100
    if read_index:
        assert all(len(a.read_index_get(g)[0]) == q.count[g] for g in range(0, s.n, 997))
    a.close()


# --------------------------------------------------------------------------- 3. 1M leaders


def leaders_1m(rng, n, term=7):
    """n five-voter leaders at `term` (term_start last + 1, vote = id 1, RAFTGPU_VOTER_LEADER) on the device and in the
    oracle -> (arena, columns, votes, table, last_index)."""
    a = B.Arena(n)
    assert a.group_alloc_range(n) == 0
    g = np.arange(n, dtype=np.uint32)
    last = rng.integers(10, 1 << 30, n).astype(np.uint64)
    com = last - rng.integers(0, 10, n).astype(np.uint64)
    setup = np.zeros(4 * n, B.CTL_CMD_DTYPE)
    setup["group"] = np.tile(g, 4)
    setup["op"][:n], setup["a"][:n, 0], setup["a"][:n, 3] = B.CTL_SET_CONF, 0x1F, last + 1
    setup["op"][n:2 * n] = B.CTL_RESET
    setup["a"][n:2 * n] = np.stack([last + 1, last, com, last], 1)
    setup["op"][2 * n:3 * n], setup["a"][2 * n:3 * n, 0] = B.CTL_SET_TERM, term
    setup["op"][3 * n:] = B.CTL_BECOME_LEADER
    assert np.all(a.control(setup)["status"] == 0)
    c = O.new_columns(n, n)
    c.term_start[:] = B.NO_TERM_START
    vt = np.zeros((O.SLOTS, n), np.uint8)
    CO.arena_control(c, vt, setup)
    table = Q.voters(n)
    table["id"], table["vote"], table["last_term"], table["persisted"], table["commit_term"] = 1, 1, term, last, term
    table["flags"] = B.VOTER_LEADER
    return a, c, vt, table, c.last_index[:n].copy()   # (the leader's empty entry at term_start)


def bursts(rng, n, last, table, term=7):
    """The three bursts as SYNTH_VOTE_REQUEST_DTYPE entries, shuffled: the winners' late same-term requests (1-2 per
    group, rejected), pre-votes at term + 1 in lease (half of the groups: IGNORED) and out of it, and MsgRequestVote
    at term + 1 out of lease for a third of the groups (bumps) -> {name: entries}."""
    g = np.arange(n, dtype=np.uint32)

    def req(gs, typ, t):
        e = np.zeros(len(gs), B.SYNTH_VOTE_REQUEST_DTYPE)
        e["hdr"], e["msg_type"], e["to"], e["from"] = gs << 4 | 1, typ, 1, rng.integers(2, 6, len(gs))
        e["term"], e["log_term"] = t, term
        e["index"] = last[gs] + rng.integers(0, 2, len(gs)).astype(np.uint64) - 1
        return e[rng.permutation(len(e))]

    lease = rng.random(n) < 0.5
    third = np.flatnonzero(rng.random(n) < 1 / 3).astype(np.uint32)
    return {"late": req(np.concatenate([g, np.flatnonzero(rng.random(n) < 0.5).astype(np.uint32)]), Q.VOTE, term),
            "pre_vote": req(g, Q.PRE_VOTE, term + 1), "vote": req(third, Q.VOTE, term + 1)}, lease


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_1m_leaders_in_three_bursts(device):
    rng = np.random.default_rng(0x7601 + device)
    n = 1_000_000
    a, c, vt, table, last = leaders_1m(rng, n)
    bs, lease = bursts(rng, n, last, table)
    seen = {}
    for name in ("late", "pre_vote", "vote"):
        t = table.copy()
        if name == "pre_vote":
            t["flags"][lease] |= B.VOTER_LEASE
        blob, off = B.synth_encode_vote_requests(bs[name])
        want = LV.batch(c, None, vt, blob, off, t, n_bytes=int(off[-1]))
        got = PF.run(a, "leader_vote_request_wire", blob[: off[-1]], off, t, device=device)
        PF.equal(want, got, LQ.NAMES, name)
        seen[name] = np.bincount(got[0], minlength=256)
    check_columns(a, c, vt, n)
    assert seen["late"][B.WIRE_OK << 4] > n and seen["late"][B.WIRE_OK << 4 | B.VREQ_GRANTED] == 0
    assert seen["pre_vote"][B.WIRE_IGNORED << 4] > n // 3 and seen["pre_vote"][B.WIRE_OK << 4 | B.VREQ_GRANTED] > n // 8
    bumped = seen["vote"][B.WIRE_OK << 4 | B.VREQ_GRANTED | B.VREQ_VOTED | B.VREQ_BUMPED] + seen["vote"][B.WIRE_OK << 4 |
                                                                                                  B.VREQ_BUMPED]
    assert bumped > n // 4 and np.count_nonzero(c.term[:n] == 8) == bumped
    a.close()


# --------------------------------------------------------------------------- 4. refusals


def test_no_frames_and_refusals():
    a = B.Arena(64)
    assert a.group_alloc_range(16) == 0
    a.control(cmds(*[(B.CTL_SET_CONF, g, 0, 0, (0x7, 0, 0, 11)) for g in range(16)],
                   *[(B.CTL_RESET, g, 0, 0, (11, 10, 10, 10)) for g in range(16)],
                   *[(B.CTL_SET_TERM, g, 0, 0, (3,)) for g in range(16)]))
    t = Q.voters(64)
    t["id"], t["vote"], t["flags"] = 1, 1, B.VOTER_LEADER
    got = PF.device(a, "leader_vote_request_wire", np.zeros(0, np.uint8), np.zeros(1, np.uint32), t)
    assert got[0].size == 0 and got[4].tolist() == [0, 0]
    got = a.leader_vote_request_wire(F.Frames([]), t)
    assert got[0].size == 0 and got[4].tolist() == [0, 0]
    L_, h = a._L, a._h
    n = 16
    blob, off = F.batch([F.frame(g, 0, Q.request(Q.VOTE, 4, 1, 10, frm=2)) for g in range(n)])
    blob = np.concatenate([blob, np.zeros(16, np.uint8)])
    bound = B.vote_request_wire_bound(n)
    nb = int(off[-1])
    with PF.refusals(a, "leader_vote_request_wire", blob, off, t, n_bytes=nb) as r:
        dev, d = r.call, r.args
        refused = [dev(cap=bound - 1), dev(b=d["b"] + 4), dev(v=d["v"] + 8), dev(rb=d["rb"] + 4), dev(nb=1 << 32),
                   dev(n=1 << 32, cap=1 << 40), dev(n=(1 << 26) + 1, cap=1 << 40), dev(v=None), dev(st=None), dev(b=None),
                   dev(o=None), dev(rb=None), dev(t=None), dev(ro=None)]
        assert refused == [B.ERR_INVALID] * len(refused), refused
        assert r.untouched()                                                  # nothing was launched
        assert np.all(a.column_read(B.COL_TERM, 0, 0, 16, np.uint64) == 3)
        st, out, rb, ro, tot = np.zeros(n, np.uint8), np.zeros(2 * n, np.uint64), np.zeros(bound, np.uint8), \
            np.zeros(n + 1, np.uint32), np.zeros(2, np.uint64)
        assert L_.raftgpu_leader_vote_request_wire(h, blob.ctypes.data, nb, off.ctypes.data, n, t.ctypes.data,
                                                   st.ctypes.data, out.ctypes.data, rb.ctypes.data, bound - 1,
                                                   ro.ctypes.data, tot.ctypes.data) == B.ERR_INVALID
        assert L_.raftgpu_leader_vote_request_wire(h, blob.ctypes.data, nb, off.ctypes.data, n, None, st.ctypes.data,
                                                   out.ctypes.data, rb.ctypes.data, bound, ro.ctypes.data,
                                                   tot.ctypes.data) == B.ERR_INVALID
        assert dev() == B.OK                                                  # the same call with every rule kept
        assert r.read("t", np.zeros(2, np.uint64)).tolist()[0] == n
        assert np.all(r.read("st", np.zeros(n, np.uint8)) == B.WIRE_OK << 4 | B.VREQ_GRANTED | B.VREQ_VOTED | B.VREQ_BUMPED)
        assert np.all(a.column_read(B.COL_TERM, 0, 0, 16, np.uint64) == 4)
        assert np.all(a.column_read(B.COL_TERM_START, 0, 0, 16, np.uint64) == B.NO_TERM_START)
    a.close()


# --------------------------------------------------------------------------- 5. one partition-heal buffer


def test_partition_heal_buffer_through_the_leader_side():
    """A store of leaders hears, in one buffer, what a healed partition sends: the isolated peers' MsgRequestPreVote and
    MsgRequestVote at and above each leader's term, and the six types raftgpu_leader_term_wire takes.  On the device:
    raftgpu_leader_term_wire and its host side, then this pass, its host side and raftgpu_vote_request_wire on the
    frames of the groups either pass deposed, until no frame is left -- each call against its batch oracle.  (The
    leader passes and the follower passes, which take frames of other types, have their own tests.)"""
    rng = np.random.default_rng(0x7640)
    s = L.scenario(rng, 40_000, 1_000)
    s.leader[:] = s.table["id"]
    a = arena_of(s)
    c, vt = Q.state_of(s)
    lt_frames, meta = L.frames(rng, s, per_group=(0, 3))
    vr_frames = s.frames(rng, per_group=(1, 3), noise=False, commit_vote=False)
    frames_ = lt_frames + vr_frames
    perm = rng.permutation(len(frames_))
    frames_ = [frames_[i] for i in perm]
    is_vr = perm >= len(lt_frames)
    table, role, leader = s.table.copy(), s.role.copy(), s.leader.copy()
    blob, off = F.batch(frames_)
    want = LT.batch(c, None, vt, blob, off, table)
    got = a.leader_term_wire(PF.host_batch(blob, off), table)
    PF.equal(want, got, LQ.NAMES, "leader term")
    st = got[0]
    assert np.all(st[is_vr] == B.WIRE_SKIP_TYPE << 4)
    lt_at = np.flatnonzero(~is_vr)
    L.host_side(table, role, leader, st[lt_at], got[1][lt_at], [meta[perm[i]] for i in lt_at])
    passes = _checked(_device_passes(a, True), LQ.oracle_passes(c, None, vt), (a, c, vt, s.n))
    _, rounds, kinds = LQ.settle(c, None, vt, role, table, [frames_[i] for i in np.flatnonzero(is_vr)], *passes)
    assert kinds[0][B.WIRE_ROLE] > 1000 and kinds[0][B.WIRE_OK] > 1000 and kinds[0][B.WIRE_DUP] > 1000
    assert np.count_nonzero(st & B.FTERM_BUMPED) > 1000 and rounds > 2
    a.close()
