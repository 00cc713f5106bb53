"""The term prefix of the frames that reach a leader on the GPU (raftgpu_leader_term_wire[_device]) against the batch
oracle (oracle/leader_term_oracle.c), byte for byte: random 100K-group batches with wide pairs, read queues, Inflights
and leader runs, hostile terms, one group's 10 000 frames, n = 0 and the refusals, the host form between a wire step's
begin and its wait; then a deposed leader and a won election as round trips through the other passes.  Run with -m gpu."""
import numpy as np
import pytest

from oracle import oracle as O
from oracle import control_oracle as CO
from oracle import leader_term_oracle as LT
from oracle import read_oracle as RO
from helpers import B, arena_of, check_columns, ARENA_COLUMNS
from control_cmds import cmds
import app_follow as A
import follow_term as T
import hb_follow as HB
import hb_frames as F
import leader_term as L
import pass_forms as PF
import vote_request_frames as Q

pytestmark = pytest.mark.gpu


NAMES = ("status", "out", "bytes", "offsets", "totals")


# --------------------------------------------------------------------------- 1. random 100K-group batches


@pytest.mark.parametrize("device,read_index,inflights,runs", [(False, False, 0, False), (True, False, 0, False),
                                                              (True, True, 0, False), (True, False, 4, False),
                                                              (True, False, 0, True)],
                         ids=["host", "device", "device-read-queues", "device-inflights", "device-leader-runs"])
def test_random_batches_vs_oracle(device, read_index, inflights, runs):
    rng = np.random.default_rng(0x7500 + 8 * runs + 4 * device + 2 * read_index + (inflights > 0))
    s = T.scenario(rng, 96_000, 2_000, p_role=(0.1, 0.0, 0.0, 0.9))
    a = arena_of(s, read_index, inflights, runs)
    c, vt = Q.state_of(s)
    q = None
    if read_index:
        q = RO.ReadQueues(c.cap, 8)
        q.allocated[: s.n] = 1
    if inflights:
        O.enable_inflights(c, inflights)
        adds = cmds(*[(B.CTL_PROGRESS_OP, int(g), int(sl), B.POP_INS_ADD, (int(s.last[g]) + k,))
                      for g in rng.choice(s.lows, 20_000) for sl in (1, 2) for k in (1, 2)])
        got = a.control(adds)
        assert np.array_equal(got, CO.arena_control(c, vt, adds))
        check_columns(a, c, vt, s.n, ins=True)
    leaders = np.array([g for g in s.lows if s.role[g] == Q.LEADER])
    if runs:
        rows = np.zeros(len(leaders), B.LEADER_RUNS_DTYPE)
        rows["group"], rows["term"], rows["term_start"] = leaders, s.term[leaders], s.last[leaders] + 1
        rows["run_start"][:, 0], rows["run_term"][:, 0] = 1, 1
        assert np.all(a.leader_runs_set(rows) == 0)
    table, role, leader = s.table.copy(), s.role.copy(), s.leader.copy()
    kinds = np.zeros(16, np.int64)
    for rnd in range(2):
        frames_, meta = L.frames(rng, s, per_group=(1, 3))
        frames_ += L.noise(rng, s, 3000)
        frames_ = [frames_[i] for i in rng.permutation(len(frames_))]
        blob, off = F.batch(frames_)
        want = LT.batch(c, q, vt, blob, off, table)
        got = PF.run(a, "leader_term_wire", *F.batch(frames_), table, device=device)
        PF.equal(want, got, NAMES, rnd)
        check_columns(a, c, vt, s.n, ins=bool(inflights))
        if read_index:
            assert all(len(a.read_index_get(g)[0]) == q.count[g] for g in range(0, s.n, 997))
        s.term[:] = c.term[: s.n]
        kinds += np.bincount(got[0] >> 4, minlength=16)
    for k in (B.WIRE_OK, B.WIRE_STALE, B.WIRE_IGNORED, B.WIRE_ROLE, B.WIRE_TERM, B.WIRE_SKIP_TYPE, B.WIRE_MALFORMED):
        assert kinds[k] > 100, (k, kinds)
    if runs:   # a bumped leader's row is inert: its rejections are the host's again
        bumped = leaders[c.term_start[leaders] == B.NO_TERM_START][:500]
        assert len(bumped) > 100
        rej = [F.frame(int(g), 1, F.message(4, int(c.term[g]), index=5, reject=True, reject_hint=3, frm=2) +
                       F.varint(5 << 3) + F.varint(1)) for g in bumped]   # log_term 1
        a.step_begin_wire(F.Frames(rej), B.STEP_READ_COMMITTED)
        a.step_wait()
        assert np.all(a.wire_status() >> 4 == B.WIRE_NEEDS_LOG)
    a.close()


# --------------------------------------------------------------------------- 2. edges


def _small(n_groups=6, term=5):
    """n_groups leaders at `term` (voters 0-2, term_start 11) on the device and in the oracle."""
    ops = cmds(*[(B.CTL_SET_CONF, g, 0, 0, (0b111, 0, 0, 11)) for g in range(n_groups)],
               *[(B.CTL_RESET, g, 0, 0, (B.NO_TERM_START, 10, 8, 10)) for g in range(n_groups)],
               *[(B.CTL_SET_TERM, g, 0, 0, (term,)) for g in range(n_groups)],
               *[(B.CTL_RESET, g, 0, 0, (11, 10, 8, 10)) for g in range(n_groups)],
               *[(B.CTL_BECOME_LEADER, g) for g in range(n_groups)])
    a = B.Arena(64)
    assert a.group_alloc_range(n_groups) == 0
    assert np.all(a.control(ops)["status"] == 0)
    c = O.new_columns(64, n_groups)
    c.term_start[:] = B.NO_TERM_START
    vt = np.zeros((O.SLOTS, c.cap), np.uint8)
    assert np.all(CO.arena_control(c, vt, ops)["status"] == 0)
    t = Q.voters(n_groups)
    t["id"], t["persisted"], t["flags"] = np.arange(1, n_groups + 1), 10, B.VOTER_STALE_REPLY
    return a, c, vt, t


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_hostile_terms(device):
    """Terms, froms and ids up to 2^64 - 1: replies at the widest varints, bumps to the top term."""
    a, c, vt, t = _small(4, 5)
    top = (1 << 64) - 1
    t["id"][1] = top
    frames_ = [F.frame(0, 3, F.message(6, top, reject=True, frm=top)), F.frame(0, 1, F.message(3, 1 << 63, frm=top)),
               F.frame(0, 2, F.message(8, 4, frm=top)), F.frame(1, 15, F.message(3, 4, frm=top)),
               F.frame(1, 2, F.message(9, 1 << 32, frm=1 << 63)), F.frame(1, 0, F.message(8, 128, frm=127)),
               F.frame(2, 0, F.message(8, top - 1, frm=0)), F.frame(2, 1, F.message(18, top, frm=0)),
               F.frame(3, 0, F.message(3, 5, frm=7)), F.frame(3, 1, F.message(4, 5, frm=7))]
    blob, off = F.batch(frames_)
    want = LT.batch(c, None, vt, blob, off, t)
    got = PF.run(a, "leader_term_wire", *F.batch(frames_), t, device=device)
    PF.equal(want, got, NAMES, "hostile")
    check_columns(a, c, vt, 4)
    assert c.term[:4].tolist() == [top, 1 << 32, top - 1, 5]
    assert int(got[4][0]) == 4   # frames 1, 2 (group 0), 3 and 5 (group 1) are MsgAppend / MsgHeartbeat below T
    a.close()


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_ten_thousand_frames_of_one_group(device):
    rng = np.random.default_rng(0x7501)
    a, c, vt, t = _small(2, 1000)
    terms = rng.integers(900, 1100, 10_000)
    typs = rng.choice(L.TYPES, 10_000)
    frames_ = [F.frame(1, k % 16, A.message(3, int(x), frm=T.leader_of(int(x))) if y == 3 else
                       F.message(int(y), int(x), reject=True, frm=T.leader_of(int(x))))
               for k, (x, y) in enumerate(zip(terms.tolist(), typs.tolist()))]
    blob, off = F.batch(frames_)
    want = LT.batch(c, None, vt, blob, off, t)
    got = PF.run(a, "leader_term_wire", *F.batch(frames_), t, device=device)
    PF.equal(want, got, NAMES, "one group")
    check_columns(a, c, vt, 2)
    st = got[0]
    assert c.term[1] == terms.max() and np.count_nonzero(st & B.FTERM_BUMPED) == 1
    assert np.flatnonzero(st & B.FTERM_BUMPED)[0] == np.flatnonzero(terms == terms.max())[0]
    assert np.count_nonzero(st >> 4 == B.WIRE_STALE) == np.count_nonzero((terms < terms.max()) & (terms != 1000))
    a.close()


def test_no_frames():
    a, c, vt, t = _small(2)
    st, out, rb, ro, tot = PF.device(a, "leader_term_wire", np.zeros(0, np.uint8), np.zeros(1, np.uint32), t)
    assert st.size == 0 and tot.tolist() == [0, 0] and ro.tolist() == [0]
    st, out, rb, ro, tot = a.leader_term_wire(F.Frames([]), t)
    assert st.size == 0 and tot.tolist() == [0, 0] and ro.tolist() == [0]
    check_columns(a, c, vt, 2)
    a.close()


def test_refusals_before_any_launch():
    a, c, vt, t = _small(16, 3)
    Lb, h = a._L, a._h
    n = 16
    blob, off = F.batch([F.frame(g, 1, F.message(4, 4, frm=2)) for g in range(n)])
    blob = np.concatenate([blob, np.zeros(16, np.uint8)])
    t = Q.voters(64)
    bound = B.follower_term_wire_bound(n)
    nb = off[-1]
    with PF.refusals(a, "leader_term_wire", blob, off, t, n_bytes=nb) as r:
        dev, d = r.call, r.args
        refused = [dev(cap=bound - 1), dev(b=d["b"] + 4), dev(v=d["v"] + 8), dev(rb=d["rb"] + 4), dev(nb=1 << 32),
                   dev(n=1 << 32, cap=1 << 40), dev(n=(1 << 32) // 39 + 1, cap=1 << 40), dev(v=None), dev(st=None),
                   dev(b=None), dev(o=None), dev(rb=None), dev(t=None), dev(ro=None)]
        assert refused == [B.ERR_INVALID] * len(refused), refused
        assert r.untouched()                                                  # nothing was launched
        assert np.all(a.column_read(B.COL_TERM, 0, 0, 16, np.uint64) == 3)
        st, out, rb, ro, tot = np.zeros(n, np.uint8), np.zeros(2 * n, np.uint64), np.zeros(bound, np.uint8), \
            np.zeros(n + 1, np.uint32), np.zeros(2, np.uint64)
        assert Lb.raftgpu_leader_term_wire(h, blob.ctypes.data, nb, off.ctypes.data, n, t.ctypes.data, st.ctypes.data,
                                           out.ctypes.data, rb.ctypes.data, bound - 1, ro.ctypes.data, tot.ctypes.data) == B.ERR_INVALID
        assert Lb.raftgpu_leader_term_wire(h, blob.ctypes.data, nb, off.ctypes.data, n, None, st.ctypes.data,
                                           out.ctypes.data, rb.ctypes.data, bound, ro.ctypes.data, tot.ctypes.data) == B.ERR_INVALID
        assert dev() == B.OK                                                      # the same call with every rule kept
        gst = r.read("st", np.zeros(n, np.uint8))
        assert np.all(gst == (B.WIRE_OK << 4 | B.FTERM_BUMPED)) and np.all(a.column_read(B.COL_TERM, 0, 0, 16, np.uint64) == 4)
    a.close()


def test_host_form_between_a_wire_steps_begin_and_its_wait():
    """The host form called while a wire step is in flight runs after it, in submission order: the step's accepts at
    the term are applied first, then this pass deposes the groups that hear a higher term."""
    rng = np.random.default_rng(0x7502)
    s = T.scenario(rng, 20_000, 500, p_role=(0.0, 0.0, 0.0, 1.0))
    a = arena_of(s)
    c, vt = Q.state_of(s)
    step = [F.frame(g, 1, F.message(4, int(s.term[g]), index=int(s.last[g]), frm=2)) for g in s.lows]
    frames_, _ = L.frames(rng, s, per_group=(1, 3))
    L.leader_passes(c, step)
    blob, off = F.batch(frames_)
    want = LT.batch(c, None, vt, blob, off, s.table)
    a.step_begin_wire(F.Frames(step), B.STEP_READ_COMMITTED)
    got = a.leader_term_wire(F.Frames(frames_), s.table)
    a.step_wait()
    assert np.all(a.wire_status() >> 4 == B.WIRE_OK)
    PF.equal(want, got, NAMES, "overlap")
    check_columns(a, c, vt, s.n)
    a.close()


# --------------------------------------------------------------------------- 3. round trips


def test_disruptive_follower_round_trip():
    """test_disruptive_follower on devices: 5 000 leaders at term t still send heartbeats (raftgpu_heartbeat_frames) to
    followers that moved to t + 1; raftgpu_follower_term_wire answers them with stale MsgAppendResponse frames at
    t + 1; the leaders' wire step returns them TERM, and this pass deposes every leader: term t + 1, no leader."""
    rng = np.random.default_rng(0x7503)
    n, P, t, li = 5_000, 5, 7, 1000
    old = T.leaders(n, P, t, li)
    ids = np.zeros((B.SLOTS + 1, n), np.uint64)
    ids[:B.SLOTS] = (np.arange(B.SLOTS) + 1)[:, None]
    ids[B.SLOTS] = 1
    _, hb, hoff, _ = old.heartbeat_frames(0, n, ids)
    nf = n * (P - 1)
    fa, ftable = T.followers(nf, t + 1, li, P, rng)
    to_f = T.to_followers(hb, hoff, P)
    fst, _, rb, ro, tot = PF.device(fa, "follower_term_wire", to_f, hoff, ftable)
    assert np.all(fst == B.WIRE_STALE << 4 | B.RES_OK) and int(tot[0]) == nf
    fa.close()
    back = T.to_leaders(rb, ro, P)
    frames_ = [bytes(back[a0:b0]) for a0, b0 in zip(ro[:-1].tolist(), ro[1:].tolist())]
    old.step_begin_wire(F.Frames(frames_), B.STEP_READ_COMMITTED)
    old.step_wait()
    assert np.all(old.wire_status() >> 4 == B.WIRE_TERM)
    table = Q.voters(n)
    table["id"], table["persisted"], table["flags"] = 1, li + 1, B.VOTER_STALE_REPLY
    st, out, _, _, tot = old.leader_term_wire(F.Frames(frames_), table)
    g = HB.headers(back, ro) >> 4
    first = np.zeros(n, np.int64) - 1
    for i in range(len(g) - 1, -1, -1):
        first[g[i]] = i
    bumped = np.zeros(len(g), bool)
    bumped[first] = True
    assert np.array_equal(st, np.where(bumped, B.WIRE_OK << 4 | B.FTERM_BUMPED, B.WIRE_IGNORED << 4).astype(np.uint8))
    assert np.all(out[bumped] == [0, t + 1]) and not out[~bumped].any() and tot.tolist() == [0, 0]
    cols = old.read_columns(n)
    assert np.all(old.column_read(B.COL_TERM, 0, 0, n, np.uint64) == t + 1)
    assert np.all(cols.term_start == B.NO_TERM_START) and np.all(cols.committed == li)
    old.close()


def test_election_round_trip():
    """A store-wide election: 10 000 candidates at term t win on the first two grants of raftgpu_vote_wire, the caller
    runs raftgpu_control's BECOME_LEADER for them, and the late vote responses of the same election come back IGNORED
    here, with nothing changed; a rejection at a higher term still deposes."""
    n, P, t, li = 10_000, 5, 9, 500
    a = B.Arena(n + 64)
    assert a.group_alloc_range(n) == 0
    ops = []
    for g in range(n):
        ops += [(B.CTL_SET_CONF, g, 0, 0, ((1 << P) - 1, 0, 0, li + 1)), (B.CTL_RESET, g, 0, 0, (B.NO_TERM_START, li, li, li)),
                (B.CTL_SET_TERM, g, 0, 0, (t,)), (B.CTL_RESET_VOTES, g), (B.CTL_RECORD_VOTE, g, 0, 1)]
    assert np.all(a.control(cmds(*ops))["status"] == 0)
    sel = HB.bitmap(np.arange(a.cap) < n)
    early = [F.frame(g, s, F.message(6, t, frm=s + 1)) for g in range(n) for s in (1, 2)]
    vst, outcomes = a.vote_wire(F.Frames(early), sel)
    assert np.all(vst >> 4 == B.WIRE_OK) and len(outcomes) == n
    assert np.all(outcomes["result"] & 0xFF == B.VOTE_WON)
    lead = [(B.CTL_RESET, int(g), 0, 0, (li + 1, li, li, li)) for g in outcomes["group"]]
    lead += [(B.CTL_BECOME_LEADER, int(g)) for g in outcomes["group"]]
    assert np.all(a.control(cmds(*lead))["status"] == 0)
    before = a.read_columns(n)
    late = [F.frame(g, s, F.message(6, t, reject=s == 4, frm=s + 1)) for g in range(n) for s in (3, 4)]
    late += [F.frame(g, 3, F.message(18, t + 1, frm=4)) for g in range(0, n, 7)]
    table = Q.voters(n)
    table["id"], table["persisted"] = 1, li
    st, out, _, _, tot = a.leader_term_wire(F.Frames(late), table)
    assert np.all(st == B.WIRE_IGNORED << 4) and not out.any() and tot.tolist() == [0, 0]
    after = a.read_columns(n)
    for name in ARENA_COLUMNS:
        assert np.array_equal(getattr(before, name), getattr(after, name)), name
    st, out, _, _, _ = a.leader_term_wire(F.Frames([F.frame(5, 4, F.message(6, t + 2, reject=True, frm=5))]), table)
    assert st.tolist() == [B.WIRE_OK << 4 | B.FTERM_BUMPED] and out.tolist() == [[0, t + 2]]
    assert a.column_read(B.COL_TERM, 0, 0, n, np.uint64)[5] == t + 2
    a.close()
