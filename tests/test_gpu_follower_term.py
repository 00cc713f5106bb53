"""The term prefix of MsgAppend / MsgHeartbeat at a follower on the GPU (raftgpu_follower_term_wire[_device]) against the
batch oracle (oracle/follow_term_oracle.c), byte for byte: random 100K-group batches with wide pairs, read queues and
Inflights, hostile terms, one group's 10 000 frames, n = 0 and the refusals; then a store's restart and a stale leader
as round trips through the broadcast, follower and leader passes.  Run with -m gpu."""
import numpy as np
import pytest

from oracle import oracle as O
from oracle import control_oracle as CO
from oracle import follow_term_oracle as FT
from oracle import read_oracle as RO
from helpers import B, arena_of, check_columns, ARENA_COLUMNS
from control_cmds import cmds
import follow_term as T
import hb_follow as HB
import hb_frames as F
import pass_forms as PF
import vote_request_frames as Q

pytestmark = pytest.mark.gpu

NAMES = ("status", "out", "bytes", "offsets", "totals")


# --------------------------------------------------------------------------- 1. random 100K-group batches


@pytest.mark.parametrize("device,read_index,inflights", [(False, False, 0), (True, False, 0), (True, True, 0),
                                                         (True, False, 4)],
                         ids=["host", "device", "device-read-queues", "device-inflights"])
def test_random_batches_vs_oracle(device, read_index, inflights):
    rng = np.random.default_rng(0x7400 + 4 * device + 2 * read_index + (inflights > 0))
    s = T.scenario(rng, 96_000, 2_000)
    a = arena_of(s, read_index, inflights)
    c, vt = Q.state_of(s)
    q = None
    if read_index:
        q = RO.ReadQueues(c.cap, 8)
        q.allocated[: s.n] = 1
    if inflights:
        O.enable_inflights(c, inflights)
        adds = cmds(*[(B.CTL_PROGRESS_OP, int(g), int(sl), B.POP_INS_ADD, (int(s.last[g]) + k,))
                      for g in rng.choice(s.lows, 20_000) for sl in (0, 1) for k in (1, 2)])
        got = a.control(adds)
        assert np.array_equal(got, CO.arena_control(c, vt, adds))
        assert (got["status"] == 0).sum() > 10_000
        check_columns(a, c, vt, s.n, ins=True)
    table, role, leader = s.table.copy(), s.role.copy(), s.leader.copy()
    kinds = np.zeros(16, np.int64)
    for rnd in range(2):
        frames_ = T.frames(rng, s, per_group=(1, 3)) + T.noise(rng, s, 3000)
        frames_ = [frames_[i] for i in rng.permutation(len(frames_))]
        blob, off = F.batch(frames_)
        want = FT.batch(c, q, vt, blob, off, table)
        got = PF.run(a, "follower_term_wire", *F.batch(frames_), table, device=device)
        PF.equal(want, got, NAMES, rnd)
        check_columns(a, c, vt, s.n, ins=bool(inflights))
        if read_index:
            assert all(len(a.read_index_get(g)[0]) == q.count[g] for g in range(0, s.n, 997))
        T.host_side(table, role, leader, got[0], got[1], frames_)
        s.term[:] = c.term[: s.n]
        kinds += np.bincount(got[0] >> 4, minlength=16)
    for k in (B.WIRE_OK, B.WIRE_STALE, B.WIRE_ROLE, B.WIRE_TERM, B.WIRE_SKIP_TYPE, B.WIRE_MALFORMED):
        assert kinds[k] > 100, (k, kinds)
    a.close()


# --------------------------------------------------------------------------- 2. edges


def _small(n_groups=6, term=5):
    a = B.Arena(64)
    assert a.group_alloc_range(n_groups) == 0
    a.control(cmds(*[(B.CTL_SET_CONF, g, 0, 0, (0b111, 0, 0, 11)) for g in range(n_groups)],
                   *[(B.CTL_RESET, g, 0, 0, (B.NO_TERM_START, 10, 8, 10)) for g in range(n_groups)],
                   *[(B.CTL_SET_TERM, g, 0, 0, (term,)) for g in range(n_groups)]))
    c = O.new_columns(64, n_groups)
    vt = np.zeros((O.SLOTS, c.cap), np.uint8)
    CO.arena_control(c, vt, cmds(*[(B.CTL_SET_CONF, g, 0, 0, (0b111, 0, 0, 11)) for g in range(n_groups)],
                                 *[(B.CTL_RESET, g, 0, 0, (B.NO_TERM_START, 10, 8, 10)) for g in range(n_groups)],
                                 *[(B.CTL_SET_TERM, g, 0, 0, (term,)) for g in range(n_groups)]))
    t = Q.voters(n_groups)
    t["id"], t["persisted"], t["flags"] = np.arange(1, n_groups + 1), 10, B.VOTER_SELECT | B.VOTER_STALE_REPLY
    return a, c, vt, t


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_hostile_terms(device):
    """Terms, froms and ids up to 2^64 - 1: replies at the widest varints, bumps to the top term."""
    a, c, vt, t = _small(4, 5)
    top = (1 << 64) - 1
    t["id"][1] = top
    frames_ = [F.frame(0, 3, F.message(8, top, frm=top)), F.frame(0, 1, F.message(3, 1 << 63, frm=top)),
               F.frame(0, 2, F.message(8, 4, frm=top)), F.frame(1, 15, F.message(3, 4, frm=top)),
               F.frame(1, 0, F.message(8, 1 << 32, frm=1 << 63)), F.frame(1, 0, F.message(8, 128, frm=127)),
               F.frame(2, 0, F.message(8, top - 1, frm=0)), F.frame(2, 0, F.message(8, top, frm=0)),
               F.frame(3, 0, F.message(3, 5, frm=7))]
    blob, off = F.batch(frames_)
    want = FT.batch(c, None, vt, blob, off, t)
    got = PF.run(a, "follower_term_wire", *F.batch(frames_), t, device=device)
    PF.equal(want, got, NAMES, "hostile")
    check_columns(a, c, vt, 4)
    assert c.term[:4].tolist() == [top, 1 << 32, top, 5]
    assert int(got[4][0]) == 5   # frames 1, 2 (group 0), 3, 5 (group 1) and 6 (group 2) are below their group's T
    a.close()


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_ten_thousand_frames_of_one_group(device):
    rng = np.random.default_rng(0x7401)
    a, c, vt, t = _small(2, 1000)
    terms = rng.integers(900, 1100, 10_000)
    frames_ = [F.frame(1, int(k) % 16, (F.message(8, int(x), frm=T.leader_of(int(x))) if k % 3 else
                                        F.message(3, int(x), frm=T.leader_of(int(x)))))
               for k, x in enumerate(terms.tolist())]
    blob, off = F.batch(frames_)
    want = FT.batch(c, None, vt, blob, off, t)
    got = PF.run(a, "follower_term_wire", *F.batch(frames_), t, device=device)
    PF.equal(want, got, NAMES, "one group")
    check_columns(a, c, vt, 2)
    st = got[0]
    assert c.term[1] == terms.max() and np.count_nonzero(st & B.FTERM_BUMPED) == 1
    assert np.flatnonzero(st & B.FTERM_BUMPED)[0] == np.flatnonzero(terms == terms.max())[0]
    assert np.count_nonzero(st >> 4 == B.WIRE_STALE) == np.count_nonzero(terms < terms.max())
    a.close()


def test_no_frames():
    a, c, vt, t = _small(2)
    st, out, rb, ro, tot = PF.device(a, "follower_term_wire", np.zeros(0, np.uint8), np.zeros(1, np.uint32), t)
    assert st.size == 0 and tot.tolist() == [0, 0] and ro.tolist() == [0]
    st, out, rb, ro, tot = a.follower_term_wire(F.Frames([]), t)
    assert st.size == 0 and tot.tolist() == [0, 0] and ro.tolist() == [0]
    check_columns(a, c, vt, 2)
    a.close()


def test_refusals_before_any_launch():
    a, c, vt, t = _small(16, 3)
    L, h = a._L, a._h
    n = 16
    blob, off = F.batch([F.frame(g, 0, F.message(8, 4, frm=2)) for g in range(n)])
    blob = np.concatenate([blob, np.zeros(16, np.uint8)])
    t = Q.voters(64)
    t["flags"] = B.VOTER_SELECT
    bound = B.follower_term_wire_bound(n)
    assert bound == 39 * n
    nb = off[-1]
    with PF.refusals(a, "follower_term_wire", blob, off, t, n_bytes=nb) as r:
        dev, d = r.call, r.args
        refused = [dev(cap=bound - 1), dev(b=d["b"] + 4), dev(v=d["v"] + 8), dev(rb=d["rb"] + 4), dev(nb=1 << 32),
                   dev(n=1 << 32, cap=1 << 40), dev(n=(1 << 32) // 39 + 1, cap=1 << 40), dev(v=None), dev(st=None),
                   dev(b=None), dev(o=None), dev(rb=None), dev(t=None), dev(ro=None)]
        assert refused == [B.ERR_INVALID] * len(refused), refused
        assert r.untouched()                                                  # nothing was launched
        assert np.all(a.column_read(B.COL_TERM, 0, 0, 16, np.uint64) == 3)
        st, out, rb, ro, tot = np.zeros(n, np.uint8), np.zeros(2 * n, np.uint64), np.zeros(bound, np.uint8), \
            np.zeros(n + 1, np.uint32), np.zeros(2, np.uint64)
        assert L.raftgpu_follower_term_wire(h, blob.ctypes.data, nb, off.ctypes.data, n, t.ctypes.data, st.ctypes.data,
                                            out.ctypes.data, rb.ctypes.data, bound - 1, ro.ctypes.data, tot.ctypes.data) == B.ERR_INVALID
        assert L.raftgpu_follower_term_wire(h, blob.ctypes.data, nb, off.ctypes.data, n, None, st.ctypes.data,
                                            out.ctypes.data, rb.ctypes.data, bound, ro.ctypes.data, tot.ctypes.data) == B.ERR_INVALID
        assert dev() == B.OK                                                      # the same call with every rule kept
        gst = r.read("st", np.zeros(n, np.uint8))
        assert np.all(gst == (B.WIRE_OK << 4 | B.FTERM_BUMPED)) and np.all(a.column_read(B.COL_TERM, 0, 0, 16, np.uint64) == 4)
    a.close()


# --------------------------------------------------------------------------- 3. round trips


def test_restart_round_trip():
    """A store restarts: its 20K x 4 follower groups are at term t, their leaders (5 voters) were elected at t + 1 and
    appended their empty entry.  The leaders' raftgpu_heartbeat_frames and raftgpu_append_frames go through this pass,
    then raftgpu_follower_heartbeat, then raftgpu_follower_append; the responses come back through
    raftgpu_heartbeat_wire and raftgpu_step_begin_wire.  Every follower ends at t + 1 with its leader's committed, the
    append is rejected at the follower's last index and decided from the leader's stated run, and no frame is the
    host's on either side."""
    rng = np.random.default_rng(0x7402)
    n, P, t, li = 20_000, 5, 7, 1000
    la = T.leaders(n, P, t + 1, li)
    ids = np.zeros((B.SLOTS + 1, n), np.uint64)
    ids[:B.SLOTS] = (np.arange(B.SLOTS) + 1)[:, None]
    ids[B.SLOTS] = 1
    _, hb, hoff, htot = la.heartbeat_frames(0, n, ids)
    _, ap, aoff, _, atot = la.append_frames(0, n, ids)
    assert int(htot[0]) == int(atot[0]) == n * (P - 1)
    frames_ = HB.frames_of(T.to_followers(hb, hoff, P), hoff) + HB.frames_of(T.to_followers(ap, aoff, P), aoff)
    frames_ = [np.array([h], "<u4").tobytes() + b for h, b in frames_]
    frames_ = [frames_[i] for i in rng.permutation(len(frames_))]
    nf = n * (P - 1)
    fa, table = T.followers(nf, t, li, P, rng)
    blob, off = F.batch(frames_)
    st, out, _, _, tot = PF.device(fa, "follower_term_wire", blob, off, table)
    assert np.all(st >> 4 == B.WIRE_OK) and np.count_nonzero(st & B.FTERM_BUMPED) == nf and tot.tolist() == [0, 0]
    assert np.all(fa.column_read(B.COL_TERM, 0, 0, nf, np.uint64) == t + 1)
    role, leader = np.zeros(nf, np.uint8), np.zeros(nf, np.uint64)
    T.host_side(table, role, leader, st, out, frames_)
    assert np.all(leader == 1)
    typ = T.types_of(frames_)
    hbs = [f for f, k in zip(frames_, typ) if k == T.HEARTBEAT]
    aps = [f for f, k in zip(frames_, typ) if k == T.APPEND]
    self_ids = np.zeros(fa.cap, np.uint64)
    self_ids[:nf] = table["id"]
    hst, _, hrb, hro, _ = fa.follower_heartbeat(F.Frames(hbs), self_ids, HB.bitmap(np.arange(fa.cap) < nf))
    assert np.all(hst == B.WIRE_OK << 4 | B.RES_OK)
    logs = np.zeros(nf, B.FOLLOWER_LOG_DTYPE)
    logs["id"], logs["run_start"], logs["run_term"], logs["flags"] = table["id"], 1, t, B.FOLLOWER_SELECT
    ast, _, arb, aro, _ = fa.follower_append(F.Frames(aps), logs)
    assert np.all(ast == B.WIRE_OK << 4 | B.RES_OK | B.FAPP_REJECT)
    assert np.all(fa.column_read(B.COL_COMMITTED, 0, 0, nf, np.uint64) == li)   # the leaders' committed
    assert np.all(fa.column_read(B.COL_TERM, 0, 0, nf, np.uint64) == t + 1)
    fa.close()
    # the responses at the leaders
    lst, _ = la.heartbeat_wire(F.Frames([bytes(x) for x in np.split(T.to_leaders(hrb, hro, P), hro[1:-1])]))
    assert np.all(lst >> 4 == B.WIRE_OK)
    back = T.to_leaders(arb, aro, P)
    wb = F.Frames([bytes(back[a0:b0]) for a0, b0 in zip(aro[:-1].tolist(), aro[1:].tolist())])
    la.step_begin_wire(wb, B.STEP_READ_COMMITTED)
    la.step_wait()
    assert np.all(la.wire_status() >> 4 == B.WIRE_OK)
    lc = la.read_columns(n)
    assert np.all(lc.next_idx[1:P, :n] == li + 1)   # find_conflict_by_term(li, t) from the stated run: the probe at li
    la.close()


def test_stale_round_trip():
    """A deposed leader at term t keeps sending heartbeats to followers that moved to t + 1: with check_quorum they
    answer with an empty MsgAppendResponse at t + 1, which its raftgpu_step_begin_wire returns TERM (the host steps the
    leader down, as before); without it they drop the heartbeats."""
    rng = np.random.default_rng(0x7403)
    n, P, t, li = 5_000, 5, 7, 1000
    old = T.leaders(n, P, t, li)
    ids = np.zeros((B.SLOTS + 1, n), np.uint64)
    ids[:B.SLOTS] = (np.arange(B.SLOTS) + 1)[:, None]
    ids[B.SLOTS] = 1
    _, hb, hoff, _ = old.heartbeat_frames(0, n, ids)
    nf = n * (P - 1)
    fa, table = T.followers(nf, t + 1, li, P, rng)
    quiet = rng.random(nf) < 0.25
    table["flags"][quiet] = B.VOTER_SELECT
    to_f = T.to_followers(hb, hoff, P)
    st, out, rb, ro, tot = PF.device(fa, "follower_term_wire", to_f, hoff, table)
    g = HB.headers(to_f, hoff) >> 4
    assert np.array_equal(st, np.where(quiet[g], B.WIRE_STALE << 4, B.WIRE_STALE << 4 | B.RES_OK).astype(np.uint8))
    assert int(tot[0]) == np.count_nonzero(~quiet) and not out.any()
    assert np.all(fa.column_read(B.COL_TERM, 0, 0, nf, np.uint64) == t + 1)
    for k in range(0, int(tot[0]), 997):
        m = O.wire_decode_message(rb[ro[k] + 4:ro[k + 1]].tobytes())
        assert (m["msg_type"], m["to"], m["term"], m["index"], m["commit"], m["reject"]) == (4, 1, t + 1, 0, 0, 0)
    fa.close()
    before = old.read_columns(n)
    back = T.to_leaders(rb, ro, P)
    old.step_begin_wire(F.Frames([bytes(back[a0:b0]) for a0, b0 in zip(ro[:-1].tolist(), ro[1:].tolist())]),
                        B.STEP_READ_COMMITTED)
    old.step_wait()
    assert np.all(old.wire_status() >> 4 == B.WIRE_TERM)
    after = old.read_columns(n)
    for name in ARENA_COLUMNS:
        assert np.array_equal(getattr(before, name), getattr(after, name)), name
    old.close()
