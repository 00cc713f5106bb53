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
from helpers import B
from control_cmds import cmds
import follow_term as T
import hb_follow as HB
import hb_frames as F
import test_oracle_vote_request as TV
import vote_request_frames as Q

pytestmark = pytest.mark.gpu

ARENA_COLUMNS = ("term_start", "committed", "last_index", "matched", "next_idx", "peer_committed", "pflags")
NAMES = ("status", "out", "bytes", "offsets", "totals")


def _device(a, blob, off, voters, n_bytes=None):
    """The device form over buffers from raftgpu_device_alloc -> (status, out, response blob, offsets, totals)."""
    n = len(off) - 1
    n_bytes = len(blob) if n_bytes is None else n_bytes
    blob = np.concatenate([blob, np.zeros(16, np.uint8)])
    bound = B.follower_term_wire_bound(n)
    vt = np.ascontiguousarray(voters, B.VOTER_DTYPE)
    sizes = (len(blob), 4 * (n + 1), max(64, vt.nbytes), max(1, n), max(16, 16 * n), max(16, bound), 4 * (n + 1), 16)
    bufs = [a.device_alloc(x) for x in sizes]
    d_b, d_o, d_v, d_st, d_out, d_rb, d_ro, d_t = bufs
    for p, x in ((d_b, blob), (d_o, off), (d_v, vt)):
        a.h2d(p, x)
    a.follower_term_wire_device(d_b, n_bytes, d_o, n, d_v, d_st, d_out, d_rb, bound, d_ro, d_t)
    a.synchronize()
    tot = np.zeros(2, np.uint64)
    a.d2h(tot, d_t)
    st, out = np.zeros(n, np.uint8), np.zeros((n, 2), np.uint64)
    rb, ro = np.zeros(int(tot[1]), np.uint8), np.zeros(int(tot[0]) + 1, np.uint32)
    for arr, p in ((st, d_st), (out, d_out), (ro, d_ro), (rb, d_rb)):
        if arr.size:
            a.d2h(arr, p)
    for p in bufs:
        a.device_free(p)
    return st, out, rb, ro, tot


def _run(a, frames_, voters, device):
    if device:
        blob, off = F.batch(frames_)
        return _device(a, blob, off, voters)
    return a.follower_term_wire(F.Frames(frames_), voters)


def _equal(want, got, what):
    for w, g, name in zip(want, got, NAMES):
        assert np.array_equal(w, g), (what, name, np.flatnonzero(w != g)[:5] if w.shape == g.shape else (w.shape, g.shape))


def _check_columns(a, c, vt, n, ins=False):
    cols = a.read_columns(n)
    for name in ARENA_COLUMNS:
        assert np.array_equal(getattr(cols, name), getattr(c, name)[..., :n]), name
    assert np.array_equal(a.column_read(B.COL_TERM, 0, 0, n, np.uint64), c.term[:n])
    assert np.array_equal(np.stack([a.column_read(B.COL_VOTES, s, 0, n, np.uint8) for s in range(O.SLOTS)]), vt[:, :n])
    if ins:
        for s in range(O.SLOTS):
            assert np.array_equal(a.column_read(B.COL_INS_META, s, 0, n, np.uint32), c.ins_meta[s, :n]), s


def _noise(rng, s, k):
    """Frames the checks before the verdict settle: other types, garbage, truncated frames, high halves, m.term 0 and
    groups past the arena's highest slot."""
    out = []
    for _ in range(k):
        g = int(rng.choice(s.lows))
        term = int(s.term[g])
        kind = int(rng.integers(6))
        if kind == 0:
            out.append(F.frame(g, 0, F.message(int(rng.choice([4, 9, 5, 7, 10])), term + 1, frm=2)))
        elif kind == 1:
            out.append(F.frame(g, 0, rng.integers(0, 256, int(rng.integers(1, 12)), dtype=np.uint8).tobytes()))
        elif kind == 2:
            out.append(F.frame(g, 0, F.message(8, term + 1, 1 << 40, frm=2)[:-3]))
        elif kind == 3:
            out.append(F.frame(g + 1 if s.wide[g] else g, 0, F.message(8, term + 1 if s.wide[g] else 0, frm=2)))
        elif kind == 4:
            out.append(F.frame(g, 0, F.message(3, 0, frm=2)))
        else:
            out.append(F.frame(s.n + int(rng.integers(1, 100)), 0, F.message(8, term + 1, frm=2)))
    return out


def _arena_of(s, read_index=False, inflights=0):
    a = B.Arena(s.n + 64)
    if read_index:
        a.enable_read_index()
    if inflights:
        a.enable_inflights(inflights)
    if s.n_narrow:
        assert a.group_alloc_range(s.n_narrow) == 0
    for k in range(s.n_wide):
        assert a.group_alloc_wide() == s.n_narrow + 2 * k
    assert np.all(a.control(s.setup)["status"] == 0)
    return a


# --------------------------------------------------------------------------- 1. random 100K-group batches


@pytest.mark.parametrize("device,read_index,inflights", [(False, False, 0), (True, False, 0), (True, True, 0),
                                                         (True, False, 4)],
                         ids=["host", "device", "device-read-queues", "device-inflights"])
def test_random_batches_vs_oracle(device, read_index, inflights):
    rng = np.random.default_rng(0x7400 + 4 * device + 2 * read_index + (inflights > 0))
    s = T.scenario(rng, 96_000, 2_000)
    a = _arena_of(s, read_index, inflights)
    c, vt = TV.state_of(s)
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
        _check_columns(a, c, vt, s.n, ins=True)
    table, role, leader = s.table.copy(), s.role.copy(), s.leader.copy()
    kinds = np.zeros(16, np.int64)
    for rnd in range(2):
        frames_ = T.frames(rng, s, per_group=(1, 3)) + _noise(rng, s, 3000)
        frames_ = [frames_[i] for i in rng.permutation(len(frames_))]
        blob, off = F.batch(frames_)
        want = FT.batch(c, q, vt, blob, off, table)
        got = _run(a, frames_, table, device)
        _equal(want, got, rnd)
        _check_columns(a, c, vt, s.n, ins=bool(inflights))
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
    got = _run(a, frames_, t, device)
    _equal(want, got, "hostile")
    _check_columns(a, c, vt, 4)
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
    got = _run(a, frames_, t, device)
    _equal(want, got, "one group")
    _check_columns(a, c, vt, 2)
    st = got[0]
    assert c.term[1] == terms.max() and np.count_nonzero(st & B.FTERM_BUMPED) == 1
    assert np.flatnonzero(st & B.FTERM_BUMPED)[0] == np.flatnonzero(terms == terms.max())[0]
    assert np.count_nonzero(st >> 4 == B.WIRE_STALE) == np.count_nonzero(terms < terms.max())
    a.close()


def test_no_frames():
    a, c, vt, t = _small(2)
    st, out, rb, ro, tot = _device(a, np.zeros(0, np.uint8), np.zeros(1, np.uint32), t)
    assert st.size == 0 and tot.tolist() == [0, 0] and ro.tolist() == [0]
    st, out, rb, ro, tot = a.follower_term_wire(F.Frames([]), t)
    assert st.size == 0 and tot.tolist() == [0, 0] and ro.tolist() == [0]
    _check_columns(a, c, vt, 2)
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
    d_b, d_o, d_v = a.device_alloc(len(blob)), a.device_alloc(4 * (n + 1)), a.device_alloc(t.nbytes + 64)
    d_st, d_out, d_rb, d_ro, d_t = (a.device_alloc(x) for x in (n, 16 * n, bound + 16, 4 * (n + 1), 16))
    for p, x in ((d_b, blob), (d_o, off), (d_v, t), (d_st, np.full(n, 0xEE, np.uint8)), (d_t, np.full(2, 77, np.uint64))):
        a.h2d(p, x)
    nb = off[-1]
    dev = lambda **k: L.raftgpu_follower_term_wire_device(
        h, None, k.get("b", d_b), k.get("nb", nb), k.get("o", d_o), k.get("n", n), k.get("v", d_v), k.get("st", d_st),
        k.get("out", d_out), k.get("rb", d_rb), k.get("cap", bound), k.get("ro", d_ro), k.get("t", d_t))
    refused = [dev(cap=bound - 1), dev(b=d_b + 4), dev(v=d_v + 8), dev(rb=d_rb + 4), dev(nb=1 << 32),
               dev(n=1 << 32, cap=1 << 40), dev(n=(1 << 32) // 39 + 1, cap=1 << 40), dev(v=None), dev(st=None),
               dev(b=None), dev(o=None), dev(rb=None), dev(t=None), dev(ro=None)]
    assert refused == [B.ERR_INVALID] * len(refused), refused
    a.synchronize()
    gst, gt = np.zeros(n, np.uint8), np.zeros(2, np.uint64)
    a.d2h(gst, d_st), a.d2h(gt, d_t)
    assert np.all(gst == 0xEE) and gt.tolist() == [77, 77]                    # nothing was launched
    assert np.all(a.column_read(B.COL_TERM, 0, 0, 16, np.uint64) == 3)
    st, out, rb, ro, tot = np.zeros(n, np.uint8), np.zeros(2 * n, np.uint64), np.zeros(bound, np.uint8), \
        np.zeros(n + 1, np.uint32), np.zeros(2, np.uint64)
    assert L.raftgpu_follower_term_wire(h, blob.ctypes.data, nb, off.ctypes.data, n, t.ctypes.data, st.ctypes.data,
                                        out.ctypes.data, rb.ctypes.data, bound - 1, ro.ctypes.data, tot.ctypes.data) == B.ERR_INVALID
    assert L.raftgpu_follower_term_wire(h, blob.ctypes.data, nb, off.ctypes.data, n, None, st.ctypes.data,
                                        out.ctypes.data, rb.ctypes.data, bound, ro.ctypes.data, tot.ctypes.data) == B.ERR_INVALID
    assert dev() == B.OK                                                      # the same call with every rule kept
    a.synchronize()
    a.d2h(gst, d_st)
    assert np.all(gst == (B.WIRE_OK << 4 | B.FTERM_BUMPED)) and np.all(a.column_read(B.COL_TERM, 0, 0, 16, np.uint64) == 4)
    a.close()


# --------------------------------------------------------------------------- 3. round trips


def _leaders(n, P, term, li):
    """n narrow leader groups of P voters (self slot 0) at `term`: the empty entry at li + 1 = term_start, committed li,
    every peer a Replicate peer matched at li that was sent the empty entry (next li + 2), and the earlier run [1, li]
    at term - 1 stated."""
    a = B.Arena(n + 64)
    a.enable_leader_runs()
    assert a.group_alloc_range(n) == 0
    ops = []
    for g in range(n):
        ops += [(B.CTL_SET_CONF, g, 0, 0, ((1 << P) - 1, 0, 0, li + 1)), (B.CTL_RESET, g, 0, 0, (li + 1, li, li, li)),
                (B.CTL_SET_TERM, g, 0, 0, (term,)), (B.CTL_BECOME_LEADER, g)]
        for s in range(1, P):
            ops += [(B.CTL_PROGRESS_OP, g, s, B.POP_MAYBE_UPDATE, (li,)), (B.CTL_PROGRESS_OP, g, s, B.POP_BECOME_REPLICATE),
                    (B.CTL_PROGRESS_OP, g, s, B.POP_OPTIMISTIC_UPDATE, (li + 1,))]
    assert np.all(a.control(cmds(*ops))["status"] == 0)
    rows = np.zeros(n, B.LEADER_RUNS_DTYPE)
    rows["group"], rows["term"], rows["term_start"] = np.arange(n), term, li + 1
    rows["run_start"][:, 0], rows["run_term"][:, 0] = 1, term - 1
    assert np.all(a.leader_runs_set(rows) == 0)
    return a


def _to_followers(blob, off, P):
    """The transport: leader cell (g, s) -> follower group g * (P - 1) + s - 1, x = s."""
    h = HB.headers(blob, off)
    return HB.with_headers(blob, off, (((h >> 4) * (P - 1) + (h & 15) - 1) << 4 | (h & 15)).astype(np.uint32))


def _to_leaders(blob, off, P):
    h = HB.headers(blob, off)
    return HB.with_headers(blob, off, (((h >> 4) // (P - 1)) << 4 | (h & 15)).astype(np.uint32))


def _followers(nf, term, li, P, rng):
    fa = B.Arena(nf + 64)
    assert fa.group_alloc_range(nf) == 0
    fcom = (li - rng.integers(0, 4, nf)).astype(np.uint64)
    for col, arr in ((B.COL_TERM, np.full(nf, term, np.uint64)), (B.COL_LAST_INDEX, np.full(nf, li, np.uint64)),
                     (B.COL_COMMITTED, fcom), (B.COL_TERM_START, np.full(nf, B.NO_TERM_START, np.uint64))):
        fa.column_write(col, 0, 0, arr)
    table = Q.voters(nf)
    table["id"] = np.arange(nf) % (P - 1) + 2
    table["persisted"], table["last_term"] = li, term
    table["flags"] = B.VOTER_SELECT | B.VOTER_STALE_REPLY
    return fa, table


def test_restart_round_trip():
    """A store restarts: its 20K x 4 follower groups are at term t, their leaders (5 voters) were elected at t + 1 and
    appended their empty entry.  The leaders' raftgpu_heartbeat_frames and raftgpu_append_frames go through this pass,
    then raftgpu_follower_heartbeat, then raftgpu_follower_append; the responses come back through
    raftgpu_heartbeat_wire and raftgpu_step_begin_wire.  Every follower ends at t + 1 with its leader's committed, the
    append is rejected at the follower's last index and decided from the leader's stated run, and no frame is the
    host's on either side."""
    rng = np.random.default_rng(0x7402)
    n, P, t, li = 20_000, 5, 7, 1000
    la = _leaders(n, P, t + 1, li)
    ids = np.zeros((B.SLOTS + 1, n), np.uint64)
    ids[:B.SLOTS] = (np.arange(B.SLOTS) + 1)[:, None]
    ids[B.SLOTS] = 1
    _, hb, hoff, htot = la.heartbeat_frames(0, n, ids)
    _, ap, aoff, _, atot = la.append_frames(0, n, ids)
    assert int(htot[0]) == int(atot[0]) == n * (P - 1)
    frames_ = HB.frames_of(_to_followers(hb, hoff, P), hoff) + HB.frames_of(_to_followers(ap, aoff, P), aoff)
    frames_ = [np.array([h], "<u4").tobytes() + b for h, b in frames_]
    frames_ = [frames_[i] for i in rng.permutation(len(frames_))]
    nf = n * (P - 1)
    fa, table = _followers(nf, t, li, P, rng)
    blob, off = F.batch(frames_)
    st, out, _, _, tot = _device(fa, blob, off, table)
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
    lst, _ = la.heartbeat_wire(F.Frames([bytes(x) for x in np.split(_to_leaders(hrb, hro, P), hro[1:-1])]))
    assert np.all(lst >> 4 == B.WIRE_OK)
    back = _to_leaders(arb, aro, P)
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
    old = _leaders(n, P, t, li)
    ids = np.zeros((B.SLOTS + 1, n), np.uint64)
    ids[:B.SLOTS] = (np.arange(B.SLOTS) + 1)[:, None]
    ids[B.SLOTS] = 1
    _, hb, hoff, _ = old.heartbeat_frames(0, n, ids)
    nf = n * (P - 1)
    fa, table = _followers(nf, t + 1, li, P, rng)
    quiet = rng.random(nf) < 0.25
    table["flags"][quiet] = B.VOTER_SELECT
    to_f = _to_followers(hb, hoff, P)
    st, out, rb, ro, tot = _device(fa, to_f, hoff, table)
    g = HB.headers(to_f, hoff) >> 4
    assert np.array_equal(st, np.where(quiet[g], B.WIRE_STALE << 4, B.WIRE_STALE << 4 | B.RES_OK).astype(np.uint8))
    assert int(tot[0]) == np.count_nonzero(~quiet) and not out.any()
    assert np.all(fa.column_read(B.COL_TERM, 0, 0, nf, np.uint64) == t + 1)
    for k in range(0, int(tot[0]), 997):
        m = O.wire_decode_message(rb[ro[k] + 4:ro[k + 1]].tobytes())
        assert (m["msg_type"], m["to"], m["term"], m["index"], m["commit"], m["reject"]) == (4, 1, t + 1, 0, 0, 0)
    fa.close()
    before = old.read_columns(n)
    back = _to_leaders(rb, ro, P)
    old.step_begin_wire(F.Frames([bytes(back[a0:b0]) for a0, b0 in zip(ro[:-1].tolist(), ro[1:].tolist())]),
                        B.STEP_READ_COMMITTED)
    old.step_wait()
    assert np.all(old.wire_status() >> 4 == B.WIRE_TERM)
    after = old.read_columns(n)
    for name in ARENA_COLUMNS:
        assert np.array_equal(getattr(before, name), getattr(after, name)), name
    old.close()
