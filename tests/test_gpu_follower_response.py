"""The responses that reach a follower or a candidate on the GPU (raftgpu_follower_response_wire[_device]) and the
candidate's step-down in raftgpu_follower_term_wire, against the two batch forms of oracle/follow_resp_oracle.c byte
for byte: random 40K-group bursts with wide pairs in both forms, on arenas with read queues and with Inflights,
frames across the shared-memory stage, n = 0 and the refusals; then one partition-heal buffer through the documented
pass order.  Run with -m gpu."""
import numpy as np
import pytest

from oracle import oracle as O
from oracle import control_oracle as CO
from oracle import follow_resp_oracle as FR
from oracle import read_oracle as RO
from oracle import vote_wire_oracle as VW
from helpers import B, arena_of, check_columns
from control_cmds import cmds
import follow_resp as R
import follow_term as T
import hb_follow as HB
import hb_frames as F
import leader_term as L
import pass_forms as PF
import vote_request_frames as Q
import wire_batches as WB

pytestmark = pytest.mark.gpu

NAMES = ("status", "out")
TERM_NAMES = ("status", "out", "bytes", "offsets", "totals")


def _setup(rng, n_narrow, n_wide, read_index, inflights, p_role=(0.4, 0.2, 0.3, 0.1)):
    s = R.scenario(rng, n_narrow, n_wide, p_role=p_role)
    a = arena_of(s, read_index, inflights)
    c, vt = Q.state_of(s)
    q = None
    if read_index:
        q = RO.ReadQueues(c.cap, 8)
        q.allocated[: s.n] = 1
    if inflights:
        O.enable_inflights(c, inflights)
        adds = cmds(*[(B.CTL_PROGRESS_OP, int(g), int(sl), B.POP_INS_ADD, (int(s.last[g]) + k,))
                      for g in rng.choice(s.lows, 20_000) for sl in (1, 2) for k in (1, 2)])
        assert np.array_equal(a.control(adds), CO.arena_control(c, vt, adds))
        check_columns(a, c, vt, s.n, ins=True)
    return s, a, c, vt, q


# --------------------------------------------------------------------------- 1. random bursts


@pytest.mark.parametrize("device,read_index,inflights", [(False, False, 0), (True, False, 0), (True, True, 0),
                                                         (False, False, 4), (True, False, 4)],
                         ids=["host", "device", "device-read-queues", "host-inflights", "device-inflights"])
def test_responses_vs_oracle(device, read_index, inflights):
    """Deposed leaders' late 4 / 9, lost candidates' late 6 / 18 and higher-term rejections at (Pre)Candidates."""
    rng = np.random.default_rng(0x7700 + 4 * device + 2 * read_index + (inflights > 0))
    s, a, c, vt, q = _setup(rng, 40_000, 1_000, read_index, inflights)
    kinds = np.zeros(16, np.int64)
    for rnd in range(2):
        frames_, _ = R.frames(rng, s, per_group=(1, 4))
        frames_ += L.noise(rng, s, 3000)
        frames_ = [frames_[i] for i in rng.permutation(len(frames_))]
        blob, off = F.batch(frames_)
        want = FR.batch(c, q, vt, blob, off, s.table)
        got = PF.run(a, "follower_response_wire", blob, off, s.table, device=device)
        PF.equal(want, got, NAMES, rnd)
        check_columns(a, c, vt, s.n, ins=bool(inflights))
        if read_index:
            assert all(len(a.read_index_get(g)[0]) == q.count[g] for g in range(0, s.n, 997))
        s.term[:] = c.term[: s.n]
        kinds += np.bincount(got[0] >> 4, minlength=16)
    for k in (B.WIRE_OK, B.WIRE_STALE, B.WIRE_IGNORED, B.WIRE_ROLE, B.WIRE_TERM, B.WIRE_SKIP_TYPE, B.WIRE_MALFORMED):
        assert kinds[k] > 100, (k, kinds)
    a.close()


@pytest.mark.parametrize("device,read_index,inflights", [(False, False, 0), (True, False, 0), (True, True, 0),
                                                         (True, False, 4)],
                         ids=["host", "device", "device-read-queues", "device-inflights"])
def test_step_downs_vs_oracle(device, read_index, inflights):
    """raftgpu_follower_term_wire with the candidate flags: step-downs at the term, bumps above it, stale replies."""
    rng = np.random.default_rng(0x7710 + 4 * device + 2 * read_index + (inflights > 0))
    s, a, c, vt, q = _setup(rng, 40_000, 1_000, read_index, inflights, p_role=(0.3, 0.3, 0.3, 0.1))
    frames_ = T.frames(rng, s, per_group=(1, 3), deltas=(-1, 0, 0, 0, 1)) + T.noise(rng, s, 3000)
    frames_ = [frames_[i] for i in rng.permutation(len(frames_))]
    blob, off = F.batch(frames_)
    want = FR.term_batch(c, q, vt, blob, off, s.table)
    got = PF.run(a, "follower_term_wire", blob, off, s.table, device=device)
    PF.equal(want, got, TERM_NAMES, "step-downs")
    check_columns(a, c, vt, s.n, ins=bool(inflights))
    if read_index:
        assert all(len(a.read_index_get(g)[0]) == q.count[g] for g in range(0, s.n, 997))
    st = got[0]
    assert np.count_nonzero(st & 0xF == B.FTERM_STEPPED) > 500 and np.count_nonzero(st & 0xF == B.FTERM_BUMPED) > 500
    a.close()


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_across_the_stage(device):
    """Both passes over frames interleaved with ballast so that blocks cross the shared-memory stage's edges."""
    rng = np.random.default_rng(0x7720 + device)
    s, a, c, vt, _ = _setup(rng, 10_000, 500, False, 0)
    frames_, _ = R.frames(rng, s, per_group=(1, 2))
    frames_ += T.frames(rng, s, per_group=(0, 1), deltas=(-1, 0, 0, 1))
    frames_ = [frames_[i] for i in rng.permutation(len(frames_))]
    frames_, ballast = WB.across_the_stage(frames_, rng)
    blob, off = F.batch(frames_)
    want = FR.batch(c, None, vt, blob, off, s.table)
    got = PF.run(a, "follower_response_wire", blob, off, s.table, device=device)
    PF.equal(want, got, NAMES, "stage")
    assert np.all(got[0][ballast] == B.WIRE_SKIP_TYPE << 4)
    want = FR.term_batch(c, None, vt, blob, off, s.table)
    got = PF.run(a, "follower_term_wire", blob, off, s.table, device=device)
    PF.equal(want, got, TERM_NAMES, "stage, term")
    check_columns(a, c, vt, s.n)
    a.close()


# --------------------------------------------------------------------------- 2. edges


def test_no_frames_and_refusals():
    rng = np.random.default_rng(0x7730)
    s, a, c, vt, _ = _setup(rng, 16, 0, False, 0, p_role=(0.4, 0.3, 0.3, 0.0))
    st, out = PF.device(a, "follower_response_wire", np.zeros(0, np.uint8), np.zeros(1, np.uint32), s.table)
    assert st.size == 0 and out.size == 0
    st, out = a.follower_response_wire(F.Frames([]), s.table)
    assert st.size == 0 and out.size == 0
    Lb, h = a._L, a._h
    n = 16
    blob, off = F.batch([F.frame(g, 1, F.message(4, int(s.term[g]) + 1, frm=2)) for g in range(n)])
    blob = np.concatenate([blob, np.zeros(16, np.uint8)])
    t = Q.voters(64)
    t["flags"] = B.VOTER_SELECT
    with PF.device_buffers(a) as put:
        d_b, d_o, d_v = put(len(blob), blob), put(off.nbytes, off), put(t.nbytes, t)
        d_st, d_out = put(n, fill=np.full(n, PF.STATUS_SENTINEL, np.uint8)), put(8 * n)
        nb = int(off[-1])

        def dev(b=d_b, nbytes=nb, o=d_o, k=n, v=d_v, st_=d_st, out_=d_out):
            return Lb.raftgpu_follower_response_wire_device(h, None, b, nbytes, o, k, v, st_, out_)

        refused = [dev(b=d_b + 4), dev(v=d_v + 8), dev(nbytes=1 << 32), dev(k=1 << 32), dev(v=None), dev(st_=None),
                   dev(b=None), dev(o=None), Lb.raftgpu_follower_response_wire_device(None, None, d_b, nb, d_o, n, d_v,
                                                                                      d_st, d_out)]
        assert refused == [B.ERR_INVALID] * len(refused), refused
        a.synchronize()
        got = np.zeros(n, np.uint8)
        a.d2h(got, d_st)
        assert np.all(got == PF.STATUS_SENTINEL)                              # nothing was launched
        st, out = np.zeros(n, np.uint8), np.zeros(n, np.uint64)
        assert Lb.raftgpu_follower_response_wire(h, blob.ctypes.data, nb, off.ctypes.data, n, None, st.ctypes.data,
                                                 out.ctypes.data) == B.ERR_INVALID
        assert dev() == B.OK                                                  # the same call with every rule kept
        a.synchronize()
        a.d2h(got, d_st)
        want, _ = FR.batch(c, None, vt, blob[:nb], off, t)
        assert np.array_equal(got, want) and np.all(got == B.WIRE_OK << 4 | B.FTERM_BUMPED)
    check_columns(a, c, vt, s.n)
    a.close()


# --------------------------------------------------------------------------- 3. one partition-heal buffer


def test_partition_heal_buffer_through_the_pass_order():
    """A store whose groups were cut off hears, in one buffer, the late responses of the leadership and elections it
    lost, higher-term rejections, and the new leaders' MsgAppend / MsgHeartbeat at, above and below each group's term.
    On the device: raftgpu_follower_response_wire and its host side, raftgpu_follower_term_wire and its host side,
    then raftgpu_vote_wire over the frames left to it -- each against its batch oracle.  (The store leads no group, so
    the leader passes and raftgpu_leader_term_wire find nothing.)  No frame of types 3, 4, 6, 8, 9 or 18 to a selected
    group is left to the host but under the statuses the header names: vote_wire's DUP and COMMIT_VOTE.  A response
    left OK whose group step 2 steps down or bumps is settled: the step-down comes first in the reference's order."""
    rng = np.random.default_rng(0x7740)
    s, a, c, vt, _ = _setup(rng, 20_000, 500, False, 4, p_role=(0.4, 0.3, 0.3, 0.0))
    resp, _ = R.frames(rng, s, per_group=(1, 4), deltas=(-1, 0, 0, 0, 1, 2))
    app = T.frames(rng, s, per_group=(0, 2), deltas=(-1, 0, 0, 1))
    frames_ = [x for x in resp + app]
    frames_ = [frames_[i] for i in rng.permutation(len(frames_))]
    blob, off = F.batch(frames_)
    n = len(frames_)
    table, role, leader = s.table.copy(), s.role.copy(), s.leader.copy()
    # 1. the responses
    want = FR.batch(c, None, vt, blob, off, table)
    rst, rout = a.follower_response_wire(PF.host_batch(blob, off), table)
    PF.equal(want, (rst, rout), NAMES, "responses")
    lows = np.array([(lambda g: g - 1 if g >= s.n_narrow and (g - s.n_narrow) % 2 else g)(int(h >> 4))
                     for h in HB.headers(blob, off)])
    R.host_side(table, role, leader, rst, rout, lows)
    # 2. the term prefix of MsgAppend / MsgHeartbeat, with the step-down
    want = FR.term_batch(c, None, vt, blob, off, table)
    got = a.follower_term_wire(PF.host_batch(blob, off), table)
    PF.equal(want, got, TERM_NAMES, "term")
    tst = got[0]
    R.term_host_side(table, role, leader, tst, got[1], frames_)
    check_columns(a, c, vt, s.n, ins=True)
    # 3. raftgpu_vote_wire over the frames the response pass left OK, but for the groups step 2 made Followers: their
    # step-down comes first, and step_follower drops the responses (settled, as IGNORED)
    typ = T.types_of(frames_)
    moved = {int(lows[i]) for i in np.flatnonzero(tst & (B.FTERM_BUMPED | B.FTERM_STEPPED))}
    ok = [i for i in range(n) if typ[i] in (6, 18) and rst[i] == B.WIRE_OK << 4]
    left = [i for i in ok if int(lows[i]) not in moved]
    assert len(left) > 300 and len(ok) > len(left)
    sel = HB.bitmap(np.isin(role, (Q.PRE_CANDIDATE, Q.CANDIDATE)))
    pre = HB.bitmap(role == Q.PRE_CANDIDATE)
    vb, vo = F.batch([frames_[i] for i in left])
    vst, vout, _ = VW.batch(c, vt, vb, vo, sel, pre)
    gst, gout = a.vote_wire(F.Frames([frames_[i] for i in left]), sel, pre)
    assert np.array_equal(vst, gst) and np.array_equal(vout, gout)
    check_columns(a, c, vt, s.n, ins=True)
    # what went back to the host
    final = np.where(np.isin(typ, (3, 8)), tst, rst)
    final[[i for i in ok if i not in set(left)]] = B.WIRE_IGNORED << 4
    final[left] = gst
    selected = np.array([bool(s.table["flags"][g] & B.VOTER_SELECT) for g in lows])
    host = (final >> 4 != B.WIRE_OK) & (final >> 4 != B.WIRE_IGNORED) & (final >> 4 != B.WIRE_STALE)
    assert set((final[host & selected] >> 4).tolist()) <= {B.WIRE_DUP, B.WIRE_COMMIT_VOTE}
    assert np.all(final[host & ~selected] >> 4 == B.WIRE_ROLE)
    assert np.count_nonzero(rst & B.FTERM_BUMPED) > 300 and np.count_nonzero(tst & 0xF == B.FTERM_STEPPED) > 300
    a.close()
