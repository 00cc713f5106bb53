"""The five kernels that re-encode next_idx and peer_committed after the 16-bit offset tests were written, at the edges
of that window, with device Inflights windows filled, against the batch oracles byte for byte:

- vrq_apply_kernel, ftm_apply_kernel and ltm_apply_kernel (raftgpu_vote_request_wire, raftgpu_follower_term_wire and
  raftgpu_leader_term_wire, host and device forms), whose bumps reset every cell of a group (become_follower_arena,
  reset_group): each bumped group resets onto the bounds of term_wave16.bump_edges16, its full windows and read queues
  emptied;
- wire_wave_apply_kernel<false> and <true> (the wire step at 2, 4 and RAFTGPU_WIRE_WAVES_MAX waves, without and with
  leader runs, each through raftgpu_wire_apply_device and raftgpu_step_begin_wire), where a wave starts from the cells the
  wave before it left: offsets moved out of the window and back within one call, full windows freed by frames of
  wave 2 and later (term_wave16.wave_world).

Statuses, outs, replies, totals, every column, the windows, the read queues and the vote bytes are compared; that
every transition occurred is asserted from the oracle's columns, with its count.  The generators are checked on the
CPU by test_term_wave_edges.py.  Run with -m gpu."""
import numpy as np
import pytest

from helpers import B, O, assert_columns_equal
from oracle import control_oracle as CO
from oracle import wire_waves_oracle as WW
import hb_frames as F
import term_wave16 as W
import test_gpu_append_reject as GAR
import test_gpu_follower_term as GT
import test_gpu_leader_term as GL
import test_gpu_vote_request_wire as GV
import test_gpu_wire_batches as WBT

pytestmark = pytest.mark.gpu

# sizes that keep every transition's count well above W.FLOOR (test_term_wave_edges.py checks the generators at
# smaller ones) and the file's wall time near a minute
N_NARROW, N_WIDE, N_LEADERS = 6_000, 200, 6_000
RUN = {"vote_request": GV._run, "follower_term": GT._run, "leader_term": GL._run}


def _check_windows(a, c, n, rng, k=400):
    """Every cell's window word, and the ring of k random cells with a window."""
    for s in range(O.SLOTS):
        assert np.array_equal(a.column_read(B.COL_INS_META, s, 0, n, np.uint32), c.ins_meta[s, :n]), s
    ss, gs = np.nonzero((c.ins_meta[:, :n] >> 16) > 0)
    for i in rng.choice(len(gs), min(k, len(gs)), replace=False) if len(gs) else ():
        start, cnt, ring = a.inflights_get(int(gs[i]), int(ss[i]))
        m = int(c.ins_meta[ss[i], gs[i]])
        assert (start, cnt) == (m & 0xFFFF, m >> 16) and np.array_equal(ring, c.ins_buf[ss[i], gs[i]])


def _check_reads(a, q, lows):
    for g in lows:
        ctx, idx, acks = a.read_index_get(g)
        wctx, widx, wacks = q.pending(g)
        assert np.array_equal(ctx, wctx) and np.array_equal(idx, widx) and np.array_equal(acks, wacks), g


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("name", sorted(RUN))
def test_bumps_reset_onto_the_16bit_edges(name, device):
    rng = np.random.default_rng(0x16D0 + 2 * sorted(RUN).index(name) + device)
    s, c, vt, q, fill, reqs = W.bump_world(rng, name, N_NARROW, N_WIDE)
    a = B.Arena(s.n + 64)
    a.enable_inflights(W.INS_CAP)
    a.enable_read_index()
    assert a.group_alloc_range(s.n_narrow) == 0
    for k in range(s.n_wide):
        assert a.group_alloc_wide() == s.n_narrow + 2 * k
    assert np.all(a.control(s.setup)["status"] == 0)
    a.load_columns(c)
    assert np.all(a.control(fill)["status"] == 0)
    res, _ = a.read_index_request(reqs)
    assert (res == B.READ_QUEUED).sum() > 100
    GT._check_columns(a, c, vt, s.n, ins=True)
    _check_reads(a, q, s.lows)
    before, q0 = O.copy_columns(c), q.copy()
    frames_ = W.bump_frames(rng, s, name)
    frames_ += (GL._noise if name == "leader_term" else GT._noise)(rng, s, 250)
    blob, off = F.batch(frames_)
    want = W.BATCH[name](c, q, vt, blob, off, s.table)
    got = RUN[name](a, frames_, s.table, device)
    GT._equal(want, got, name)
    GT._check_columns(a, c, vt, s.n, ins=True)
    assert_columns_equal(a.read_columns(s.n), c, s.n, name)
    _check_windows(a, c, s.n, rng)
    _check_reads(a, q, s.lows)
    counts = W.bump_counts(before, c, W.persisted_of(s), s.n, q0, q)
    W.check_bump_counts(counts, name)
    a.close()


@pytest.mark.parametrize("runs", [False, True], ids=["no_runs", "runs"])
def test_wave_kernels_at_the_16bit_edges_with_inflights(runs):
    """6K leaders x 5 peers, 2-6 scripted frames per cell, at waves 2, 4 and RAFTGPU_WIRE_WAVES_MAX, each through
    raftgpu_wire_apply_device and through raftgpu_step_begin_wire, each on a new arena."""
    rng = np.random.default_rng(0x16E0 + runs)
    n = N_LEADERS
    for waves, form in ((w, f) for w in (2, 4, B.WIRE_WAVES_MAX) for f in ("device", "host")):
        what = f"{form}, waves {waves}"
        c, rows, fill, blob, off, _ = W.wave_world(rng, n)
        a = B.Arena(n)
        a.enable_inflights(W.INS_CAP)
        if runs:
            a.enable_leader_runs()
        assert a.group_alloc_range(n) == 0
        a.load_columns(c)
        a.column_write(B.COL_TERM, 0, 0, c.term[:n].copy())
        if runs:
            assert np.all(a.leader_runs_set(rows) == 0)
        O.enable_inflights(c, W.INS_CAP)
        assert np.array_equal(a.control(fill), CO.arena_control(c, np.zeros((O.SLOTS, c.cap), np.uint8), fill))
        r = rows if runs else None
        counts = W.wave_counts(c, r, blob, off, waves, WW.leader)
        assert a.set_wire_waves(waves) == 0
        want = WW.leader(c, r, blob, off, waves)
        if form == "device":
            got = GAR._apply_device(a, blob, off)
        else:
            a.step_begin_wire(WBT._host_batch(blob, off, len(blob)), B.STEP_READ_COMMITTED)
            a.step_wait()
            got = a.wire_status().copy()
            O.arena_recompute(c)
        bad = np.flatnonzero(got != want)
        assert len(bad) == 0, (what, [(int(i), hex(got[i]), hex(want[i])) for i in bad[:5]])
        assert_columns_equal(a.read_columns(n), c, n, what)
        _check_windows(a, c, n, rng)
        for k, v in counts.items():
            assert v >= W.FLOOR, (what, k, counts)
        a.close()
