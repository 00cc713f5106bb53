"""The commit broadcast's entry-less MsgAppend frames built on the GPU (raftgpu_append_frames[_device]), byte-equal to
the oracle (oracle/app_frames_oracle.c) in frames, offsets, rest list and totals: random arenas of every configuration
with and without device Inflights, 1M groups after steps of synthetic traffic selected by the step's advanced bitmap,
next_idx on the edges of the 16-bit offset window, the pass's read-only contract, short capacities, the refusals, the
frames fed back to a wire step, and the host form between a begin and its wait.  Run with -m gpu."""
import numpy as np
import pytest

from oracle import app_frames_oracle as AF
from helpers import B
import app_frames as A
import hb_frames as F
import pass_forms as PF
import offset16 as E

pytestmark = pytest.mark.gpu

ENTRY = ["group", "peer_slot", "flags", "next_idx"]


def _check(a, c, first, n, ids, select, what):
    """Host and device forms against the oracle over the arena's own columns c; returns the oracle's output."""
    want = AF.bcast_append(c, None, first, n, ids, select)
    rc, blob, off, rest, tot = a.append_frames(first, n, ids, select)
    assert rc == B.OK, what
    assert tot.tolist() == want[3].tolist(), (what, tot, want[3])
    assert np.array_equal(off, want[1]), what
    assert np.array_equal(blob, want[0]), (what, int(np.argmax(blob != want[0])) if len(blob) == len(want[0]) else None)
    assert np.array_equal(rest, want[2]), what
    dblob, doff, drest, dtot = PF.broadcast(a, "append_frames", first, n, ids, select)
    assert dtot.tolist() == tot.tolist() and np.array_equal(doff, off) and np.array_equal(dblob, blob), what
    assert np.array_equal(drest, rest), what
    return want


def _columns_equal(x, y):
    for name in ("matched", "next_idx", "peer_committed", "pending_snapshot", "pending_request_snapshot", "pflags", "meta",
                 "committed", "term_start", "last_index"):
        assert np.array_equal(getattr(x, name), getattr(y, name)), name


def _arena(c, n, inflights=False):
    """A GPU arena holding host columns c (groups [0, n), c.term included); returns (arena, its columns read back)."""
    a = B.Arena(c.cap)
    if inflights:
        a.enable_inflights(16)
    assert a.group_alloc_range(n) == 0
    a.load_columns(c)
    a.column_write(B.COL_TERM, 0, 0, c.term[:n].copy())
    got = a.read_columns(n)
    got.cap, got.n_groups = c.cap, n
    _columns_pad(got, c)
    return a, got


def _columns_pad(got, c):
    """read_columns gives [n]-wide arrays: the oracle's view wants the cap-wide layout of c."""
    for name in ("matched", "next_idx", "peer_committed", "pending_snapshot", "pending_request_snapshot", "commit_group_id",
                 "pflags"):
        full = np.zeros_like(getattr(c, name))
        full[:, :got.n_groups] = getattr(got, name)
        setattr(got, name, full)
    for name in ("meta", "committed", "term_start", "last_index"):
        full = np.zeros_like(getattr(c, name))
        full[:got.n_groups] = getattr(got, name)
        setattr(got, name, full)
    got.term = c.term.copy()


# --------------------------------------------------------------------------- 1. random arenas

@pytest.mark.parametrize("inflights", [False, True], ids=["host_inflights", "device_inflights"])
def test_random_arenas_vs_oracle(inflights):
    rng = np.random.default_rng(0xA9F + inflights)
    n, n_wide = 60_000, 800
    c = A.random_columns(rng, n, n_wide)
    a, ac = _arena(c, n, inflights)
    before = a.read_columns(n)
    sel = A.select_bits(rng, c.cap, 0.3)
    narrow = n - 2 * n_wide
    ranges = [(0, n, None), (0, n, sel), (12_345, narrow - 12_345 + 2 * 77, sel), (4_097, 2_001, None),
              (narrow + 2 * 10, 2 * 40, sel), (0, c.cap, None), (n, c.cap - n, None)]
    kinds = np.zeros(4)
    for first, m, s in ranges:
        ids = A.ids_for(rng, m)
        want = _check(a, ac, first, m, ids, s, (first, m, s is not None))
        kinds += want[3]
        # the frames and the rest list partition the send list of the same selection over the groups that send
        cells = A.frame_cells(want[0], want[1]) + [tuple(x) for x in want[2][["group", "peer_slot"]].tolist()]
        sl = A.send_list_of_senders(ac, first, m, s)
        assert sorted(cells) == sorted(tuple(x) for x in sl[["group", "peer_slot"]].tolist()), (first, m)
    assert kinds[0] > 50_000 and kinds[2] > 50_000 and kinds[3] > 1_000, kinds
    _columns_equal(a.read_columns(n), before)   # read-only
    a.close()


# --------------------------------------------------------------------------- 2. 1M groups after synthetic traffic

def test_1m_groups_after_steps():
    n = 1_000_000
    s = B.Synth(n, 0xA9F1, k_peers=5)
    a = B.Arena(n)
    assert a.group_alloc_range(n) == 0
    a.load_columns(s.initial)
    rng = np.random.default_rng(7)
    terms = rng.integers(1, 1000, n).astype(np.uint64)
    a.column_write(B.COL_TERM, 0, 0, terms)
    for _ in range(3):
        a.step_begin_records(s.next_round().copy(), B.STEP_READ_COMMITTED)
        a.step_wait()
    bm = a.step_results(n)[0].copy()
    sl = a.step_send_list(8 * n)
    c = a.read_columns(n)
    c.term = terms.copy()
    ids = A.ids_for(rng, n)
    want = _check(a, c, 0, n, ids, bm, "1M")
    assert int(want[3][2]) > n // 10, want[3]
    cells = A.frame_cells(want[0], want[1]) + [tuple(x) for x in want[2][["group", "peer_slot"]].tolist()]
    assert sorted(cells) == sorted(tuple(x) for x in sl[["group", "peer_slot"]].tolist())
    # every follower caught up: all frames, no rest entries
    c.next_idx[:] =c.last_index[None, :] + 1
    for k in range(B.SLOTS):
        a.column_write(B.COL_NEXT_IDX, k, 0, c.next_idx[k].copy())
    c.pflags[:] = np.where((c.pflags & 3) == B.STATE_SNAPSHOT, c.pflags, B.STATE_REPLICATE)
    for k in range(B.SLOTS):
        a.column_write(B.COL_PFLAGS, k, 0, c.pflags[k].copy())
    want = _check(a, c, 0, n, ids, None, "1M caught up")
    assert int(want[3][0]) > 3 * n and np.all(want[2]["flags"] == B.SEND_SNAPSHOT), want[3]
    a.close()


# --------------------------------------------------------------------------- 3. the 16-bit offset window

def test_offset16_edges():
    """next_idx escaped or on the window's bounds, last_index around 2^15, so that next_idx = last_index + 1 crosses the
    bound both ways."""
    rng = np.random.default_rng(0xA916)
    n = 20_000
    c = A.random_columns(rng, n, 100, base=np.full(n, 3, np.uint64))
    E.edge_state16(c, rng, 0.4, n)
    half = rng.random((8, n)) < 0.5
    last = np.array(E.RESET16_LAST[:3] + (2 ** 15 + 1,), np.uint64)[rng.integers(0, 4, n)]
    c.last_index[:n] = last
    nx = last[None, :] + rng.integers(0, 3, (8, n)).astype(np.uint64)
    c.next_idx[:, :n] = np.where(half, nx, c.next_idx[:, :n])
    c.matched[:, :n] = np.where(half, rng.choice(np.array([0, 1], np.uint64), (8, n)), c.matched[:, :n])
    c.pflags[:, :n] = np.where(half, B.STATE_REPLICATE, c.pflags[:, :n])
    a, ac = _arena(c, n)
    assert E.escaped16(ac, n).sum() > 10_000 and (~E.escaped16(ac, n)).sum() > 10_000
    want = _check(a, ac, 0, n, A.ids_for(rng, n), None, "offset16")
    assert int(want[3][0]) > 10_000 and int(want[3][2]) > 10_000, want[3]
    a.close()


# --------------------------------------------------------------------------- 4. short capacities, refusals

def _small():
    rng = np.random.default_rng(3)
    n = 256
    c = A.random_columns(rng, n, 8, cap=288)
    a, ac = _arena(c, n)
    return a, ac, n, A.ids_for(rng, n)


def test_short_capacities_write_nothing():
    a, ac, n, ids = _small()
    rc, blob, off, rest, tot = a.append_frames(0, n, ids)
    assert rc == B.OK and min(int(tot[0]), int(tot[2])) > 50
    F_, N_, R_ = int(tot[0]), int(tot[1]), int(tot[2])
    for short in ((1, 0, 0), (0, 1, 0), (0, 0, 1), (1, 1, 1)):
        bout = np.full(N_ + 64, 0xA5, np.uint8)
        oout = np.full(F_ + 8, 0x5A5A5A5A, np.uint32)
        rout = np.zeros(R_ + 8, B.SEND_ENTRY_DTYPE)
        rout["next_idx"] = 0x7777
        rc, _, _, _, t = a.append_frames(0, n, ids, bytes_out=bout, offsets_out=oout, rest_out=rout, bytes_capacity=N_ - short[0],
                                         frames_capacity=F_ - short[1], rest_capacity=R_ - short[2])
        assert rc == B.ERR_FULL and t.tolist() == tot.tolist(), short
        assert np.all(bout == 0xA5) and np.all(oout == 0x5A5A5A5A) and np.all(rout["next_idx"] == 0x7777), short
        # the device form: the canaries in device memory stay as they were
        d_ids, d_bytes, d_off = a.device_alloc(ids.nbytes), a.device_alloc(N_ + 64), a.device_alloc(4 * (F_ + 8))
        d_rest, d_tot = a.device_alloc(rout.nbytes), a.device_alloc(32)
        a.h2d(d_ids, ids), a.h2d(d_bytes, bout), a.h2d(d_off, oout), a.h2d(d_rest, rout)
        a.append_frames_device(0, n, None, d_ids, d_bytes, N_ - short[0], d_off, F_ - short[1], d_rest, R_ - short[2], d_tot)
        a.synchronize()
        gb, go, gr, gt = np.zeros_like(bout), np.zeros_like(oout), np.zeros_like(rout), np.zeros(4, np.uint64)
        a.d2h(gb, d_bytes), a.d2h(go, d_off), a.d2h(gr, d_rest), a.d2h(gt, d_tot)
        assert np.all(gb == 0xA5) and np.all(go == 0x5A5A5A5A) and np.array_equal(gr, rout) and gt.tolist() == tot.tolist()
        for p in (d_ids, d_bytes, d_off, d_rest, d_tot):
            a.device_free(p)
    # the retry with exact capacities succeeds, and nothing is written past them
    bout = np.full(N_ + 64, 0xA5, np.uint8)
    oout = np.full(F_ + 8, 0x5A5A5A5A, np.uint32)
    rout = np.zeros(R_ + 8, B.SEND_ENTRY_DTYPE)
    rout["next_idx"] = 0x7777
    rc, b2, o2, r2, _ = a.append_frames(0, n, ids, bytes_out=bout, offsets_out=oout, rest_out=rout, bytes_capacity=N_,
                                        frames_capacity=F_, rest_capacity=R_)
    assert rc == B.OK and np.array_equal(b2, blob) and np.array_equal(o2, off) and np.array_equal(r2, rest)
    assert np.all(bout[N_:] == 0xA5) and np.all(oout[F_ + 1:] == 0x5A5A5A5A) and np.all(rout["next_idx"][R_:] == 0x7777)
    a.close()


def test_refusals_before_any_launch():
    a, ac, n, _ = _small()
    L, h = a._L, a._h
    wide = n - 2                                           # the last wide pair's low half
    ids = np.ones((9, 256), np.uint64)
    d_ids, d_bytes, d_off, d_rest, d_tot = (a.device_alloc(ids.nbytes), a.device_alloc(64 << 10), a.device_alloc(4 << 10),
                                            a.device_alloc(32 << 10), a.device_alloc(32))
    a.h2d(d_tot, np.full(4, 77, np.uint64))
    totals = np.zeros(4, np.uint64)
    bbuf, obuf, rbuf = np.zeros(64 << 10, np.uint8), np.zeros(1 << 10, np.uint32), np.zeros(2048, B.SEND_ENTRY_DTYPE)
    dev = L.raftgpu_append_frames_device
    refused = [
        dev(h, None, wide + 1, 1, None, d_ids, d_bytes, 64 << 10, d_off, 1000, d_rest, 2000, d_tot),   # starts at a high half
        dev(h, None, 0, wide + 1, None, d_ids, d_bytes, 64 << 10, d_off, 1000, d_rest, 2000, d_tot),   # ends at a low half
        dev(h, None, 0, 8, None, d_ids, d_bytes + 4, 64 << 10, d_off, 1000, d_rest, 2000, d_tot),      # unaligned
        dev(h, None, 0, 8, None, None, d_bytes, 64 << 10, d_off, 1000, d_rest, 2000, d_tot),
        dev(h, None, 0, 8, None, d_ids, d_bytes, 64 << 10, d_off, 1000, d_rest, 2000, None),
        dev(h, None, 0, 8, None, d_ids, None, 64, d_off, 1000, d_rest, 2000, d_tot),
        dev(h, None, 0, 8, None, d_ids, d_bytes, 64 << 10, d_off, 1000, None, 2000, d_tot),
        L.raftgpu_append_frames(h, wide + 1, 1, None, ids.ctypes.data, bbuf.ctypes.data, len(bbuf), obuf.ctypes.data, 1000,
                                rbuf.ctypes.data, 2000, totals.ctypes.data),
        L.raftgpu_append_frames(h, 0, 8, None, ids.ctypes.data, bbuf.ctypes.data, len(bbuf), obuf.ctypes.data, 1000,
                                rbuf.ctypes.data, 2000, None),
    ]
    assert refused == [B.ERR_INVALID] * len(refused), refused
    assert dev(h, None, 0, a.cap + 1, None, d_ids, d_bytes, 1, d_off, 1, d_rest, 1, d_tot) == B.ERR_RANGE
    # a range of 7_456_541 slots or more is refused: its bound exceeds u32 offsets
    assert B.append_frames_bound(7_456_540) < (1 << 32) <= B.append_frames_bound(7_456_541)
    big = B.Arena(7_456_544)
    assert big._L.raftgpu_append_frames_device(big._h, None, 0, 7_456_541, None, d_ids, None, 0, None, 0, None, 0,
                                               d_tot) == B.ERR_INVALID
    big.close()
    a.synchronize()
    tot = np.zeros(4, np.uint64)
    a.d2h(tot, d_tot)
    assert tot.tolist() == [77] * 4           # nothing was launched
    a.close()


# --------------------------------------------------------------------------- 5. back through a wire step

def test_frames_through_a_wire_step_are_skip_type():
    """Every frame of the pass comes back SKIP_TYPE from a wire step, and the frames change nothing: the arena ends as
    a twin arena does after a wire step with only the first frame (the step's own maybe_commit runs in both)."""
    a, ac, n, ids = _small()
    twin = _small()[0]
    rc, blob, off, rest, tot = a.append_frames(0, n, ids)
    assert rc == B.OK and int(tot[0]) > 50
    fb = F.Frames([])
    fb.bytes, fb.offsets, fb.n, fb.n_bytes = blob.copy(), off.copy(), int(tot[0]), int(tot[1])
    a.step_begin_wire(fb)
    a.step_wait()
    assert np.all(a.wire_status() == B.WIRE_SKIP_TYPE << 4)
    one = F.Frames([bytes(blob[off[0]:off[1]])])
    twin.step_begin_wire(one)
    twin.step_wait()
    assert np.all(twin.wire_status() == B.WIRE_SKIP_TYPE << 4)
    _columns_equal(a.read_columns(n), twin.read_columns(n))
    twin.close()
    a.close()


# --------------------------------------------------------------------------- 6. between a begin and its wait

def test_host_form_between_begin_and_wait():
    n = 100_000
    s = B.Synth(n, 0xA9F2, k_peers=5)
    a = B.Arena(n)
    assert a.group_alloc_range(n) == 0
    a.load_columns(s.initial)
    a.column_write(B.COL_TERM, 0, 0, np.full(n, 5, np.uint64))
    ids = A.ids_for(np.random.default_rng(8), n)
    for _ in range(3):
        a.step_begin_records(s.next_round().copy(), B.STEP_READ_COMMITTED)
        during = a.append_frames(0, n, ids)
        during = [x.copy() for x in during[1:]]
        a.step_wait()
        after = a.append_frames(0, n, ids)[1:]
        for x, y in zip(during, after):
            assert np.array_equal(x, y)
    a.close()
