"""Entry-less MsgAppend frames at the follower on the GPU (raftgpu_follower_append[_device]) against the batch oracle
(oracle/app_follow_oracle.c), byte for byte: status, from, response bytes and offsets, totals and every group column.
Random 100K-group follower arenas fed with raftgpu_append_frames output and hostile frames, values at the edges, the
shared stage and hostile offsets, the refusals, and the whole commit loop at 1M groups x 5 peers.  Run with -m gpu."""
import numpy as np
import pytest

from oracle import app_follow_oracle as AL
from oracle import app_frames_oracle as AF
from helpers import B, O
import app_follow as A
import hb_follow as FL
import hb_frames as F
import pass_forms as PF
import wire_batches as WB

pytestmark = pytest.mark.gpu

P = 8
U64 = A.U64
OK = A.LOG_STATUS_OK


def _compare(a, c, q, blob, off, table, device, what, n_bytes=None):
    want = AL.batch(c, q, table, blob, off, n_bytes=n_bytes)
    got = PF.device(a, "follower_append", blob, off, table, n_bytes=n_bytes) if device else \
        A.host_form(a, blob, off, table, n_bytes)
    PF.equal(want, got, A.NAMES, what)
    s = FL.group_state(a, c.n_groups)
    for name, col in s.items():
        assert np.array_equal(col, getattr(c, name)[: c.n_groups]), (what, name)
    return want


# --------------------------------------------------------------------------- 1. random 100K-group follower arenas

def _leader_frames(seed, n_l):
    """raftgpu_append_frames (device form) of n_l leaders x 5 peers, every peer caught up -> [(term, index, commit,
    frame body)]."""
    rng = np.random.default_rng(seed)
    s = B.Synth(n_l, seed, k_peers=5)
    la = B.Arena(n_l)
    assert la.group_alloc_range(n_l) == 0
    la.load_columns(s.initial)
    la.column_write(B.COL_TERM, 0, 0, rng.integers(1, 1 << 40, n_l).astype(np.uint64))
    for _ in range(2):
        la.step_begin_records(s.next_round().copy(), B.STEP_READ_COMMITTED)
        la.step_wait()
    c = la.read_columns(n_l)
    la.column_write(B.COL_TERM_START, 0, 0, np.minimum(c.term_start[:n_l], c.last_index[:n_l]))
    for k in range(B.SLOTS):
        la.column_write(B.COL_NEXT_IDX, k, 0, (c.last_index[:n_l] + 1).astype(np.uint64))
        la.column_write(B.COL_PFLAGS, k, 0, np.full(n_l, B.STATE_REPLICATE, np.uint8))
    blob, off, rest, tot = PF.broadcast(la, "append_frames", 0, n_l, rng.integers(1, 1 << 63, (9, n_l), dtype=np.uint64), None)
    la.close()
    assert int(tot[0]) > 3 * n_l
    out = []
    for _, body in FL.frames_of(blob, off):
        m = O.wire_decode_message(body)
        out.append((m["term"], m["index"], m["commit"], body))
    return out


N_NARROW, N_WIDE = 99_000, 500


@pytest.mark.parametrize("reads", [True, False], ids=["read_queues", "no_read_queues"])
def test_random_arenas_vs_oracle(reads):
    rng = np.random.default_rng(0xAF10 + reads)
    n = N_NARROW + 2 * N_WIDE
    leader = _leader_frames(0xAF11 + reads, 25_000)
    nl = len(leader)
    fg = rng.integers(0, n, nl)
    hi = np.arange(N_NARROW + 1, n, 2)
    fg[np.isin(fg, hi)] -= 1                                           # a pair is addressed by its low half (mostly)
    fg[rng.random(nl) < 0.01] = hi[0]
    lt = np.array([t for t, _, _, _ in leader], np.uint64)
    li = np.array([i for _, i, _, _ in leader], np.uint64)
    terms = rng.integers(1, 1000, n).astype(np.uint64)
    last = rng.integers(0, 1 << 20, n).astype(np.uint64)
    hit = rng.random(nl) < 0.92
    terms[fg[hit]] = lt[hit]
    last[fg] = li + rng.integers(0, 4, nl).astype(np.uint64) - np.minimum(li, rng.integers(0, 3, nl).astype(np.uint64))
    committed = last - np.minimum(last, rng.integers(0, 60, n).astype(np.uint64))
    terms[hi] = terms[hi - 1]
    term_start = np.where(rng.random(n) < 0.05, np.uint64(1), np.uint64(A.NO_TERM_START))
    cols = {B.COL_TERM: terms, B.COL_LAST_INDEX: last, B.COL_COMMITTED: committed, B.COL_TERM_START: term_start}
    a, c, q = A.follower_arena(N_NARROW, N_WIDE, cols, reads)
    table = np.zeros(n, AL.LOG_DTYPE)
    table["id"] = rng.integers(1, 1 << 63, n, dtype=np.uint64)
    table["flags"] = np.where(rng.random(n) < 0.95, AL.SELECT, 0)
    top = np.maximum(c.last_index[:n], np.concatenate([c.last_index[1:n], [0]]))
    table["run_start"] = np.where(rng.random(n) < 0.8, top - np.minimum(top, rng.integers(0, 5, n).astype(np.uint64)),
                                  top + 1)
    table["run_term"] = terms                                          # the leader's frames carry log_term = its term
    kinds = np.zeros(16, np.int64)
    for rnd, device in enumerate((False, True, True)):
        order = rng.permutation(nl)
        order = np.concatenate([order, order[rng.random(nl) < 0.15]])   # repeated frames: DUP
        frames = [A.frame(int(fg[i]), int(rng.integers(16)), leader[i][3]) for i in order]
        frames += A.hostile(rng, terms, nl // 20)
        frames = [frames[i] for i in rng.permutation(len(frames))]
        blob, off = A.batch(frames)
        st = _compare(a, c, q, blob, off, table, device, ("round", rnd))[0]
        kinds += np.bincount(st >> 4, minlength=16)
    assert kinds[B.WIRE_OK] > 20_000 and kinds[B.WIRE_DUP] > 5_000, kinds
    for k in (B.WIRE_MALFORMED, B.WIRE_SKIP_TYPE, B.WIRE_ROLE, B.WIRE_TERM, B.WIRE_NEEDS_LOG, B.WIRE_COMMIT_RANGE):
        assert kinds[k] > 50, (k, kinds)
    a.close()


# --------------------------------------------------------------------------- 2. values at the edges

EDGE = [0, 1, 2, 1 << 63, U64 - 1, U64]


def test_edges():
    """Indexes, terms and commits at 0, 1, 2^63 and 2^64 - 1, runs that are empty, of length one or end exactly at
    m.index, through both forms."""
    rng = np.random.default_rng(0xAF20)
    n = 4096
    pick = lambda k: np.array(EDGE, np.uint64)[rng.integers(0, len(EDGE), k)]
    terms = pick(n)
    terms[terms == 0] = 1
    last = pick(n)
    committed = np.minimum(last, pick(n))
    cols = {B.COL_TERM: terms, B.COL_LAST_INDEX: last, B.COL_COMMITTED: committed,
            B.COL_TERM_START: np.full(n, A.NO_TERM_START, np.uint64)}
    a, c, _ = A.follower_arena(n, 0, cols)
    table = np.zeros(n, AL.LOG_DTYPE)
    table["id"], table["flags"] = pick(n), AL.SELECT
    kind = rng.integers(0, 3, n)                                       # empty, length one, from an edge value
    table["run_start"] = np.where(kind == 0, last + np.uint64(1), np.where(kind == 1, last, np.minimum(last, pick(n))))
    table["run_term"] = pick(n)
    kinds = np.zeros(16, np.int64)
    for rnd, device in enumerate((False, True, True, False)):
        frames = []
        for g in rng.permutation(n)[: 3 * n // 4].tolist():
            idx = int(rng.choice([int(last[g]), int(table["run_start"][g]), int(rng.choice(EDGE))]))
            lterm = int(rng.choice([int(table["run_term"][g]), 0, int(rng.choice(EDGE))]))
            frames.append(A.frame(g, rng.integers(16), A.message(3, term=int(terms[g]), log_term=lterm, index=idx,
                                                                  commit=int(rng.choice(EDGE)), frm=int(rng.choice(EDGE)))))
        st = _compare(a, c, None, *A.batch(frames), table, device, ("edges", rnd))[0]
        kinds += np.bincount(st >> 4, minlength=16)
    assert kinds[B.WIRE_OK] > 1000 and kinds[B.WIRE_NEEDS_LOG] > 100 and kinds[B.WIRE_COMMIT_RANGE] > 100, kinds
    a.close()


# --------------------------------------------------------------------------- 3. the stage and hostile offsets

class Followers:
    """The scenario protocol of test_gpu_wire_batches (frames / fresh / run / check) for this pass.  Group 0, which the
    ballast frames name, is not selected: its MsgAppend ballast is ROLE (its MsgSnapshot ballast SKIP_TYPE), so that
    the ballast never claims a group."""

    PER_FRAME = (0, 1)

    def __init__(self, seed, n):
        rng = np.random.default_rng(seed)
        self.n = n
        self.w = A.World(rng, n)
        self.table = self.w.table(self.w.runs(rng, 0.3))
        self.table["flags"][0] = 0

    def frames(self, rng):
        out = [A.frame(g, int(rng.integers(16)), A.random_append(rng, self.w, g))
               for g in rng.integers(1, self.n, 3 * self.n // 2).tolist()]
        return out

    def fresh(self):
        c = self.w.columns()
        cols = {B.COL_TERM: c.term, B.COL_LAST_INDEX: c.last_index, B.COL_COMMITTED: c.committed,
                B.COL_TERM_START: c.term_start}
        a, hc, _ = A.follower_arena(self.n, 0, cols)
        return a, hc

    def run(self, a, c, buf, n_bytes, off, device, what):
        want = AL.batch(c, None, self.table, buf, off, n_bytes=n_bytes)
        got = PF.device(a, "follower_append", buf, off, self.table, n_bytes=n_bytes) if device else \
            A.host_form(a, buf, off, self.table, n_bytes)
        PF.equal(want, got, A.NAMES, what)
        return got

    def check(self, a, c, what):
        s = FL.group_state(a, self.n)
        for name, col in s.items():
            assert np.array_equal(col, getattr(c, name)[: self.n]), (what, name)


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_across_the_stage(device):
    sc = Followers(0xAF30, 20_000)
    frames, ballast = WB.stage_batch(sc, 0xAF31)
    blob, off = F.batch(frames)
    assert WB.geometry(off, len(blob)) >= {WB.STAGED, WB.SPAN, "frame>16K", "frame>64K"}
    a, c = sc.fresh()
    got = sc.run(a, c, blob, len(blob), off, device, "ballast")
    sc.check(a, c, "ballast")
    assert np.all(np.isin(got[0][ballast] >> 4, [B.WIRE_ROLE, B.WIRE_SKIP_TYPE]))   # MsgAppend / MsgSnapshot ballast
    assert np.count_nonzero(got[0][~ballast] >> 4 == B.WIRE_OK) > 1000
    a2, c2 = sc.fresh()
    blob2, off2 = F.batch([f for f, b in zip(frames, ballast) if not b])
    got2 = sc.run(a2, c2, blob2, len(blob2), off2, device, "plain")
    for k, (x, y) in enumerate(zip(got, got2)):
        assert np.array_equal(x[~ballast] if k in sc.PER_FRAME else x, y), ("output", k)
    sc.check(a2, c, "plain against the ballast run")
    a.close()
    a2.close()


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_hostile_offsets(device):
    sc = Followers(0xAF32, 2_000)
    a, c = sc.fresh()
    seen = np.zeros(16, np.int64)
    if not device:
        blob, off = F.batch(sc.frames(np.random.default_rng(1)))
        sc.run(a, c, blob, len(blob), off, False, "valid")
    for k, (buf, n_bytes, off) in enumerate(WB.hostile_batches(sc, 0xAF33, device)):
        got = sc.run(a, c, buf, n_bytes, off, device, k)[0]
        sc.check(a, c, k)
        seen += np.bincount(got >> 4, minlength=16)
    assert seen[B.WIRE_MALFORMED] > 100 and seen[B.WIRE_OK] > 100, seen
    a.close()


# --------------------------------------------------------------------------- 4. refusals

def test_refusals_before_any_launch():
    n_g = 64
    cols = {B.COL_TERM: np.full(n_g, 3, np.uint64), B.COL_LAST_INDEX: np.full(n_g, 9, np.uint64),
            B.COL_TERM_START: np.full(n_g, A.NO_TERM_START, np.uint64)}
    a, c, _ = A.follower_arena(n_g, 0, cols)
    before = FL.group_state(a, n_g)
    L, h = a._L, a._h
    n = 16
    blob, off = A.batch([A.frame(g, 0, A.message(3, term=3, log_term=3, index=9, commit=7, frm=2)) for g in range(n)])
    bound = B.follower_append_bound(n)
    assert bound == 85 * n
    table = np.zeros(a.get_info().hi, AL.LOG_DTYPE)
    table["id"], table["run_start"], table["run_term"], table["flags"] = 5, 1, 3, AL.SELECT
    nb = len(blob)
    with PF.refusals(a, "follower_append", blob, off, table) as r:
        dev, d = r.call, r.args
        a.h2d(d["rb"], np.full(bound + 64, 0xCD, np.uint8))
        big = (1 << 32) // 85 + 1                                   # the first n whose bound exceeds u32 offsets
        assert B.follower_append_bound(big - 1) < (1 << 32) <= B.follower_append_bound(big)
        refused = [dev(cap=bound - 1), dev(cap=0), dev(b=d["b"] + 4), dev(rb=d["rb"] + 8), dev(l=d["l"] + 8), dev(n=big, cap=85 * big),
                   dev(n=1 << 32, cap=U64), dev(nb=1 << 32), dev(l=None), dev(ro=None), dev(t=None), dev(b=None)]
        assert refused == [B.ERR_INVALID] * len(refused), refused
        st, tot, rb = np.zeros(n, np.uint8), np.zeros(2, np.uint64), np.zeros(bound, np.uint8)
        ro = np.zeros(n + 1, np.uint32)
        host = lambda cap, t=table: L.raftgpu_follower_append(h, blob.ctypes.data, nb, off.ctypes.data, n,
                                                              None if t is None else t.ctypes.data, st.ctypes.data, None,
                                                              rb.ctypes.data, cap, ro.ctypes.data, tot.ctypes.data)
        assert host(bound - 1) == B.ERR_INVALID and host(bound, None) == B.ERR_INVALID
        grb = r.read("rb", np.zeros(bound + 64, np.uint8))
        assert r.untouched() and np.all(grb == 0xCD)   # nothing was launched
        after = FL.group_state(a, n_g)
        assert all(np.array_equal(before[k], after[k]) for k in before)
        # the exact bound is accepted, and the host form equals the device form
        assert host(bound) == B.OK and tot.tolist()[0] == n and np.all(st == OK)
        assert np.all(a.read_columns(n_g).committed[:n] == 7)
    a.close()


# --------------------------------------------------------------------------- 5. the commit loop at 1M x 5

def test_full_commit_loop_1m():
    """A leader arena of 1M groups x 5 peers after synthetic steps, every follower caught up, selected by the advanced
    bitmap -> raftgpu_append_frames_device -> one follower arena per follower slot, raftgpu_follower_append_device (the
    header (g << 4 | slot) names the follower's own group g, x = slot) -> the responses back through
    raftgpu_wire_apply_device and raftgpu_recompute at the leader.  All five arenas equal the oracle chain; every frame
    is OK and every response WIRE_OK at the leader."""
    n = 1_000_000
    rng = np.random.default_rng(0xAF50)
    s = B.Synth(n, 0xAF51, k_peers=5)
    la = B.Arena(n)
    assert la.group_alloc_range(n) == 0
    la.load_columns(s.initial)
    terms = rng.integers(1, 1000, n).astype(np.uint64)
    la.column_write(B.COL_TERM, 0, 0, terms)
    for _ in range(3):
        la.step_begin_records(s.next_round().copy(), B.STEP_READ_COMMITTED)
        la.step_wait()
    bm = la.step_results(n)[0].copy()
    c = la.read_columns(n)
    c.term = terms.copy()
    c.next_idx[:] = c.last_index[None, :] + 1
    c.pflags[:] = np.where((c.pflags & 3) == B.STATE_SNAPSHOT, c.pflags, B.STATE_REPLICATE)
    c.term_start[:n] = np.minimum(c.term_start[:n], c.last_index[:n])
    for k in range(B.SLOTS):
        la.column_write(B.COL_NEXT_IDX, k, 0, c.next_idx[k].copy())
        la.column_write(B.COL_PFLAGS, k, 0, c.pflags[k].copy())
    la.column_write(B.COL_TERM_START, 0, 0, c.term_start[:n].copy())
    ids = rng.integers(1, 1 << 63, (9, n), dtype=np.uint64)
    sel = bm
    # the oracle chain
    want_blob, want_off, want_rest, want_tot = AF.bcast_append(c, None, 0, n, ids, sel)
    blob, off, rest, tot = PF.broadcast(la, "append_frames", 0, n, ids, sel)
    assert np.array_equal(blob, want_blob) and np.array_equal(off, want_off) and tot.tolist() == want_tot.tolist()
    frames = int(tot[0])
    assert frames > 10_000 and len(rest) < frames, tot
    hdr = FL.headers(blob, off)
    slot = hdr & 15
    fas, want_f, back_parts = [], [], []
    for s_ in range(B.SLOTS):
        idx = np.flatnonzero(slot == s_)
        if len(idx) == 0:
            continue
        sub = [blob[off[i]:off[i + 1]].tobytes() for i in idx.tolist()]
        fblob, foff = A.batch(sub)
        fc = O.new_columns(n, n)
        fc.term_start[:] = A.NO_TERM_START
        fc.term[:n], fc.last_index[:n] = c.term[:n], c.last_index[:n]
        fc.committed[:n] = np.minimum(c.peer_committed[s_, :n], c.last_index[:n])
        table = np.zeros(n, AL.LOG_DTYPE)
        table["id"], table["flags"] = ids[s_], AL.SELECT
        table["run_start"], table["run_term"] = c.term_start[:n], c.term[:n]
        fa = B.Arena(n)
        assert fa.group_alloc_range(n) == 0
        for col, name in ((B.COL_TERM, "term"), (B.COL_LAST_INDEX, "last_index"), (B.COL_COMMITTED, "committed"),
                          (B.COL_TERM_START, "term_start")):
            fa.column_write(col, 0, 0, getattr(fc, name)[:n].copy())
        w = AL.batch(fc, None, table, fblob, foff)
        assert np.all(w[0] == OK), np.bincount(w[0])
        got = PF.device(fa, "follower_append", fblob, foff, table)
        PF.equal(w, got, A.NAMES, ("follower slot", s_))
        assert np.array_equal(fa.read_columns(n).committed, fc.committed[:n]), s_
        fas.append(fa)
        back_parts.append((w[2], w[3]))
    # the responses back at the leader, one batch
    rblob = np.concatenate([b for b, _ in back_parts])
    base = np.cumsum([0] + [len(b) for b, _ in back_parts])
    roff = np.concatenate([o[:-1].astype(np.int64) + base[k] for k, (_, o) in enumerate(back_parts)] + [[base[-1]]]).astype(np.uint32)
    nr = len(roff) - 1
    assert nr == frames
    wst, recs, _, _ = O.wire_decode_batch(rblob, roff, n, c.term[:n])
    assert np.all(wst == B.WIRE_OK)
    O.arena_apply(c, recs, mode=0)
    O.arena_recompute(c)
    d_b, d_o, d_s = la.device_alloc(max(16, len(rblob) + 16)), la.device_alloc(4 * (nr + 1)), la.device_alloc(max(1, nr))
    la.h2d(d_b, np.concatenate([rblob, np.zeros(16, np.uint8)]))
    la.h2d(d_o, roff)
    la.wire_apply_device(d_b, len(rblob), d_o, nr, d_s)
    la.recompute(0, n)
    la.synchronize()
    gst = np.zeros(nr, np.uint8)
    la.d2h(gst, d_s)
    assert np.all(gst >> 4 == B.WIRE_OK)
    lc = la.read_columns(n)
    for name in ("matched", "next_idx", "peer_committed", "pflags", "committed"):
        assert np.array_equal(getattr(lc, name), getattr(c, name)[..., :n]), name
    for p in (d_b, d_o, d_s):
        la.device_free(p)
    for fa in fas:
        fa.close()
    la.close()


# --------------------------------------------------------------------------- 6. the host form between a begin and its wait

def test_host_form_between_begin_and_wait():
    """Two follower arenas in the same state take the same synthetic steps; their LOCAL records raise last_index, so
    each step changes what the pass reads.  Each round the twin steps and waits, then runs the device form; the other
    arena calls the host form between raftgpu_step_begin_records and raftgpu_step_wait, on the staging set the step
    does not hold, with its 3.2 MB log table.  Both equal the batch oracle over the columns after the step: the host
    form is ordered after the step's kernels.  The steps never move committed here (a group without term_start has
    nothing maybe_commit may commit), which their results confirm."""
    n = 100_000
    rng = np.random.default_rng(0xAF70)
    s = B.Synth(n, 0xAF71, k_peers=5)
    terms = rng.integers(1, 1 << 40, n).astype(np.uint64)
    last = rng.integers(1, 1 << 30, n).astype(np.uint64)
    committed = last - np.minimum(last, rng.integers(0, 100, n).astype(np.uint64))
    cols = {B.COL_TERM: terms, B.COL_LAST_INDEX: last, B.COL_COMMITTED: committed,
            B.COL_TERM_START: np.full(n, A.NO_TERM_START, np.uint64)}
    arenas = []
    for _ in range(2):
        x = B.Arena(n)
        assert x.group_alloc_range(n) == 0
        x.load_columns(s.initial)
        for col, arr in cols.items():
            x.column_write(col, 0, 0, arr.copy())
        arenas.append(x)
    a, twin = arenas
    table = np.zeros(n, AL.LOG_DTYPE)
    table["id"], table["flags"] = rng.integers(1, 1 << 63, n, dtype=np.uint64), AL.SELECT
    kinds = np.zeros(16, np.int64)
    for rnd in range(3):
        recs = s.next_round().copy()
        twin.step_begin_records(recs, B.STEP_READ_COMMITTED)
        assert twin.step_wait().n_advanced == 0
        c = twin.read_columns(n)
        c.term = terms.copy()
        cur = c.last_index[:n].copy()
        assert rnd > 0 or np.count_nonzero(cur != last) > n // 2      # the step moved last_index
        table["run_start"] = cur - np.minimum(cur, rng.integers(0, 8, n).astype(np.uint64))
        table["run_term"] = terms
        frames = []
        for g in rng.permutation(n)[: 3 * n // 4].tolist():
            idx = max(0, int(cur[g]) - int(rng.integers(0, 12)) + int(rng.integers(0, 3)))
            lterm = int(terms[g]) if rng.random() < 0.8 else int(rng.integers(0, 1 << 40))
            commit = int(rng.integers(0, idx + 3))
            frames.append(A.frame(g, int(rng.integers(16)), A.message(3, term=int(terms[g]), log_term=lterm, index=idx,
                                                                       commit=commit, frm=int(rng.integers(1, 1 << 40)))))
        frames += [frames[i] for i in rng.integers(0, len(frames), len(frames) // 8)]   # repeated frames: DUP
        blob, off = A.batch(frames)
        want = AL.batch(c, None, table, blob, off)
        PF.equal(want, PF.device(twin, "follower_append", blob, off, table), A.NAMES, ("device form after the step", rnd))
        a.step_begin_records(recs, B.STEP_READ_COMMITTED)
        during = [x.copy() for x in A.host_form(a, blob, off, table)]
        assert a.step_wait().n_advanced == 0
        PF.equal(want, during, A.NAMES, ("host form during the step", rnd))
        for x in (a, twin):
            st = FL.group_state(x, n)
            for name in ("committed", "last_index", "term", "term_start"):
                assert np.array_equal(st[name], getattr(c, name)[:n]), (rnd, name)
        kinds += np.bincount(want[0] >> 4, minlength=16)
    assert kinds[B.WIRE_OK] > 50_000 and kinds[B.WIRE_DUP] > 10_000 and kinds[B.WIRE_NEEDS_LOG] > 1000, kinds
    a.close()
    twin.close()
