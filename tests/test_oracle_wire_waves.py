"""The wave oracle (oracle/wire_waves_oracle.c): the wire step and the follower's append passes at
raftgpu_arena_set_wire_waves > 1.  At enough waves it equals the literal per-message forms -- the leader's
handle_append_response prefix per frame in arrival order then one maybe_commit, the follower's every frame stepped in
order -- on batches where every frame is decidable; at one wave it is the existing batch forms; a group whose claimant
is NEEDS_LOG or COMMIT_RANGE keeps its later frames DUP.  The batch builders here are shared with
tests/test_gpu_wire_waves.py."""
import numpy as np

from helpers import B, O, assert_columns_equal
from oracle import app_entries_oracle as AE
from oracle import app_follow_oracle as AL
from oracle import wire_waves_oracle as WW
import app_follow as A
import append_reject as R

DUP, NEEDS_LOG, COMMIT_RANGE = O.WIRE_DUP, O.WIRE_NEEDS_LOG, AL.WIRE_COMMIT_RANGE


# --------------------------------------------------------------------------- batch builders


def literal_leader(c, blob, off):
    """The literal per-message application: every frame decoded, its record (and a REJECT's EXT) through
    handle_append_response's prefix in arrival order, then one maybe_commit.  Statuses as the step reports them."""
    st, recs, hint, snap = _decode_all(c, blob, off)
    seq, main = [], []
    for i in range(len(st)):
        main.append(len(seq))
        seq.append(tuple(recs[i]))
        if recs["flags"][i] & B.REC_REJECT:
            seq.append((recs["group"][i], recs["peer_slot"][i], B.REC_EXT, 0, hint[i], snap[i]))
    res = O.arena_apply(c, np.array(seq, B.APPEND_RESP_DTYPE), mode=0)
    O.arena_recompute(c)
    return ((st.astype(np.uint32) << 4) | (res[main] & 0xF)).astype(np.uint8)


def _decode_all(c, blob, off):
    """Every frame's record as wo_decode_batch decodes it, one frame per batch (no duplicate rule); all must be OK."""
    n = len(off) - 1
    st = np.zeros(n, np.uint8)
    recs, hint, snap = None, np.zeros(n, np.uint64), np.zeros(n, np.uint64)
    for i in range(n):
        f = np.ascontiguousarray(blob[off[i]:off[i + 1]])
        s, r, h, q = O.wire_decode_batch(f, np.array([0, len(f)], np.uint32), c.n_groups, c.term[: c.n_groups])
        assert s[0] == O.WIRE_OK
        if recs is None:
            recs = np.zeros(n, r.dtype)
        recs[i], hint[i], snap[i] = r[0], h[0], q[0]
    return st, recs, hint, snap


# --------------------------------------------------------------------------- the leader

def _leaders(rng, n):
    logs = [R.random_log(rng, int(rng.integers(1, 5))) for _ in range(n)]
    return logs, R.leader_columns(logs, n, seed=int(rng.integers(0, 1 << 30)))


def test_leader_waves_equal_the_literal_application():
    """1-6 decidable frames per cell (accepts, stale accepts, rejections with log_term 0): at waves >= the most frames
    per cell the wave oracle equals the literal application in arrival order, every column and every status."""
    rng = np.random.default_rng(0x3A7E)
    n = 400
    logs, c = _leaders(rng, n)
    blob, off = A.batch(R.leader_frames(rng, c, range(n), range(1, 5), 6))
    lit = O.copy_columns(c)
    want = literal_leader(lit, blob, off)
    for waves in (6, 9, 64):
        ref = O.copy_columns(c)
        got = WW.leader(ref, None, blob, off, waves)
        O.arena_recompute(ref)
        assert np.array_equal(got, want), waves
        assert_columns_equal(ref, lit, n, f"waves {waves}")
    assert ((want >> 4) == O.WIRE_OK).all() and len(want) > 4 * n * 2


def test_leader_fewer_waves_leave_the_rest_dup():
    """At waves = k < the most frames per cell, the first k frames of every cell are applied and the rest are DUP: the
    result equals k waves' worth of the frames applied literally."""
    rng = np.random.default_rng(0x3A7F)
    n = 200
    _, c = _leaders(rng, n)
    frames = R.leader_frames(rng, c, range(n), range(1, 4), 6)
    blob, off = A.batch(frames)
    cell = np.array([int.from_bytes(f[:4], "little") for f in frames])
    rank = np.zeros(len(frames), int)
    seen = {}
    for i, x in enumerate(cell.tolist()):
        rank[i] = seen.get(x, 0)
        seen[x] = rank[i] + 1
    for k in (1, 2, 4):
        ref = O.copy_columns(c)
        got = WW.leader(ref, None, blob, off, k)
        O.arena_recompute(ref)
        keep = np.flatnonzero(rank < k)
        lit = O.copy_columns(c)
        sub = A.batch([frames[i] for i in keep])
        want = literal_leader(lit, *sub)
        assert np.array_equal(got[keep], want), k
        assert ((got[rank >= k] >> 4) == DUP).all()
        assert_columns_equal(ref, lit, n, f"k {k}")


def test_leader_one_wave_is_the_batch_form():
    """waves = 1 is the existing step, with and without leader runs, on batches with every status (NEEDS_LOG, TERM,
    hostile frames)."""
    rng = np.random.default_rng(0x3A80)
    n = 300
    logs, c = _leaders(rng, n)
    rows = R.rows_for(logs, np.ones(n), 2)
    frames = R.leader_frames(rng, c, range(n), range(1, 5), 4, needs_log=0.5)
    frames += [A.frame(3, 1, R.response(int(c.term[3]) + 1, index=1)), b"\x01\x02", A.frame(n + 7, 1, R.response(1))]
    blob, off = A.batch(frames)
    for r in (None, rows):
        ref, ref1 = O.copy_columns(c), O.copy_columns(c)
        want = R.oracle_step(ref, r, blob, off)
        got = WW.leader(ref1, r, blob, off, 1)
        assert np.array_equal(got, want)
        assert_columns_equal(ref1, ref, n, "one wave")
        assert ((want >> 4) == NEEDS_LOG).any() and ((want >> 4) == DUP).any()


# --------------------------------------------------------------------------- the follower

def _followers(rng, n):
    w = A.World(rng, n, log_cap=64, max_last=30)
    w.groups["committed"] = np.minimum(w.groups["committed"], w.groups["last_index"])
    return w


def _literal_follower(w, blob, off):
    g = w.copy()
    outcome, rb, ro, tot = AL.literal(g.groups, g.terms, blob, off)
    return g, outcome, rb, ro, tot


def test_follower_waves_equal_the_literal_form():
    """1-6 pipelined MsgAppend frames per group with entries (frame j's entries start at frame j-1's last index + 1):
    the wave oracle at waves >= 6 answers every frame, with the literal form's responses byte for byte, committed and
    last_index; the table's run is a suffix of the literal log's last run."""
    rng = np.random.default_rng(0xF011)
    n = 500
    w = _followers(rng, n)
    per_group = []
    for g in range(n):
        last = int(w.groups["last_index"][g])
        bodies = R.pipelined_appends(rng, last, int(w.terms[g, last]), int(w.groups["term"][g]),
                                   int(w.groups["committed"][g]), int(rng.integers(1, 7)))
        per_group.append((g, [A.frame(g, 0, b) for b, _ in bodies]))
    blob, off = A.batch(R.interleave(rng, per_group))
    lit, outcome, lrb, lro, ltot = _literal_follower(w, blob, off)
    assert (outcome == AL.ANSWERED).all()
    for waves in (6, 64):
        c, table = w.columns(), w.table(w.runs())
        st, frm, app, rb, ro, tot = WW.follower(c, None, table, blob, off, waves, entries=True)
        assert ((st >> 4) == O.WIRE_OK).all() and (st & AE.APPENDED).all(), waves
        assert np.array_equal(rb, lrb) and np.array_equal(ro, lro) and np.array_equal(tot, ltot), waves
        assert np.array_equal(c.committed[:n], lit.groups["committed"]) and np.array_equal(c.last_index[:n], lit.groups["last_index"])
        for g in range(n):
            last = int(lit.groups["last_index"][g])
            s, t = int(table["run_start"][g]), int(table["run_term"][g])
            assert s <= last and (lit.terms[g, s:last + 1] == t).all(), g


def test_follower_entry_less_waves_equal_the_literal_form():
    """1-6 entry-less appends per group at the log's end with rising commits: every frame answered as the literal form
    answers it, and committed is the last one's."""
    rng = np.random.default_rng(0xF012)
    n = 500
    w = _followers(rng, n)
    per_group = []
    for g in range(n):
        last = int(w.groups["last_index"][g])
        bodies = R.pipelined_appends(rng, last, int(w.terms[g, last]), int(w.groups["term"][g]),
                                   int(w.groups["committed"][g]), int(rng.integers(1, 7)), entries=False)
        per_group.append((g, [A.frame(g, 0, b) for b, _ in bodies]))
    blob, off = A.batch(R.interleave(rng, per_group))
    lit, outcome, lrb, lro, ltot = _literal_follower(w, blob, off)
    c, table = w.columns(), w.table(w.runs())
    st, frm, app, rb, ro, tot = WW.follower(c, None, table, blob, off, 6, entries=False)
    assert ((st >> 4) == O.WIRE_OK).all()
    assert np.array_equal(rb, lrb) and np.array_equal(ro, lro) and np.array_equal(tot, ltot)
    assert np.array_equal(c.committed[:n], lit.groups["committed"])


def test_follower_one_wave_is_the_batch_form():
    """waves = 1 is afl_batch / aeo_batch exactly, on random frames with several per group."""
    rng = np.random.default_rng(0xF013)
    n = 400
    w = _followers(rng, n)
    frames = [A.frame(g, 0, A.random_append(rng, w, g, entries_p=0.5)) for g in rng.integers(0, n, 3 * n).tolist()]
    blob, off = A.batch(frames)
    runs = w.runs(rng, shorten=0.3)
    for entries in (False, True):
        c1, t1, c2, t2 = w.columns(), w.table(runs), w.columns(), w.table(runs)
        want = AE.batch(c1, None, t1, blob, off) if entries else AL.batch(c1, None, t1, blob, off)
        got = WW.follower(c2, None, t2, blob, off, 1, entries=entries)
        if not entries:
            got = got[:2] + got[3:]
        for x, y in zip(want, got):
            assert np.array_equal(x, y), entries
        assert np.array_equal(t1, t2) and np.array_equal(c1.committed, c2.committed)
        assert np.array_equal(c1.last_index, c2.last_index)
        assert ((want[0] >> 4) == DUP).any()


def test_follower_stop_rule():
    """Groups of three pipelined frames whose second one, decided in wave 2, is NEEDS_LOG (entries past a gap above the
    new log) or COMMIT_RANGE (an entry-less match above last_index asking to commit past it): the third stays DUP at any
    number of waves, while the twin group whose second frame is OK has its third decided."""
    rng = np.random.default_rng(0xF014)
    w = _followers(rng, 3)
    per_group = []
    kinds = ("needs_log", "commit_range", "ok")
    for g, kind in enumerate(kinds):
        last = int(w.groups["last_index"][g])
        term = int(w.groups["term"][g])
        b = R.pipelined_appends(rng, last, int(w.terms[g, last]), term, int(w.groups["committed"][g]), 3)
        top = b[0][1]
        if kind == "needs_log":
            second = A.message(3, term=term, log_term=0, index=top + 5, commit=top, frm=9, entries=[(term, top + 6)])
        elif kind == "commit_range":
            second = A.message(3, term=term, log_term=0, index=top + 5, commit=top + 5, frm=9)
        else:
            second = b[1][0]
        per_group.append((g, [A.frame(g, 0, b[0][0]), A.frame(g, 0, second), A.frame(g, 0, b[2][0])]))
    blob, off = A.batch([f for _, fr in per_group for f in fr])
    for waves in (2, 3, 64):
        c, table = w.columns(), w.table(w.runs())
        st = WW.follower(c, None, table, blob, off, waves, entries=True)[0] >> 4
        assert st.tolist()[:6] == [O.WIRE_OK, NEEDS_LOG, DUP, O.WIRE_OK, COMMIT_RANGE, DUP], waves
        assert st.tolist()[6:] == ([O.WIRE_OK, O.WIRE_OK, DUP] if waves == 2 else [O.WIRE_OK] * 3), waves
