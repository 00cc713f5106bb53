"""MsgAppend frames with entries at the follower on the GPU (raftgpu_follower_append_entries[_device]) against the batch
oracle (oracle/app_entries_oracle.c), byte for byte: status, from, appended records, response bytes and offsets, totals,
the run table and every group column.  Random 100K-group follower arenas with 0-64 entries per frame and payloads past
the shared stage mixed in one batch, appending frames through both paths of the stage, the golden vectors' hostile
Entries, hostile offsets and the refusals, the host form against the device form on twin arenas and between
raftgpu_step_begin_records and its wait, the entry-less pass on the same batches, and the replication round trip at
100K groups x 5 peers.
Run with -m gpu."""
import numpy as np
import pytest

from oracle import app_entries_oracle as AE
from oracle import app_follow_oracle as AL
from helpers import B, O
import app_entries as E
import app_follow as A
import hb_follow as FL
import pass_forms as PF

pytestmark = pytest.mark.gpu


def _compare(a, c, q, blob, off, table, device, what, n_bytes=None):
    """One batch through the oracle (on c and a copy of table) and through the arena (on table, the full table) ->
    the oracle's result; every output, the table and the group columns must agree."""
    want_table = table.copy()
    want = AE.batch(c, q, want_table, blob, off, n_bytes=n_bytes)
    got = PF.run(a, "follower_append_entries", blob, off, table, device=device, n_bytes=n_bytes)
    PF.equal(want, tuple(got[:2]) + (got[2].view(AE.APPENDED_DTYPE),) + tuple(got[3:]), E.NAMES, what)
    assert np.array_equal(table, want_table), (what, "table")
    for name, col in FL.group_state(a, c.n_groups).items():
        assert np.array_equal(col, getattr(c, name)[: c.n_groups]), (what, name)
    return want


def _frames(rng, c, table, groups, big, hostile):
    """One random frame per listed group (a pair by its low half), from the group's current state."""
    out = []
    for g in groups.tolist():
        lo = g
        last = int(max(c.last_index[g], c.last_index[g + 1])) if c.meta[g] & E.WIDE_LO else int(c.last_index[g])
        com = int(max(c.committed[g], c.committed[g + 1])) if c.meta[g] & E.WIDE_LO else int(c.committed[g])
        body = E.random_frame(rng, last, int(table["run_start"][lo]), int(table["run_term"][lo]), int(c.term[g]), com,
                              big=big, hostile=hostile)
        out.append(A.frame(g, int(rng.integers(16)), body))
    return out


@pytest.mark.parametrize("reads", [False, True], ids=["no_read_queues", "read_queues"])
def test_random_arenas_vs_oracle(reads):
    """100K groups; each round: one frame per group for most groups (the first half with payloads up to 128 bytes, the
    second up to 20 000), repeated frames (DUP) and garbage."""
    rng = np.random.default_rng(0xAE10 + reads)
    n = E.N_NARROW + 2 * E.N_WIDE
    a, c, q, table = E.world(rng, E.N_NARROW, E.N_WIDE, reads)
    hi = set(range(E.N_NARROW + 1, n, 2))
    kinds = np.zeros(16, np.int64)
    appended = 0
    for rnd, device in enumerate((True, False, True)):
        gs = np.array([g for g in rng.permutation(n)[: n * 9 // 10] if int(g) not in hi], np.int64)
        half = len(gs) // 2
        frames = _frames(rng, c, table, gs[:half], False, 0.02) + _frames(rng, c, table, gs[half:], True, 0.02)
        frames += [frames[i] for i in rng.integers(0, len(frames), len(frames) // 20)]   # DUP
        frames += A.hostile(rng, c.term[:n], 2000)
        blob, off = A.batch(frames)
        st, _, app, *_ = _compare(a, c, q, blob, off, table, device, ("round", rnd))
        kinds += np.bincount(st >> 4, minlength=16)
        appended += int(np.count_nonzero(st & B.FAPP_APPENDED))
    assert kinds[B.WIRE_OK] > 100_000 and kinds[B.WIRE_DUP] > 5_000 and appended > 15_000, (kinds, appended)
    for s in (B.WIRE_NEEDS_LOG, B.WIRE_COMMIT_RANGE, B.WIRE_MALFORMED):
        assert kinds[s] > 0, (s, kinds)
    a.close()


KWIRE_THREADS, KWIRE_STAGE = 256, 16 * 1024   # k_wire.cuh: frames per block, staged bytes per block


def _staged_blocks(off):
    """Per block of KWIRE_THREADS frames: whether its byte range fits the stage (wire_stage_block's rule)."""
    n = len(off) - 1
    out = []
    for b in range(0, n, KWIRE_THREADS):
        lo, hi = int(off[b]), int(off[min(b + KWIRE_THREADS, n)])
        out.append(hi - (lo & ~15) <= KWIRE_STAGE)
    return np.array(out)


def _small_appends(rng, c, table, groups):
    """One appending MsgAppend per group, under 64 bytes: at index = last_index with log_term = run_term, 1-2 empty
    entries of the group's term, a small from and commit."""
    out = []
    for g in groups.tolist():
        last, t = int(c.last_index[g]), int(c.term[g])
        recs = [E.record(E.entry(t, last + 1 + j)) for j in range(int(rng.integers(1, 3)))]
        body = E.message(t, int(table["run_term"][g]), last, int(c.committed[g]), int(rng.integers(1, 100)), recs)
        out.append(A.frame(g, int(rng.integers(16)), body))
    return out


@pytest.mark.parametrize("device", [True, False], ids=["device", "host"])
def test_stage_paths_with_appended_frames(device):
    """Appending frames through both paths of wire_open: blocks whose frames fit the 16 KiB shared-memory stage (small
    frames of 1-2 empty entries, asserted to fit) and, in the same batch, blocks that do not (payloads up to 20 000
    bytes), each with many frames the pass appends."""
    rng = np.random.default_rng(0xAE20 + device)
    a, c, q, table = E.world(rng, 3000, 8, False)
    gs = rng.permutation(3000)
    # (the world's runs may start past a narrow group's last_index; these groups' runs reach it)
    table["run_start"][gs[:2048]] = np.minimum(table["run_start"][gs[:2048]], c.last_index[gs[:2048]])
    small = _small_appends(rng, c, table, gs[:1024])                 # blocks 0-3
    big = _frames(rng, c, table, gs[1024:2048], True, 0.0)           # blocks 4-7
    blob, off = A.batch(small + big)
    staged = _staged_blocks(off)
    assert staged[:4].all() and not staged[4:].any(), staged
    st = _compare(a, c, q, blob, off, table, device, "stage")[0]
    appended = (st >> 4 == B.WIRE_OK) & (st & B.FAPP_APPENDED != 0)
    assert appended[:1024].sum() > 850 and appended[1024:].sum() > 100, (appended[:1024].sum(), appended[1024:].sum())
    a.close()


@pytest.mark.parametrize("device", [True, False], ids=["device", "host"])
def test_hostile_offsets(device):
    """Offsets out of order and past the batch, and n_bytes short of the last frame, among appending frames."""
    rng = np.random.default_rng(0xAE24 + device)
    a, c, q, table = E.world(rng, 3000, 8, False)
    gs = np.arange(0, 3000)
    blob, off = A.batch(_small_appends(rng, c, table, gs[:1500]) + _frames(rng, c, table, gs[1500:], True, 0.1))
    off = off.copy()
    for j in rng.integers(1, len(off) - 1, 40):
        off[j] = int(rng.choice([int(off[j - 1]) - 1, int(off[j + 1]) + 1, len(blob) + 100, 0])) % (1 << 32)
    st = _compare(a, c, q, blob, off, table, device, "offsets", n_bytes=len(blob) - 7)[0]
    assert np.count_nonzero(st >> 4 == B.WIRE_MALFORMED) > 20 and np.count_nonzero(st & B.FAPP_APPENDED) > 500
    a.close()


@pytest.mark.parametrize("device", [True, False], ids=["device", "host"])
def test_golden_vectors_through_the_walk(device):
    """Every MsgAppend of the python-protobuf golden vectors (tests/golden/wire/append_entries.json) -- hostile ones
    included: truncated Entries, bad inner wire types, field 0, a scalar field 7, a split span -- sent to a follower
    whose log matches it at m.index, so that every frame reaches the entry walk; against the oracle."""
    import json
    import os
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "wire", "append_entries.json")
    vectors = json.load(open(path))["vectors"]
    bodies = [bytes.fromhex(v["hex"]) for v in vectors]
    # a Message cut inside an Entry's record does not parse itself: its group gets term 1 and the frame is MALFORMED
    ms = [O.wire_decode_message(b) or {"term": 1, "index": 0, "log_term": 0} for b in bodies]
    n = len(bodies)
    terms = np.array([m["term"] for m in ms], np.uint64)
    last = np.array([m["index"] for m in ms], np.uint64)
    cols = {B.COL_TERM: terms, B.COL_LAST_INDEX: last, B.COL_COMMITTED: np.zeros(n, np.uint64),
            B.COL_TERM_START: np.full(n, A.NO_TERM_START, np.uint64)}
    a, c, q = A.follower_arena(n, 0, cols)
    table = np.zeros(a.get_info().hi, AL.LOG_DTYPE)
    table["id"][:n], table["flags"][:n] = 7, AL.SELECT
    table["run_start"][:n], table["run_term"][:n] = last, [m["log_term"] for m in ms]
    blob, off = A.batch([A.frame(g, 3, b) for g, b in enumerate(bodies)])
    st = _compare(a, c, q, blob, off, table, device, "golden")[0]
    parses = np.array([v["parses"] for v in vectors])
    assert np.all((st[~parses] >> 4) == B.WIRE_MALFORMED)              # an Entry that does not parse
    assert np.all((st[parses] >> 4) != B.WIRE_MALFORMED)
    assert np.count_nonzero(st & B.FAPP_APPENDED) > 10
    a.close()


def test_refusals_before_any_launch():
    a = B.Arena(64)
    assert a.group_alloc_range(8) == 0
    n = 4
    bound = B.follower_append_bound(n)
    d = {k: a.device_alloc(s) for k, s in (("b", 256), ("o", 32), ("t", 8 * 32), ("s", 16), ("f", 64), ("ap", 256),
                                            ("rb", bound + 64), ("ro", 32), ("tot", 16))}
    L, h = B.lib(), a._h

    def call(**kw):
        args = dict(b=d["b"], nb=64, o=d["o"], n=n, t=d["t"], s=d["s"], f=d["f"], ap=d["ap"], rb=d["rb"], cap=bound,
                    ro=d["ro"], tot=d["tot"])
        args.update(kw)
        return L.raftgpu_follower_append_entries_device(h, None, args["b"], args["nb"], args["o"], args["n"], args["t"],
                                                        args["s"], args["f"], args["ap"], args["rb"], args["cap"],
                                                        args["ro"], args["tot"])

    assert call(ap=None) == B.ERR_INVALID
    assert call(t=None) == B.ERR_INVALID
    assert call(cap=bound - 1) == B.ERR_INVALID
    assert call(ap=d["ap"] + 4) == B.ERR_INVALID
    assert call(t=d["t"] + 8) == B.ERR_INVALID
    assert call(b=d["b"] + 1) == B.ERR_INVALID
    assert L.raftgpu_follower_append_entries(h, None, 0, None, 1, None, None, None, None, None, 0, None, None) == B.ERR_INVALID
    for p in d.values():
        a.device_free(p)
    a.close()


def _refresh(a, n):
    c = a.read_columns(n)
    c.term = a.column_read(B.COL_TERM, 0, 0, n, np.uint64)
    return c


def test_host_against_device_on_twins():
    """Twin arenas take the same batches, one through the host form and one through the device form, and end equal:
    outputs, tables and group columns."""
    rng = np.random.default_rng(0xAE30)
    a1, c1, _, t1 = E.world(np.random.default_rng(7), 20_000, 64, False)
    a2, _, _, t2 = E.world(np.random.default_rng(7), 20_000, 64, False)
    n = 20_000 + 128
    hi = set(range(20_001, n, 2))
    for rnd in range(3):
        gs = np.array([g for g in rng.permutation(n)[: n // 2] if int(g) not in hi], np.int64)
        blob, off = A.batch(_frames(rng, c1, t1, gs, rnd == 1, 0.05))
        r1, r2 = PF.host(a1, "follower_append_entries", blob, off, t1), PF.device(a2, "follower_append_entries", blob, off, t2)
        PF.equal(tuple(r1), tuple(r2), E.NAMES, ("twins", rnd))
        assert np.count_nonzero(r1[0] & B.FAPP_APPENDED) > 500
        assert np.array_equal(t1, t2)
        s1, s2 = FL.group_state(a1, n), FL.group_state(a2, n)
        for name in s1:
            assert np.array_equal(s1[name], s2[name]), name
        c1 = _refresh(a1, n)
    a1.close()
    a2.close()


def test_entry_less_pass_unchanged():
    """The same batches through raftgpu_follower_append: every claiming frame with entries is NEEDS_LOG, nothing is
    appended and a narrow group's last_index never moves, as its own oracle says."""
    rng = np.random.default_rng(0xAE40)
    a, c, q, table = E.world(rng, 20_000, 64, False)
    n = 20_000 + 128
    hi = set(range(20_001, n, 2))
    before = FL.group_state(a, n)["last_index"]
    for rnd in range(2):
        gs = np.array([g for g in rng.permutation(n)[: n // 2] if int(g) not in hi], np.int64)
        frames = _frames(rng, c, table, gs, rnd == 1, 0.05)
        blob, off = A.batch(frames)
        want = AL.batch(c, q, table, blob, off)
        got = a.follower_append(PF.host_batch(blob, off, len(blob)), A.full_table(a, table))
        PF.equal(want, got, A.NAMES, ("entry-less", rnd))
        decoded = [AE.decode(bytes(f[4:])) for f in frames]
        has = np.array([d is not None and len(d[1]) > 0 for d in decoded])
        st = want[0]
        assert not np.any(has & (st >> 4 == B.WIRE_OK) & ((st & (AL.STALE | AL.REJECT)) == 0))
        assert np.count_nonzero(has & (st >> 4 == B.WIRE_NEEDS_LOG)) > 1000
        for name, col in FL.group_state(a, n).items():                # as its own oracle says
            assert np.array_equal(col, getattr(c, name)[:n]), (rnd, name)
        # (a pair's commit_to evens its halves' last_index, wide_sync; a narrow group's never moves)
        assert np.array_equal(c.last_index[:20_000], before[:20_000])
    a.close()


def test_host_form_between_begin_and_wait():
    """Two follower arenas in the same state take the same synthetic steps; their LOCAL records raise last_index, so
    each step changes what the pass reads.  Each round the twin steps and waits, then runs the device form; the other
    arena calls the host form between raftgpu_step_begin_records and raftgpu_step_wait.  Both equal the batch oracle
    over the columns after the step (the host form is ordered after the step's kernels), tables included."""
    n = 100_000
    rng = np.random.default_rng(0xAE70)
    s = B.Synth(n, 0xAE71, k_peers=5)
    terms = rng.integers(2, 1 << 40, n).astype(np.uint64)
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
    base = np.zeros(n, AL.LOG_DTYPE)
    base["id"], base["flags"] = rng.integers(1, 1 << 63, n, dtype=np.uint64), AL.SELECT
    kinds = np.zeros(16, np.int64)
    appended = 0
    for rnd in range(3):
        recs = s.next_round().copy()
        twin.step_begin_records(recs, B.STEP_READ_COMMITTED)
        twin.step_wait()
        c = _refresh(twin, n)
        cur = c.last_index[:n].copy()
        table = base.copy()
        table["run_start"] = cur - np.minimum(cur, rng.integers(0, 8, n).astype(np.uint64))
        table["run_term"] = terms
        frames = []
        for g in rng.permutation(n)[: 3 * n // 4].tolist():
            frames.append(A.frame(g, int(rng.integers(16)),
                                  E.random_frame(rng, int(cur[g]), int(table["run_start"][g]), int(terms[g]),
                                                 int(terms[g]), int(c.committed[g]), hostile=0.02)))
        frames += [frames[i] for i in rng.integers(0, len(frames), len(frames) // 8)]   # repeated frames: DUP
        blob, off = A.batch(frames)
        want_table = table.copy()
        want = AE.batch(c, None, want_table, blob, off)
        t_twin, t_a = table.copy(), table.copy()
        got = PF.device(twin, "follower_append_entries", blob, off, t_twin)
        PF.equal(want, tuple(got[:2]) + (got[2].view(AE.APPENDED_DTYPE),) + tuple(got[3:]), E.NAMES,
                   ("device form after the step", rnd))
        a.step_begin_records(recs, B.STEP_READ_COMMITTED)
        during = [x.copy() for x in PF.host(a, "follower_append_entries", blob, off, t_a)]
        a.step_wait()
        PF.equal(want, tuple(during[:2]) + (during[2].view(AE.APPENDED_DTYPE),) + tuple(during[3:]), E.NAMES,
                   ("host form during the step", rnd))
        assert np.array_equal(t_twin, want_table) and np.array_equal(t_a, want_table), rnd
        for x in (a, twin):
            st = FL.group_state(x, n)
            for name in ("committed", "last_index", "term", "term_start"):
                assert np.array_equal(st[name], getattr(c, name)[:n]), (rnd, name)
        kinds += np.bincount(want[0] >> 4, minlength=16)
        appended += int(np.count_nonzero(want[0] & B.FAPP_APPENDED))
    assert kinds[B.WIRE_OK] > 50_000 and kinds[B.WIRE_DUP] > 10_000 and appended > 20_000, (kinds, appended)
    a.close()
    twin.close()


def test_replication_round_trip_100k_x5():
    """A leader arena of 100K groups x 5 peers after synthetic steps.  Its state gives every follower the leader sends
    to a MsgAppend with the last k (0-4) entries of the log, encoded here from the arena's term, term_start, last_index
    and committed and the send's ids; the leader's progress says those entries are in flight (matched = m.index,
    next_idx = last_index + 1).  One follower arena per follower slot (the header g << 4 | slot names the follower's own
    group g) appends them with raftgpu_follower_append_entries_device; the responses go back as one wire batch through
    raftgpu_step_begin_wire, which advances the leaders' commits; raftgpu_append_frames, selected by the step's advanced
    bitmap, carries the commit back through raftgpu_follower_append.  Every follower ends with the leader's committed
    and last_index, and every stage equals its oracle."""
    n = 100_000
    rng = np.random.default_rng(0xAE80)
    s = B.Synth(n, 0xAE81, k_peers=5)
    la = B.Arena(n)
    assert la.group_alloc_range(n) == 0
    la.load_columns(s.initial)
    terms = rng.integers(1, 1000, n).astype(np.uint64)
    la.column_write(B.COL_TERM, 0, 0, terms)
    for _ in range(3):
        la.step_begin_records(s.next_round().copy(), B.STEP_READ_COMMITTED)
        la.step_wait()
    c = la.read_columns(n)
    c.term = terms.copy()
    last = c.last_index[:n].copy()
    assert np.all(last >= 8)
    # every send a Replicate one, the term started at most 4 entries back, so the entries in flight are of this term
    c.term_start[:n] = np.minimum(c.term_start[:n], last - 4)
    c.next_idx[:] = c.last_index[None, :] + 1
    c.pflags[:] = np.where((c.pflags & 3) == B.STATE_SNAPSHOT, c.pflags, B.STATE_REPLICATE)
    for k in range(B.SLOTS):
        la.column_write(B.COL_NEXT_IDX, k, 0, c.next_idx[k].copy())
        la.column_write(B.COL_PFLAGS, k, 0, c.pflags[k].copy())
    la.column_write(B.COL_TERM_START, 0, 0, c.term_start[:n].copy())
    ids = rng.integers(1, 1 << 63, (9, n), dtype=np.uint64)
    # which (group, slot) the leader sends to, with the send's ids: its entry-less frames
    rc, blob0, off0, rest0, tot0 = la.append_frames(0, n, ids)
    sends = [(int(h >> 4), int(h & 15), O.wire_decode_message(bytes(blob0[a + 4:b])))
             for h, a, b in zip(FL.headers(blob0, off0), off0[:-1].tolist(), off0[1:].tolist())]
    assert len(sends) > 3 * n, len(sends)
    # the entries in flight: k per send; the leader's progress says so
    ks = rng.integers(0, 5, len(sends))
    g_of = np.array([g for g, _, _ in sends])
    s_of = np.array([sl for _, sl, _ in sends])
    c.matched[s_of, g_of] = last[g_of] - ks.astype(np.uint64)
    c.peer_committed[s_of, g_of] = np.minimum(c.peer_committed[s_of, g_of], c.matched[s_of, g_of])
    for k in range(B.SLOTS):
        for col, name in ((B.COL_MATCHED, "matched"), (B.COL_PEER_COMMITTED, "peer_committed"),
                          (B.COL_NEXT_IDX, "next_idx")):
            la.column_write(col, k, 0, getattr(c, name)[k].copy())
    lcom = c.committed[:n].copy()
    fas, back = [], []
    for sl in range(B.SLOTS):
        idx = np.flatnonzero(s_of == sl)
        if len(idx) == 0:
            continue
        fc = O.new_columns(n, n)
        fc.term_start[:] = A.NO_TERM_START
        fl_last = last.copy()
        fl_last[g_of[idx]] -= ks[idx].astype(np.uint64)
        fc.term[:n], fc.last_index[:n] = terms, fl_last
        fc.committed[:n] = np.minimum(lcom, fl_last)
        table = np.zeros(n, AL.LOG_DTYPE)
        table["id"], table["flags"] = ids[sl], AL.SELECT
        table["run_start"], table["run_term"] = c.term_start[:n], terms
        frames = []
        for j in idx.tolist():
            g, _, m = sends[j]
            i0, t = int(fl_last[g]), int(terms[g])
            recs = [E.record(E.entry(t, i0 + 1 + e, data=bytes(int(rng.integers(0, 48))))) for e in range(int(ks[j]))]
            frames.append(A.frame(g, sl, E.message(t, t, i0, int(lcom[g]), int(m["from"]), recs, to=int(m["to"]))))
        fblob, foff = A.batch(frames)
        fa = B.Arena(n)
        assert fa.group_alloc_range(n) == 0
        for col, name in ((B.COL_TERM, "term"), (B.COL_LAST_INDEX, "last_index"), (B.COL_COMMITTED, "committed"),
                          (B.COL_TERM_START, "term_start")):
            fa.column_write(col, 0, 0, getattr(fc, name)[:n].copy())
        want_table = table.copy()
        w = AE.batch(fc, None, want_table, fblob, foff)
        assert np.all(w[0] >> 4 == B.WIRE_OK), np.bincount(w[0])
        assert np.array_equal(w[0] & B.FAPP_APPENDED != 0, ks[idx] > 0)
        got = PF.device(fa, "follower_append_entries", fblob, foff, table)
        PF.equal(w, tuple(got[:2]) + (got[2].view(AE.APPENDED_DTYPE),) + tuple(got[3:]), E.NAMES, ("follower slot", sl))
        assert np.array_equal(table, want_table)
        fcols = fa.read_columns(n)
        assert np.array_equal(fcols.last_index[g_of[idx]], last[g_of[idx]]), sl      # the follower holds the log
        fas.append((sl, fa, fc, table))
        back.append((w[3], w[4]))
    # the responses at the leader: one wire batch through a step
    rblob = np.concatenate([b for b, _ in back])
    base = np.cumsum([0] + [len(b) for b, _ in back])
    roff = np.concatenate([o[:-1].astype(np.int64) + base[k] for k, (_, o) in enumerate(back)] + [[base[-1]]])
    roff = roff.astype(np.uint32)
    nr = len(roff) - 1
    assert nr == len(sends)
    wst, recs, _, _ = O.wire_decode_batch(rblob, roff, n, c.term[:n])
    assert np.all(wst == B.WIRE_OK)
    O.arena_apply(c, recs, mode=0)
    O.arena_recompute(c)
    la.step_begin_wire(PF.host_batch(rblob, roff, len(rblob)), B.STEP_READ_COMMITTED)
    la.step_wait()
    assert np.all(la.wire_status() >> 4 == B.WIRE_OK)
    bm = la.step_results(n)[0].copy()
    lc = la.read_columns(n)
    for name in ("matched", "next_idx", "peer_committed", "pflags", "committed"):
        assert np.array_equal(getattr(lc, name), getattr(c, name)[..., :n]), name
    assert np.mean(lc.committed[g_of] == last[g_of]) > 0.99         # a quorum answered: the commit reached last_index
    # the commit back: entry-less MsgAppend frames of the advanced groups through raftgpu_follower_append
    rc, blob1, off1, rest1, tot1 = la.append_frames(0, n, ids, select=bm)
    hdr1 = FL.headers(blob1, off1)
    for sl, fa, fc, table in fas:
        idx = np.flatnonzero((hdr1 & 15) == sl)
        fblob, foff = A.batch([bytes(blob1[off1[i]:off1[i + 1]]) for i in idx.tolist()])
        w = AL.batch(fc, None, table, fblob, foff)
        got = PF.device(fa, "follower_append", fblob, foff, table)
        PF.equal(w, got, A.NAMES, ("commit back", sl))
        assert np.all(w[0] == A.LOG_STATUS_OK)
        fcols = fa.read_columns(n)
        mine = g_of[s_of == sl]
        assert np.array_equal(fcols.committed[mine], lc.committed[mine]), sl
        assert np.array_equal(fcols.last_index[mine], lc.last_index[mine]), sl
        fa.close()
    la.close()

