"""Every wire-frame pass past the prologue it shares with the others (k_wire.cuh: wire_stage_block, wire_open), in its
host and device form, against its oracle: batches whose blocks lie on both sides of the 16 KiB stage (ballast frames
that every pass skips), hostile offset layouts, the golden decoder vectors through every decoder instantiation, and
one store's receive buffer through all five passes.  The batches
are built on the CPU (wire_batches.py; test_wire_batches.py checks the geometries they reach).  Run with -m gpu."""
import types

import numpy as np
import pytest

from oracle import hb_follow_oracle as HL
from oracle import hb_frames_oracle as HF
from oracle import hb_wire_oracle as H
from oracle import vote_request_oracle as VR
from oracle import vote_wire_oracle as VW
from helpers import B, O, assert_columns_equal
from control_cmds import cmds
import hb_follow as FL
import hb_frames as F
import read_cases as R
import vote_frames as V
import vote_request_frames as Q
import wire_batches as WB
import test_gpu_heartbeat_follow as HFT
import test_gpu_heartbeat_wire as HWT
import test_gpu_vote_request_wire as VRT
import test_gpu_vote_wire as VWT
import test_gpu_wire as GW
import test_oracle_vote_request as TQ
import test_oracle_vote_wire as TV

pytestmark = pytest.mark.gpu

P = 8
U64_MAX = (1 << 64) - 1


def _host_batch(blob, off, n_bytes):
    """What the host forms read: .bytes (the batch and 16 spare bytes), .n_bytes, .offsets, .n, no records."""
    fb = F.Frames([])
    fb.bytes = np.concatenate([np.asarray(blob[:n_bytes], np.uint8), np.zeros(16, np.uint8)])
    fb.offsets, fb.n, fb.n_bytes = np.ascontiguousarray(off, np.uint32), len(off) - 1, int(n_bytes)
    return fb


def _split(blob, off):
    return [blob[a:b].tobytes() for a, b in zip(off[:-1].tolist(), off[1:].tolist())]


def _equal(want, got, names, what):
    for w, g, name in zip(want, got, names):
        assert w.shape == g.shape and np.array_equal(w, g), (what, name, np.flatnonzero(w != g)[:5] if w.shape == g.shape
                                                              else (w.shape, g.shape))


# --------------------------------------------------------------------------- the five passes
# Each pass: frames(rng) builds its scenario's frames on the CPU; fresh() an arena and the oracle's state in the same
# state; run() one batch through the arena (host or device form) and the oracle, compares every output and returns the
# outputs, the status bytes (WIRE_* << 4 | low nibble) first; PER_FRAME names the outputs with one row per frame;
# check() compares the arena with the oracle's state.


class Leaders:
    """Leaders set up by a control list, with group terms in the term column and read requests queued: the
    AppendResponse step (kind "append") or the heartbeat-response pass with read queues (kind "heartbeat")."""

    PER_FRAME = (0,)

    def __init__(self, kind, n, setup, terms, reqs):
        self.kind, self.n, self.setup, self.reqs = kind, n, setup, reqs
        self.terms = np.zeros(n + 64, np.uint64)
        self.terms[:n] = terms
        self.d = self._driver()

    def _driver(self):
        d = R.OracleDriver(self.n, max_pending=P)
        d.q.control(d.c, d.votes, self.setup)
        d.c.term[: self.n] = self.terms[: self.n]
        if len(self.reqs):
            d.q.request(d.c, self.reqs)
        return d

    def frames(self, rng, k=None):
        blob, off = HWT._mixed_batch(rng, self.d, self.n, self.terms, True, k or self.n)
        return _split(blob, off)

    def fresh(self):
        a = B.Arena(self.n + 64)
        a.enable_read_index(P)
        assert a.group_alloc_range(self.n) == 0
        a.control(self.setup)
        a.column_write(B.COL_TERM, 0, 0, self.terms[: self.n].copy())
        if len(self.reqs):
            a.read_index_request(self.reqs)
        return a, self._driver()

    def run(self, a, d, buf, n_bytes, off, device, what):
        n = len(off) - 1
        if self.kind == "append":
            if device:
                bufs = [a.device_alloc(x) for x in (len(buf) + 16, 4 * (n + 1), max(1, n))]
                a.h2d(bufs[0], buf), a.h2d(bufs[1], off)
                a.wire_apply_device(bufs[0], n_bytes, bufs[1], n, bufs[2])
                a.synchronize()
                got = np.zeros(n, np.uint8)
                a.d2h(got, bufs[2])
                for p in bufs:
                    a.device_free(p)
                want = HWT._oracle_append(d.c, buf, off, self.n, self.terms, n_bytes=n_bytes)
            else:
                fb = _host_batch(buf, off, n_bytes)
                fb.records = None
                a.step_begin_wire(fb, B.STEP_READ_COMMITTED)
                sr = a.step_wait()
                got = a.wire_status().copy()
                want, bm, adv, _ = GW.oracle_wire_step(d.c, fb, self.n, self.terms)
                gbm, _ = a.step_results(self.n)
                assert np.array_equal(gbm, bm[: len(gbm)]) and sr.n_advanced == adv, what
            _equal([want], [got], ["status"], what)
            return (got,)
        if device:
            bufs = [a.device_alloc(x) for x in (len(buf) + 16, 4 * (n + 1), max(1, n), 24 * n * P, 8)]
            a.h2d(bufs[0], buf), a.h2d(bufs[1], off)
            a.heartbeat_wire_device(bufs[0], n_bytes, bufs[1], n, bufs[2], bufs[3], n * P, bufs[4])
            a.synchronize()
            st, cnt = np.zeros(n, np.uint8), np.zeros(1, np.uint64)
            a.d2h(st, bufs[2]), a.d2h(cnt, bufs[4])
            rel = np.zeros(int(cnt[0]), B.READ_STATE_DTYPE)
            if len(rel):
                a.d2h(rel, bufs[3])
            for p in bufs:
                a.device_free(p)
        else:
            st, rel = a.heartbeat_wire(_host_batch(buf, off, n_bytes))
        want, want_rel = H.apply(d.c, d.q, buf, off, self.terms, n_bytes=n_bytes)
        got = (st, R.by_group(rel))
        _equal([want, R.by_group(want_rel)], got, ["status", "released reads"], what)
        return got

    def check(self, a, d, what):
        assert_columns_equal(a.read_columns(self.n), d.c, self.n, what)
        HWT._queues_equal(a, d.q, self.n, what)


def random_leaders(kind, seed, n):
    """Leaders with random configurations (read_cases.random_setup), terms 1..3 (0 for a tenth: not checked) and
    random read requests."""
    rng = np.random.default_rng(seed)
    setup = R.random_setup(rng, n, 0)
    terms = rng.integers(1, 4, n).astype(np.uint64)
    terms[rng.random(n) < 0.1] = 0
    return Leaders(kind, n, setup, terms, R.random_requests(rng, n, 2.0, 12))


class Followers:
    """Followers whose group columns (term, last_index, term_start, committed) are written directly, with the
    selection bitmap and self ids the caller passes: the follower pass.  frames: the random scenario's heartbeats."""

    PER_FRAME = (0, 1)

    def __init__(self, n, cols, sel, ids, frames=None):
        self.n, self.cols, self.sel, self.ids, self._frames = n, cols, sel, ids, frames

    def frames(self, rng):
        return self._frames(rng)

    def fresh(self):
        a = B.Arena(self.n + 64)
        assert a.group_alloc_range(self.n) == 0
        for col, arr in self.cols.items():
            a.column_write(col, 0, 0, arr)
        c = a.read_columns(self.n)
        c.term = self.cols[B.COL_TERM].copy()
        return a, c

    def run(self, a, c, buf, n_bytes, off, device, what):
        want = HL.follower_heartbeats(c, None, buf, off, self.sel, self.ids, n_bytes=n_bytes)
        if device:
            got = HFT._device(a, buf, off, self.sel, self.ids, n_bytes=n_bytes)
        else:
            ids, sel = np.zeros(a.cap, np.uint64), np.zeros((a.cap + 31) // 32, np.uint32)
            ids[: self.n], sel[: len(self.sel)] = self.ids, self.sel
            got = a.follower_heartbeat(_host_batch(buf, off, n_bytes), ids, sel)
        _equal(want, got, ("status", "from", "response bytes", "response offsets", "totals"), what)
        return got

    def check(self, a, c, what):
        s = HFT._group_state(a, self.n)
        for name, col in s.items():
            assert np.array_equal(col, getattr(c, name)[: self.n]), (what, name)


def random_followers(seed, n):
    """Followers fed with the heartbeat-frames oracle's MsgHeartbeat frames, most at their term and below their log's
    end, a few unselected."""
    rng = np.random.default_rng(seed)
    lc = O.new_columns(n, n)
    lc.meta[:] = B.make_meta(0b11, 0, 0, 0)
    lc.term_start[:] = 1
    lc.term[:] = rng.integers(1, 1 << 33, n)
    lc.committed[:] = rng.integers(0, 1 << 40, n)
    lc.matched[1] = rng.integers(0, 1 << 40, n)
    q = R.RO.ReadQueues(n, 1)
    q.allocated[:] = 1
    q.count[:] = rng.random(n) < 0.75
    q.ctx[:, 0] = rng.integers(1, 1 << 63, n, dtype=np.uint64)
    hb, hoff, _ = HF.bcast_heartbeats(lc, q, 0, n, rng.integers(1, 1 << 63, (9, n), dtype=np.uint64))
    perm = rng.permutation(n).astype(np.uint32)
    commit = np.minimum(lc.matched[1], lc.committed)
    cols = {B.COL_TERM: np.zeros(n, np.uint64), B.COL_LAST_INDEX: np.zeros(n, np.uint64),
            B.COL_TERM_START: np.where(rng.random(n) < 0.05, np.uint64(1), np.uint64(B.NO_TERM_START))}
    cols[B.COL_TERM][perm] = lc.term + (rng.random(n) < 0.05).astype(np.uint64)
    cols[B.COL_LAST_INDEX][perm] = commit + rng.integers(0, 1000, n).astype(np.uint64) - \
        (rng.random(n) < 0.02).astype(np.uint64) * np.minimum(commit, np.uint64(1001))
    last = cols[B.COL_LAST_INDEX]
    cols[B.COL_COMMITTED] = last - np.minimum(last, rng.integers(0, 2000, n).astype(np.uint64))

    def frames(rng):
        hdr = perm << 4 | rng.integers(0, 16, n).astype(np.uint32)
        out = _split(FL.with_headers(hb, hoff, hdr), hoff)
        out += [out[i] for i in rng.integers(0, len(out), len(out) // 10)]         # repeated heartbeats: DUP
        return [out[i] for i in rng.permutation(len(out))]

    return Followers(n, cols, FL.bitmap(rng.random(n) < 0.95), HFT._self_ids(rng, n), frames)


class Candidates:
    """Candidates polling, set up like a vote_frames.Election (setup and campaign control lists; e.frames the random
    scenario's responses), with the select and pre bitmaps: the vote-response pass."""

    PER_FRAME = (0,)

    def __init__(self, e, sel, pre):
        self.e, self.n = e, e.n
        pad = np.zeros(4, np.uint32)
        self.sel, self.pre = np.concatenate([sel, pad]), np.concatenate([pre, pad])

    def frames(self, rng):
        return self.e.frames(rng, commit_vote=True)

    def fresh(self):
        return VWT._arena(self.e), TV._state(self.e)

    def run(self, a, state, buf, n_bytes, off, device, what):
        c, vt = state
        want_st, want_out, _ = VW.batch(c, vt, buf, off, self.sel, self.pre, n_bytes=n_bytes)
        got = VWT._device(a, buf, off, self.sel, self.pre, n_bytes=n_bytes) if device else \
            a.vote_wire(_host_batch(buf, off, n_bytes), self.sel, self.pre)
        _equal([want_st, want_out], got, ("status", "outcomes"), what)
        return got

    def check(self, a, state, what):
        assert np.array_equal(VWT._votes(a, self.n), state[1][:, : self.n]), what


def random_candidates(seed, n_narrow, n_wide):
    e = V.Election(np.random.default_rng(seed), n_narrow, n_wide)
    return Candidates(e, e.select(), e.pre())


class Voters:
    """Voters set up like a vote_request_frames.Scenario (s.setup, the caller's table s.table; s.frames the random
    scenario's requests): the vote-request pass."""

    PER_FRAME = (0, 1)

    def __init__(self, s):
        self.s, self.n = s, s.n

    def frames(self, rng):
        return self.s.frames(rng)

    def fresh(self):
        return VRT._arena_of(self.s), TQ.state_of(self.s)

    def run(self, a, state, buf, n_bytes, off, device, what):
        c, vt = state
        want = VR.batch(c, None, vt, buf, off, self.s.table, n_bytes=n_bytes)
        got = VRT._device(a, buf, off, self.s.table, n_bytes=n_bytes) if device else \
            a.vote_request_wire(_host_batch(buf, off, n_bytes), self.s.table)
        _equal(want, got, ("status", "out", "response bytes", "response offsets", "totals"), what)
        return got

    def check(self, a, state, what):
        c, vt = state
        cols = VRT._columns(a, self.n)
        for name in VRT.ARENA_COLUMNS + ("term",):
            assert np.array_equal(cols[name], getattr(c, name)[..., : self.n]), (what, name)
        assert np.array_equal(VRT._votes(a, self.n), vt[:, : self.n]), what


PASSES = ("append", "heartbeat", "follower", "vote", "voter")


def scenario(name, n=20_000):
    """Each pass's random scenario at about n groups (a few of them wide pairs where the pass takes them)."""
    if name in ("append", "heartbeat"):
        return random_leaders(name, 0x57A6 + len(name), n)
    if name == "follower":
        return random_followers(0x57A7, n)
    if name == "vote":
        return random_candidates(0x57A8, n - 400, 200)
    return Voters(Q.Scenario(np.random.default_rng(0x57A9), n - 400, 200))


def stage_batch(sc, seed):
    """The scenario's frames with the ballast of WB.across_the_stage -> (frames, ballast mask)."""
    rng = np.random.default_rng(seed)
    return WB.across_the_stage(sc.frames(rng), rng)


def hostile_batches(sc, seed, device):
    """WB.hostile over the scenario's frames for every case of WB.hostile_cases -> [(buf, n_bytes, offsets)]: a device
    buffer holds 4 KiB or more of valid frames past n_bytes, and only offsets that end on those frames' boundaries go past
    n_bytes; a host batch's offsets go at most 4 (n + 1) bytes past n_bytes, into the offsets the same call copies in."""
    rng = np.random.default_rng(seed)
    frames = sc.frames(rng)
    tail, bounds = WB.slack(frames[::-1])
    out = []
    for n, r in WB.hostile_cases():
        past = bounds if device else np.arange(4 * (n + 1) + 1)
        blob, off = WB.hostile(frames[int(rng.integers(0, len(frames) - n - 1)):], rng, n, r, past)
        buf = np.concatenate([blob, np.frombuffer(tail, np.uint8)]) if device else blob
        out.append((buf, len(blob), off))
    return out


# --------------------------------------------------------------------------- 1. across the stage


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("name", PASSES)
def test_every_pass_across_the_stage(name, device):
    """A batch whose blocks are staged, unstaged by their span at 16384 / 16385 bytes from both ends of a 16-byte line,
    or hold frames past 16 KiB and 64 KiB, against the oracle; and the same frames without the ballast through a
    second arena: the same statuses and outputs for every frame, the same arena."""
    sc = scenario(name)
    frames, ballast = stage_batch(sc, 0x5B00 + PASSES.index(name))
    blob, off = F.batch(frames)
    assert WB.geometry(off, len(blob)) >= {WB.STAGED, WB.SPAN, "frame>16K", "frame>64K"}
    a, st = sc.fresh()
    got = sc.run(a, st, blob, len(blob), off, device, (name, "ballast"))
    sc.check(a, st, (name, "ballast"))
    assert np.all(got[0][ballast] >> 4 == B.WIRE_SKIP_TYPE)
    assert np.count_nonzero(got[0][~ballast] >> 4 == B.WIRE_OK) > 1000
    # the oracle-free property: without the ballast, every other frame is decided the same way
    a2, st2 = sc.fresh()
    blob2, off2 = F.batch([f for f, b in zip(frames, ballast) if not b])
    got2 = sc.run(a2, st2, blob2, len(blob2), off2, device, (name, "plain"))
    for k, (x, y) in enumerate(zip(got, got2)):
        assert np.array_equal(x[~ballast] if k in sc.PER_FRAME else x, y), (name, "output", k)
    sc.check(a2, st, (name, "plain against the ballast run"))
    a.close()
    a2.close()


# --------------------------------------------------------------------------- 2. hostile offsets


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("name", PASSES)
def test_hostile_offsets(name, device):
    """Descending offsets, frames past n_bytes, frames of 0 to 3 bytes, a valid frame before offsets[0], n_bytes at every
    residue mod 16 and n in {1, 255, 256, 257}: statuses equal the oracle's, and the arena stays the oracle's (a
    MALFORMED frame changes nothing).  The device form is the one that catches a missing `b > n_bytes` guard: its buffer
    holds valid frames past n_bytes, and its frames past n_bytes end on their boundaries.  The host form copies only the
    batch, and its offsets past n_bytes reach only the offsets the same call copies in (after at most 15 bytes left by
    the batch of valid frames it runs first); that keeps every read inside the staging buffer."""
    sc = scenario(name, 2_000)
    a, st = sc.fresh()
    seen = np.zeros(16, np.int64)
    if not device:
        blob, off = F.batch(sc.frames(np.random.default_rng(1)))
        sc.run(a, st, blob, len(blob), off, False, (name, "valid"))
    for k, (buf, n_bytes, off) in enumerate(hostile_batches(sc, 0x5B10 + PASSES.index(name), device)):
        got = sc.run(a, st, buf, n_bytes, off, device, (name, k))[0]
        sc.check(a, st, (name, k))
        seen += np.bincount(got >> 4, minlength=16)
    assert seen[B.WIRE_MALFORMED] > 100 and seen[B.WIRE_SKIP_TYPE] + seen[B.WIRE_OK] > 100, seen
    a.close()


# --------------------------------------------------------------------------- 3. the golden encodings, every decoder

GOLDEN_TYPE = {"append": 4, "heartbeat": 9, "follower": 8, "vote": 6, "voter": 5}
CAP = 1 << 62                                            # log positions stay below this (SET_CONF takes last + 1)


def golden_scenario(name, variant):
    """One group per messages.json vector (WB.retarget to the pass's type; a rejected vector as it is), its state
    derived from the vector's decoded fields so that most frames reach the pass's decision:
      append, heartbeat: a leader of voters {0, 1, 2} at m.term, a read pending under an 8-byte context;
      follower: a selected follower at m.term whose log reaches m.commit, self id g + 1;
      vote: a candidate at m.term whose committed is m.commit (variant 0) or one below it (variant 1: a rejection with
        commit_term is COMMIT_VOTE);
      voter: a selected follower at m.term with last_index = m.index and last_term = m.log_term (up to date), whose
        priority is m.priority (variant 0: granted) or one more (variant 1: rejected, committed one below m.commit).
    -> (scenario, frames, the vectors' kinds, their python-protobuf verdicts)."""
    vs = WB.golden()
    n = len(vs)
    typ = GOLDEN_TYPE[name]
    raws, fields = zip(*[WB.retarget(v, typ) for v in vs])
    f = [x or {} for x in fields]
    get = lambda k: np.array([int(x.get(k, 0)) for x in f], dtype=np.uint64)
    term, commit, index = get("term"), get("commit"), get("index")
    frames = [F.frame(g, 1, raws[g]) for g in range(n)]
    kinds = np.array([v["kind"] for v in vs])
    ok = np.array([v["ok"] for v in vs])
    if name in ("append", "heartbeat"):
        setup = cmds(*[r for g in range(n) for r in ((B.CTL_SET_CONF, g, 0, 0, (0b111, 0, 0, 11)),
                                                     (B.CTL_RESET, g, 0, 0, (11, 10, 5, 10)), (B.CTL_BECOME_LEADER, g))])
        ctx = [(g, int.from_bytes(m["context"], "little")) for g, m in enumerate(H.decode_message(r) for r in raws)
               if m is not None and len(m["context"]) == 8]
        return Leaders(name, n, setup, term, R.reqs(*ctx)), frames, kinds, ok
    capped = np.minimum(commit, np.uint64(CAP))
    if name == "follower":
        cols = {B.COL_TERM: term, B.COL_LAST_INDEX: np.maximum(capped, np.uint64(10)),
                B.COL_COMMITTED: np.full(n, 5, np.uint64), B.COL_TERM_START: np.full(n, B.NO_TERM_START, np.uint64)}
        return Followers(n, cols, FL.bitmap(np.ones(n, bool)), np.arange(1, n + 1, dtype=np.uint64)), frames, kinds, ok
    below = ((commit > 0) & (commit <= CAP)).astype(np.uint64)
    if name == "vote":
        com = capped - below * np.uint64(variant)
        last = com + np.uint64(10)
    else:
        last = np.minimum(index, np.uint64(CAP))
        com = np.minimum(capped - below, last)
    rows, camp = [], []
    for g in range(n):
        rows += [(B.CTL_SET_CONF, g, 0, 0, (0b111, 0, 0, int(last[g]) + 1)),
                 (B.CTL_RESET, g, 0, 0, (B.NO_TERM_START, int(last[g]), int(com[g]), int(last[g])))]
        if term[g]:
            rows.append((B.CTL_SET_TERM, g, 0, 0, (int(term[g]),)))
        camp += [(B.CTL_RESET_VOTES, g), (B.CTL_RECORD_VOTE, g, 0, 1), (B.CTL_VOTE_RESULT, g)]
    e = types.SimpleNamespace(n=n, n_narrow=n, n_wide=0, setup=cmds(*rows), campaign=cmds(*camp))
    if name == "vote":
        return Candidates(e, V.bitmap(np.ones(n, bool)), V.bitmap(np.zeros(n, bool))), frames, kinds, ok
    e.campaign = None
    e.table = Q.voters(n)
    e.table["id"], e.table["last_term"], e.table["persisted"] = np.arange(1, n + 1), get("log_term"), last
    e.table["commit_term"], e.table["flags"] = 3, B.VOTER_SELECT
    pri = get("priority")
    e.table["priority"] = pri if variant == 0 else np.where(pri < np.uint64(U64_MAX), pri + np.uint64(1), pri)
    return Voters(e), frames, kinds, ok


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("name", PASSES)
def test_golden_encodings_through_every_decoder(name, device):
    """python-protobuf's verdicts on canonical, non-canonical and edge encodings (padded varints, repeated fields,
    unknown fields, known fields of the wrong wire type, 10-byte varints) through every wire_decode instantiation:
    every output against the oracle, so the fields each pass echoes or decides on -- from (3: d_from, d_out, the
    response's to), term, context (12), priority (14), commit_term (15) and commit -- are the golden ones.  A rejected
    vector is MALFORMED everywhere; both the non_canonical and the edge vectors reach OK."""
    seen = {}
    for variant in (0, 1) if name in ("vote", "voter") else (0,):
        sc, frames, kinds, ok = golden_scenario(name, variant)
        blob, off = F.batch(frames)
        a, st = sc.fresh()
        got = sc.run(a, st, blob, len(blob), off, device, (name, variant))
        sc.check(a, st, (name, variant))
        a.close()
        status = got[0] >> 4
        assert np.all(status[~ok] == B.WIRE_MALFORMED), (name, variant)
        assert np.all(status[ok] != B.WIRE_MALFORMED), (name, variant, np.flatnonzero(ok & (status == B.WIRE_MALFORMED)))
        for k in ("non_canonical", "edge"):
            seen[k] = seen.get(k, 0) + int(np.count_nonzero((kinds == k) & (status == B.WIRE_OK)))
        seen["ok"] = seen.get("ok", 0) + int(np.count_nonzero(status == B.WIRE_OK))
    assert seen["non_canonical"] > 0 and seen["edge"] > 0 and seen["ok"] > len(frames) // 3, (name, seen)


# --------------------------------------------------------------------------- 4. one receive buffer, five passes


def test_store_buffer_through_every_pass():
    """One store's receive buffer -- MsgAppendResponse (4) and MsgHeartbeatResponse (9) to leaders, vote responses (6)
    to candidates, MsgHeartbeat (8) to followers, MsgRequestVote (5) and MsgRequestPreVote (17) to followers and
    candidates, and ballast -- through the five passes in a fixed order on one arena, each against its oracle on the
    shared oracle state: a frame is OK in at most one pass, and in the pass of its type whenever it is well-formed for
    it."""
    rng = np.random.default_rng(0x5B20)
    e = V.Election(rng, 6000, 0, p_role=(0.3, 0.2, 0.25, 0.25))
    n = e.n
    a = VWT._arena(e)
    c, vt = TV._state(e)
    table = Q.voters(n)
    table["id"] = e.self_slot + 1
    table["last_term"] = e.term
    table["flags"] = np.where(e.role == V.LEADER, 0, B.VOTER_SELECT)
    follower = e.role == V.FOLLOWER
    ids = (e.self_slot + 1).astype(np.uint64)
    frames, kind = [], []
    for g in range(n):
        t, com, li = int(e.term[g]), int(e.committed[g]), int(e.last[g])
        peers = [s for s in range(1, 5) if int(e.present[g]) >> s & 1 and s != e.self_slot[g]]
        if e.role[g] == V.LEADER:
            for s in peers:
                frames += [F.frame(g, s, F.message(4, term=t, index=li)), F.frame(g, s, F.message(9, term=t, commit=com))]
                kind += [4, 9]
        if follower[g]:
            frames.append(F.frame(g, 1, F.message(8, term=t, commit=min(com, li), frm=2)))
            kind.append(8)
        if e.role[g] != V.LEADER and rng.random() < 0.5:
            typ = Q.PRE_VOTE if rng.random() < 0.5 else Q.VOTE
            frames.append(F.frame(g, 0, Q.request(typ, t + 1, t, li, frm=int(rng.integers(1, 6)))))
            kind.append(typ)
    for f in e.frames(rng, noise=False):
        frames.append(f)
        kind.append(6)
    order = rng.permutation(len(frames))
    frames, kind = [frames[i] for i in order], np.array(kind)[order]
    frames, ballast = WB.across_the_stage(frames, rng)
    kinds = np.zeros(len(frames), np.int64)
    kinds[~ballast] = kind
    blob, off = F.batch(frames)
    assert WB.geometry(off, len(blob)) >= {WB.STAGED, WB.SPAN, "frame>16K", "frame>64K"}
    nb = len(blob)
    terms = np.zeros(a.cap, np.uint64)
    terms[:n] = c.term[:n]
    sel_f, pad = FL.bitmap(follower), np.zeros(4, np.uint32)
    sel_v, pre_v = np.concatenate([e.select(), pad]), np.concatenate([e.pre(), pad])
    ok = []
    # 1. the AppendResponse step
    fb = _host_batch(blob, off, nb)
    fb.records = None
    a.step_begin_wire(fb)
    a.step_wait()
    got = a.wire_status().copy()
    want, _, _, _ = GW.oracle_wire_step(c, fb, n, terms)
    _equal([want], [got], ["status"], "append")
    ok.append((got >> 4 == B.WIRE_OK, 4))
    # 2. heartbeat responses
    got, _ = a.heartbeat_wire(fb)
    want, _ = H.apply(c, None, blob, off, terms)
    _equal([want], [got], ["status"], "heartbeat")
    ok.append((got >> 4 == B.WIRE_OK, 9))
    # 3. vote responses
    got = a.vote_wire(fb, sel_v, pre_v)
    want = VW.batch(c, vt, blob, off, sel_v, pre_v)[:2]
    _equal(want, got, ("status", "outcomes"), "vote")
    ok.append((got[0] >> 4 == B.WIRE_OK, 6))
    # 4. heartbeats at the followers
    full_ids, full_sel = np.zeros(a.cap, np.uint64), np.zeros((a.cap + 31) // 32, np.uint32)
    full_ids[:n], full_sel[: len(sel_f)] = ids, sel_f
    got = a.follower_heartbeat(fb, full_ids, full_sel)
    want = HL.follower_heartbeats(c, None, blob, off, sel_f, ids)
    _equal(want, got, ("status", "from", "response bytes", "response offsets", "totals"), "follower")
    ok.append((got[0] >> 4 == B.WIRE_OK, 8))
    # 5. vote requests
    got = a.vote_request_wire(fb, table)
    want = VR.batch(c, None, vt, blob, off, table)
    _equal(want, got, ("status", "out", "response bytes", "response offsets", "totals"), "voter")
    ok.append((got[0] >> 4 == B.WIRE_OK, (5, 17)))
    assert_columns_equal(a.read_columns(n), c, n, "store buffer")
    assert np.array_equal(VWT._votes(a, n), vt[:, :n])
    assert np.array_equal(a.column_read(B.COL_TERM, 0, 0, n, np.uint64), c.term[:n])
    hits = np.stack([x for x, _ in ok])
    assert np.all(hits.sum(0) <= 1)
    for row, (x, k) in enumerate(ok):
        mine = np.isin(kinds, k)
        assert np.all(x <= mine) and x[mine].mean() > 0.5, (k, x[mine].mean())
    assert not hits[:, ballast].any()
    a.close()
