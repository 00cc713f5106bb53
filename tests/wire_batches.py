"""Wire batches at the edges of the prologue every wire-frame pass shares (k_wire.cuh: wire_stage_block, wire_open,
wire_decode): the stage rule restated, ballast frames that place a batch's blocks on both sides of the 16 KiB stage,
hostile offset layouts, the golden decoder vectors retargeted to another message type, and each pass's scenario --
an arena and its oracle state in step, one batch through both and the comparison.  The CPU tests
(test_wire_batches.py) check what these batches reach, the GPU tests (test_gpu_wire_batches.py) run them."""
import json
import os
import types

import numpy as np

from oracle import hb_follow_oracle as HL
from oracle import hb_frames_oracle as HF
from oracle import hb_wire_oracle as H
from oracle import vote_request_oracle as VR
from oracle import vote_wire_oracle as VW
from helpers import B, O, arena_of, assert_columns_equal, check_columns, oracle_wire_step, oracle_wire_apply, votes
from control_cmds import cmds
import hb_follow as FL
import hb_frames as F
import pass_forms as PF
import read_cases as R
import vote_frames as V
import vote_request_frames as Q

THREADS, STAGE = 256, 16 * 1024            # kWireThreads, kWireStage
STAGED, SPAN, ORDER, PAST = "staged", "span", "order", "past"
MSG_APPEND, MSG_SNAPSHOT = 3, 7            # the ballast types: SKIP_TYPE in every pass
HERE = os.path.dirname(os.path.abspath(__file__))


def stage_blocks(offsets, n_bytes):
    """wire_stage_block for every block of 256 frames: STAGED when offsets[first] <= offsets[last] <= n_bytes and
    offsets[last] - (offsets[first] & ~15) <= 16384, else why not -- ORDER, PAST or SPAN, checked in that order."""
    off = np.asarray(offsets, np.int64)
    n = len(off) - 1
    out = []
    for first in range(0, n, THREADS):
        lo, hi = int(off[first]), int(off[min(first + THREADS, n)])
        out.append(ORDER if lo > hi else PAST if hi > n_bytes else SPAN if hi - (lo & ~15) > STAGE else STAGED)
    return out


def geometry(offsets, n_bytes):
    """The stage geometries a batch reaches: the set of stage_blocks' verdicts, plus ("span", span, lo % 16, staged) for
    blocks that span exactly 16384 or 16385 bytes, "partial" for a last block of fewer than 256 frames, and "frame>16K" /
    "frame>64K" for frames (inside the batch) that long."""
    off = np.asarray(offsets, np.int64)
    n = len(off) - 1
    got = set(stage_blocks(off, n_bytes))
    for first in range(0, n, THREADS):
        lo, hi = int(off[first]), int(off[min(first + THREADS, n)])
        if hi - (lo & ~15) in (STAGE, STAGE + 1):
            got.add(("span", hi - (lo & ~15), lo % 16, hi - (lo & ~15) <= STAGE))
    if n % THREADS:
        got.add("partial")
    sizes = np.diff(off)[(np.diff(off) > 0) & (off[1:] <= n_bytes)]
    if (sizes > STAGE).any():
        got.add("frame>16K")
    if (sizes > 64 * 1024).any():
        got.add("frame>64K")
    return got


# every geometry the GPU tests must reach (the stage rule's four verdicts, both sides of its span limit at both ends of
# a 16-byte line, a partial last block and frames past 16 KiB and 64 KiB)
WANT_GEOMETRY = {STAGED, SPAN, ORDER, PAST, "partial", "frame>16K", "frame>64K"} | \
    {("span", s, r, s == STAGE) for s in (STAGE, STAGE + 1) for r in (0, 15)}


def _payload(k):
    return (np.arange(k, dtype=np.int64) * 37 % 251).astype(np.uint8).tobytes()


def ballast(size, kind=MSG_APPEND, group=0):
    """A frame of exactly `size` (>= 8) bytes, header included, naming `group` slot 0: a MsgAppend whose entries field
    (7) holds the bytes, or a MsgSnapshot whose snapshot field (9) does.  Every pass skips it (SKIP_TYPE)."""
    field = 7 if kind == MSG_APPEND else 9
    for pad in (b"", F.varint(6 << 3) + b"\x01"):      # index = 1 bridges the sizes a longer length varint skips
        head = bytes([0x08, kind]) + pad + F.varint(field << 3 | 2)
        for vl in (1, 2, 3, 4):
            p = size - 4 - len(head) - vl
            if p >= 0 and len(F.varint(p)) == vl:
                return F.frame(group, 0, head + F.varint(p) + _payload(p))
    raise ValueError(size)


def across_the_stage(frames, rng, group=0):
    """The frames in order with ballast frames interleaved so that the batch reaches WANT_GEOMETRY's valid geometries:
    blocks spanning exactly 16384 and 16385 bytes from offsets[first] % 16 = 0 and 15 (each after a staged block whose
    last frame is the ballast that sets that residue), a block holding a frame past 16 KiB, one holding a frame past
    64 KiB, small ballast frames everywhere else, and a partial last block -> (frames, ballast mask)."""
    out, mask, it = [], [], iter(frames)
    pos = 0

    def put(f, is_ballast):
        nonlocal pos
        out.append(f)
        mask.append(is_ballast)
        pos += len(f)

    def take(k):
        got = [next(it) for _ in range(k)]
        return got, sum(len(f) for f in got)

    def block(kind, size_of):
        """255 scenario frames and one ballast frame at a random place in the block, sized by size_of(bytes of the 255)"""
        got, nb = take(THREADS - 1)
        at = int(rng.integers(0, THREADS))
        for f in got[:at] + [None] + got[at:]:
            put(ballast(size_of(nb), kind, group) if f is None else f, f is None)

    for k, (span, r) in enumerate([(STAGE, 0), (STAGE, 15), (STAGE + 1, 0), (STAGE + 1, 15), (None, 0), (None, 1)]):
        got, nb = take(THREADS - 1)                    # a staged block that ends on the residue r
        for f in got:
            put(f, False)
        put(ballast(24 + (r - pos - 24) % 16, MSG_SNAPSHOT, group), True)
        assert pos % 16 == r
        kind = MSG_APPEND if k % 2 else MSG_SNAPSHOT
        if span is not None:
            block(kind, lambda nb: span - r - nb)
        else:                                          # one frame past 16 KiB, or past 64 KiB
            big = STAGE + 1 if r == 0 else 64 * 1024 + 1
            block(kind, lambda nb: big + int(rng.integers(0, 4096)))
    for f in it:
        put(f, False)
        if rng.random() < 0.02:
            put(ballast(int(rng.integers(8, 400)), int(rng.choice([MSG_APPEND, MSG_SNAPSHOT])), group), True)
    if len(out) % THREADS == 0:
        put(ballast(40, MSG_APPEND, group), True)
    return out, np.array(mask, bool)


def slack(frames, at_least=4096):
    """Valid frames of at least `at_least` bytes, for the bytes a device buffer holds past n_bytes -> (bytes, the frame
    boundaries relative to n_bytes)."""
    got, nb = [], 0
    for f in frames:
        if nb >= at_least:
            break
        got.append(f)
        nb += len(f)
    assert nb >= at_least
    return b"".join(got), np.concatenate([[0], np.cumsum([len(f) for f in got])]).astype(np.int64)


def hostile(frames, rng, n, residue, past):
    """n frames over a batch of n_bytes = residue (mod 16) bytes, with a valid frame and some bytes before offsets[0],
    descending offset pairs, frames of 0 to 3 bytes and frames that end past n_bytes.  past: the offsets past n_bytes a
    frame may use, relative to n_bytes and > 0 (the boundaries of the valid frames of `slack`, or the bytes the host
    form copies in after the batch).  The last offset is past n_bytes when residue // 4 is 0, below offsets[0] when it
    is 1 -> (blob of n_bytes bytes, offsets u32[n + 1])."""
    frames = [frames[k % len(frames)] for k in range(n + 1)]
    body = frames[1:]
    nb = len(frames[0]) + sum(len(f) for f in body)
    prefix = frames[0] + bytes(int(rng.integers(0, 16)) * 16 + (residue - nb) % 16)
    blob = np.frombuffer(prefix + b"".join(body), np.uint8).copy()
    n_bytes = len(blob)
    assert n_bytes % 16 == residue
    off = np.concatenate([[len(prefix)], len(prefix) + np.cumsum([len(f) for f in body])]).astype(np.int64)
    past = np.asarray([p for p in past if p > 0], np.int64)
    edits = rng.choice(n, max(1, n // 12), replace=False) if n > 1 else [0]
    for i in edits:
        kind = int(rng.integers(3)) if n > 1 else residue % 3
        if kind == 0:          # a frame of 0 to 3 bytes (the next one starts inside this one's bytes)
            off[i + 1] = min(off[i] + int(rng.integers(0, 4)), n_bytes)
        elif kind == 1:        # a descending pair
            off[i + 1] = max(0, off[i] - int(rng.integers(1, 64)))
        elif i + 1 < n:        # a frame from a slack boundary to the next one, past n_bytes
            k = int(rng.integers(0, len(past) - 1))
            off[i], off[i + 1] = n_bytes + past[k] if k else off[i], n_bytes + past[k + 1]
    if residue // 4 == 0:
        off[n] = n_bytes + int(past[-1])
    elif residue // 4 == 1:
        off[n] = off[0] - 1
    assert off.min() >= 0 and off.max() <= n_bytes + past.max()
    return blob, off.astype(np.uint32)


def hostile_cases():
    """(n, residue) of the hostile batches: every residue of n_bytes mod 16, n cycling through 1, 255, 256 and 257."""
    return [((1, 255, 256, 257)[r % 4], r) for r in range(16)]


# --------------------------------------------------------------------------- the golden decoder vectors


def golden():
    with open(os.path.join(HERE, "golden", "wire", "messages.json")) as f:
        return json.load(f)["vectors"]


def retarget(vector, msg_type):
    """A messages.json vector as a message of type msg_type: an accepted one gets 0x08 <type> appended (field 1 is a
    scalar, so the last value wins and every other field keeps python-protobuf's verdict), a rejected one stays as it
    is -> (Message bytes, its fields with msg_type replaced, or None for a rejected vector)."""
    raw = bytes.fromhex(vector["hex"])
    if not vector["ok"]:
        return raw, None
    return raw + bytes([0x08, msg_type]), dict(vector["fields"], msg_type=msg_type)


# --------------------------------------------------------------------------- the five passes
# Each pass: frames(rng) builds its scenario's frames on the CPU; fresh() an arena and the oracle's state in the same
# state; run() one batch through the arena (host or device form) and the oracle, compares every output and returns the
# outputs, the status bytes (WIRE_* << 4 | low nibble) first; PER_FRAME names the outputs with one row per frame;
# check() compares the arena with the oracle's state.

P = 8
U64_MAX = (1 << 64) - 1


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
        blob, off = R.mixed_batch(rng, self.d, self.n, self.terms, True, k or self.n)
        return PF.split(blob, off)

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
        if self.kind == "append":
            if device:
                got, = PF.device(a, "wire_apply", buf, off, n_bytes=n_bytes)
                want = oracle_wire_apply(d.c, buf, off, self.n, self.terms, n_bytes=n_bytes)
            else:
                fb = PF.host_batch(buf, off, n_bytes)
                fb.records = None
                a.step_begin_wire(fb, B.STEP_READ_COMMITTED)
                sr = a.step_wait()
                got = a.wire_status().copy()
                want, bm, adv, _ = oracle_wire_step(d.c, fb, self.n, self.terms)
                gbm, _ = a.step_results(self.n)
                assert np.array_equal(gbm, bm[: len(gbm)]) and sr.n_advanced == adv, what
            PF.equal([want], [got], ["status"], what)
            return (got,)
        st, rel = PF.run(a, "heartbeat_wire", buf, off, device=device, n_bytes=n_bytes)
        want, want_rel = H.apply(d.c, d.q, buf, off, self.terms, n_bytes=n_bytes)
        got = (st, R.by_group(rel))
        PF.equal([want, R.by_group(want_rel)], got, ["status", "released reads"], what)
        return got

    def check(self, a, d, what):
        assert_columns_equal(a.read_columns(self.n), d.c, self.n, what)
        R.queues_equal(a, d.q, self.n, what)


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
            got = PF.device(a, "follower_heartbeat", buf, off, self.sel, self.ids, n_bytes=n_bytes)
        else:
            ids, sel = np.zeros(a.cap, np.uint64), np.zeros((a.cap + 31) // 32, np.uint32)
            ids[: self.n], sel[: len(self.sel)] = self.ids, self.sel
            got = a.follower_heartbeat(PF.host_batch(buf, off, n_bytes), ids, sel)
        PF.equal(want, got, ("status", "from", "response bytes", "response offsets", "totals"), what)
        return got

    def check(self, a, c, what):
        s = FL.group_state(a, self.n)
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
        out = PF.split(FL.with_headers(hb, hoff, hdr), hoff)
        out += [out[i] for i in rng.integers(0, len(out), len(out) // 10)]         # repeated heartbeats: DUP
        return [out[i] for i in rng.permutation(len(out))]

    return Followers(n, cols, FL.bitmap(rng.random(n) < 0.95), FL.self_ids(rng, n), frames)


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
        return arena_of(self.e), V.state_of(self.e)

    def run(self, a, state, buf, n_bytes, off, device, what):
        c, vt = state
        want_st, want_out, _ = VW.batch(c, vt, buf, off, self.sel, self.pre, n_bytes=n_bytes)
        got = PF.device(a, "vote_wire", buf, off, self.sel, self.pre, n_bytes=n_bytes) if device else \
            a.vote_wire(PF.host_batch(buf, off, n_bytes), self.sel, self.pre)
        PF.equal([want_st, want_out], got, ("status", "outcomes"), what)
        return got

    def check(self, a, state, what):
        assert np.array_equal(votes(a, self.n), state[1][:, : self.n]), what


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
        return arena_of(self.s), Q.state_of(self.s)

    def run(self, a, state, buf, n_bytes, off, device, what):
        c, vt = state
        want = VR.batch(c, None, vt, buf, off, self.s.table, n_bytes=n_bytes)
        got = PF.device(a, "vote_request_wire", buf, off, self.s.table, n_bytes=n_bytes) if device else \
            a.vote_request_wire(PF.host_batch(buf, off, n_bytes), self.s.table)
        PF.equal(want, got, ("status", "out", "response bytes", "response offsets", "totals"), what)
        return got

    def check(self, a, state, what):
        check_columns(a, *state, self.n)


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
    """The scenario's frames with the ballast of across_the_stage -> (frames, ballast mask)."""
    rng = np.random.default_rng(seed)
    return across_the_stage(sc.frames(rng), rng)


def hostile_batches(sc, seed, device):
    """hostile over the scenario's frames for every case of hostile_cases -> [(buf, n_bytes, offsets)]: a device
    buffer holds 4 KiB or more of valid frames past n_bytes, and only offsets that end on those frames' boundaries go past
    n_bytes; a host batch's offsets go at most 4 (n + 1) bytes past n_bytes, into the offsets the same call copies in."""
    rng = np.random.default_rng(seed)
    frames = sc.frames(rng)
    tail, bounds = slack(frames[::-1])
    out = []
    for n, r in hostile_cases():
        past = bounds if device else np.arange(4 * (n + 1) + 1)
        blob, off = hostile(frames[int(rng.integers(0, len(frames) - n - 1)):], rng, n, r, past)
        buf = np.concatenate([blob, np.frombuffer(tail, np.uint8)]) if device else blob
        out.append((buf, len(blob), off))
    return out


GOLDEN_TYPE = {"append": 4, "heartbeat": 9, "follower": 8, "vote": 6, "voter": 5}


CAP = 1 << 62                                            # log positions stay below this (SET_CONF takes last + 1)


def golden_scenario(name, variant):
    """One group per messages.json vector (retarget to the pass's type; a rejected vector as it is), its state
    derived from the vector's decoded fields so that most frames reach the pass's decision:
      append, heartbeat: a leader of voters {0, 1, 2} at m.term, a read pending under an 8-byte context;
      follower: a selected follower at m.term whose log reaches m.commit, self id g + 1;
      vote: a candidate at m.term whose committed is m.commit (variant 0) or one below it (variant 1: a rejection with
        commit_term is COMMIT_VOTE);
      voter: a selected follower at m.term with last_index = m.index and last_term = m.log_term (up to date), whose
        priority is m.priority (variant 0: granted) or one more (variant 1: rejected, committed one below m.commit).
    -> (scenario, frames, the vectors' kinds, their python-protobuf verdicts)."""
    vs = golden()
    n = len(vs)
    typ = GOLDEN_TYPE[name]
    raws, fields = zip(*[retarget(v, typ) for v in vs])
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
