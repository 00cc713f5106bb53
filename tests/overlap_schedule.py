"""Schedules of overlapped ticks: steps kept in flight while the other calls of a tick run, and the sequential model
they are checked against.  Pure Python over the oracles; tests/test_gpu_overlap.py replays them on an arena.

A schedule is a list of events: begin(form, batch), wait(), call(kind, args).  The model applies them to the oracle in
submission order: a begin takes effect on the columns when it is submitted, and its outcome (advanced count, bitmap,
committed of the advanced groups, result bytes) is recorded then and reported at its wait; a call takes effect when it
is made.  Every batch and frame list is built from the oracle's state at its place in the schedule, and the calls aim
on purpose at the groups the steps still in flight advanced."""
from dataclasses import dataclass, field

import numpy as np

from oracle import oracle as O
from oracle import read_oracle as RO
from oracle import hb_wire_oracle as HW
from oracle import hb_frames_oracle as HF
from oracle import hb_follow_oracle as HL
from oracle import vote_wire_oracle as VW
from oracle import vote_request_oracle as VR
from helpers import B, Shape, bitmap_to_bool, is_simple5, random_batch, random_state
from control_cmds import NO_TERM_START, META_WIDE_LO, META_WIDE_HI, cmds
import hb_frames as F
import read_cases as R
import vote_frames as V
import vote_request_frames as Q

P = 8                     # read queue depth of every arena
INS_CAP = 4               # Inflights window of the inflights shape
RC, RR = B.STEP_READ_COMMITTED, B.STEP_READ_RESULTS

# the step forms: the records API on a group-sorted batch (the fused compact kernel, or bulk staging with Inflights)
# and on a shuffled one (the scatter kernel and the recompute pass), RAW and HYBRID from host_alloc memory, the packed
# and compact zero-copy forms, the wire form, and enqueue_append_resp + step_begin
FORMS = ("records_sorted", "records_shuffled", "raw", "hybrid", "packed", "compact", "wire", "ring")
ZERO_COPY = ("packed", "compact")                     # these report slot results (READ_RESULTS)
ONE_PER_CELL = ("raw", "hybrid", "packed", "compact", "wire")
CALLS = ("commit_to", "set_conf", "control", "heartbeat_resp", "update_state", "read_index_request", "read_index_ack",
         "read_index_recheck", "heartbeat_wire", "heartbeat_frames", "follower_heartbeat", "vote_wire",
         "vote_request_wire", "step_send_list", "step_results", "slot_results", "column_read", "counters_read",
         "read_index_get", "read_index_read")
# where a call is made: with 0, 1 or 2 steps in flight, or right after a wait that left one in flight
POINTS = ("0", "1", "2", "1w")

# (name, arena shape, groups, seed, rounds, fraction of a window's groups a batch draws from, groups in the window).
# A batch draws from one window of consecutive groups, dense enough that the group-ordered forms tile (a unit block
# of the compact stream spans at most 4095 groups); the window moves from batch to batch.  The plain schedules run
# eight rounds or more, so that every form begins once on each launch plan (schedule()).
SCHEDULES = (
    ("plain_32k", "plain", 32_768, 0x0E1, 8, 0.5, 32_768),
    ("random_24k", "random", 24_000, 0x0E2, 4, 0.5, 24_000),
    ("inflights_8k", "inflights", 8_192, 0x0E3, 4, 0.5, 8_192),
    ("plain_1m", "plain", 1 << 20, 0x0E4, 12, 0.5, 1 << 17),
)


def side_len(n):
    """Length of the caller's per-group tables (ids, select words, voter rows): past any arena's capacity for n groups."""
    return (n + 64 + 1023) // 1024 * 1024 + 1024


class World:
    """The oracle's copy of an arena (columns, votes, read queues, Inflights) and the recipe that builds the arena:
    plain: every group the plain 5-voter configuration (the kSimple5 kernels); random: R.random_setup's narrow groups,
    wide pairs, leaders and followers, group commit; inflights: any configuration, Inflights windows of INS_CAP."""

    def __init__(self, shape, n, seed):
        rng = np.random.default_rng(seed)
        self.shape, self.n, self.rng = shape, n, rng
        self.inflights = shape == "inflights"
        self.n_wide = max(1, n // 100) if shape == "random" else 0
        self.n_narrow = n - 2 * self.n_wide
        c = O.new_columns(n + 64, n)
        self.init = self.setup = None
        if shape == "random":
            c.term_start[:] = NO_TERM_START
            for k in range(self.n_wide):
                lo = self.n_narrow + 2 * k
                c.meta[lo], c.meta[lo + 1] = META_WIDE_LO, META_WIDE_HI
            lows = list(range(self.n_narrow)) + list(range(self.n_narrow, n, 2))
            gc = rng.choice(self.n_narrow, self.n_narrow // 20, replace=False)
            self.setup = np.concatenate([R.random_setup(rng, self.n_narrow, self.n_wide),
                                         cmds(*[(B.CTL_SET_GROUP_COMMIT, int(g), 0, 1) for g in gc]),
                                         cmds(*[(B.CTL_SET_TERM, g, 0, 0, (int(rng.integers(1, 50)),)) for g in lows])])
        else:
            shp = Shape(((0x1F, 0, 0xE0),)) if shape == "plain" else Shape(None, group_commit=True)
            init = random_state(n, shp, rng)
            if self.inflights:
                init.pflags &= np.uint8(~O.PF_INS_FULL & 0xFF)       # the windows decide fullness
            for name in list(B.COLUMNS) + ["term"]:
                getattr(c, name)[..., :n] = getattr(init, name)
            self.init = init
        if self.inflights:
            O.enable_inflights(c, INS_CAP)
        self.c = c
        self.votes = np.zeros((O.SLOTS, c.cap), np.uint8)
        self.q = RO.ReadQueues(c.cap, P)
        self.q.allocated[:n] = 1
        self.hi_half = (c.meta[:n] & META_WIDE_HI) != 0 if self.n_wide else np.zeros(n, bool)
        self.setup_want = self.q.control(c, self.votes, self.setup) if self.setup is not None else None

    def plan(self):
        """The launch plan the meta column implies: True while every group is the plain 5-voter configuration."""
        return bool(np.all(is_simple5(self.c.meta[: self.n])))


@dataclass
class Outcome:
    """What a step reports at its wait, recorded when it was submitted."""
    form: str
    flags: int
    n_advanced: int
    bitmap: np.ndarray
    committed: np.ndarray        # committed of every group right after the step
    results: np.ndarray          # result byte of every record of the batch (oracle order)
    advanced: np.ndarray = field(default=None)

    def __post_init__(self):
        self.advanced = bitmap_to_bool(self.bitmap, len(self.committed))


@dataclass
class Event:
    op: str                      # begin | wait | call
    name: str                    # the form, "wait", or the call kind
    point: str                   # POINTS: steps in flight when it is made
    args: dict
    want: object
    info: dict = field(default_factory=dict)


class Model:
    """The sequential model: every event applied to the World in submission order."""

    def __init__(self, w: World, frac: float, window: int | None = None):
        self.w, self.frac = w, frac     # frac: the fraction of a window's groups a batch draws from
        self.window = w.n if window is None else min(window, w.n)
        self.rng = w.rng
        self.pending = []        # outcomes of the steps in flight, oldest first
        self.last = None         # outcome of the last completed step while the arena still holds it
        self.after_wait = False
        self.totals = {"advanced": 0, "recomputes": 0, "votes_tallied": 0}
        self.conf_six = []       # groups a set_conf gave a sixth voter, restored by the next one
        self.want_six = False    # the plan the next set_conf leaves: conf_six held (True) or empty (False)

    # ---------------------------------------------------------------- helpers
    def point(self):
        k = len(self.pending)
        return "1w" if k == 1 and self.after_wait else str(k)

    def hot(self, k, lows_only=True):
        """Up to k groups the newest step in flight advanced (else the last completed one), then random groups."""
        w, n = self.w, self.w.n
        src = self.pending[-1] if self.pending else self.last
        ok = ~w.hi_half if lows_only else np.ones(n, bool)
        g = np.flatnonzero(src.advanced & ok) if src is not None else np.zeros(0, np.int64)
        g = self.rng.permutation(g)[:k]
        if len(g) < k:
            extra = self.rng.choice(np.flatnonzero(ok), k - len(g), replace=False)
            g = np.concatenate([g, extra])
        return np.unique(g).astype(np.int64)

    def inflight_advanced(self):
        m = np.zeros(self.w.n, bool)
        for o in self.pending:
            m |= o.advanced
        return m

    # ---------------------------------------------------------------- steps
    def begin(self, form):
        w, c, rng = self.w, self.w.c, self.rng
        first = int(rng.integers(0, w.n - self.window + 1))
        if self.conf_six:         # (the window holds the groups with a sixth voter: they came from the last one)
            first = min(min(self.conf_six), w.n - self.window)
        keep = np.zeros(w.n, bool)
        keep[first:first + self.window] = rng.random(self.window) < self.frac
        if form in ONE_PER_CELL:
            recs = random_batch(c, rng, 1, keep=keep)
        else:   # a fifth of the groups get up to two records per cell (the later waves' staging holds cap / 4 records)
            two = keep & (rng.random(w.n) < 0.2)
            recs = np.concatenate([random_batch(c, rng, 1, keep=keep & ~two), random_batch(c, rng, 2, keep=two)])
            recs = np.ascontiguousarray(recs[np.argsort(recs["group"], kind="stable")])
        if self.conf_six:         # the groups with a sixth voter: three of their six voters reach last_index
            six = np.asarray(self.conf_six)
            rows = []
            for g in six.tolist():
                meta = int(c.meta[g])
                me = (meta >> 24) & 7 if meta & O.META_HAS_SELF else -1
                rows += [(g, s, B.REC_LOCAL if s == me else 0, 0, int(c.last_index[g]), 0) for s in (0, 1, 2)]
            recs = recs[~np.isin(recs["group"], six)]
            recs = np.concatenate([recs, np.array(rows, dtype=B.APPEND_RESP_DTYPE)])
            recs = np.ascontiguousarray(recs[np.argsort(recs["group"], kind="stable")])
        if form == "records_shuffled":                 # groups in a random order, each group's records kept in order
            starts = np.flatnonzero(np.r_[True, recs["group"][1:] != recs["group"][:-1]])
            ends = np.r_[starts[1:], len(recs)]
            order = rng.permutation(len(starts))
            recs = np.ascontiguousarray(np.concatenate([recs[starts[i]:ends[i]] for i in order]))
        flags = RC | (RR if form in ZERO_COPY else 0)
        point = self.point()
        res = O.arena_apply(c, recs, mode=0)
        adv, bm, _, _ = O.arena_recompute(c)
        o = Outcome(form, flags, int(adv), bm[: (w.n + 31) // 32].copy(), c.committed[: w.n].copy(), res)
        self.pending.append(o)
        if len(self.pending) == 2:
            self.last = None       # the third staging set is the one that held it
        self.after_wait = False
        self.totals["advanced"] += int(adv)
        self.totals["recomputes"] += w.n - w.n_wide      # a wide pair is recomputed once
        return Event("begin", form, point, {"recs": recs, "flags": flags, "term": c.term.copy()}, o,
                     {"plan": w.plan()})

    def wait(self):
        point = self.point()
        o = self.pending.pop(0)
        self.last = o
        self.after_wait = True
        return Event("wait", "wait", point, {"totals": dict(self.totals)}, o)

    # ---------------------------------------------------------------- calls
    def call(self, kind):
        w, c, rng, n = self.w, self.w.c, self.rng, self.w.n
        point = self.point()
        adv_inflight = self.inflight_advanced()
        before = c.committed[:n].copy()
        plan_before = w.plan()
        args, want = getattr(self, "_" + kind)(w, c, rng, n)
        changed = c.committed[:n] != before
        info = {"commit_hits": int(np.count_nonzero(changed & adv_inflight)), "plan_changed": plan_before != w.plan()}
        return Event("call", kind, point, args, want, info)

    def _control_list(self, lst):
        res = self.w.q.control(self.w.c, self.w.votes, lst)
        self.totals["votes_tallied"] += int(np.count_nonzero((lst["op"] == B.CTL_VOTE_RESULT) & (res["status"] == B.OK)))
        return res

    def _conf_rows(self, gs, c, keep=False):
        """SET_CONF rows: the plain voters {0..4} get a sixth one (slot 5), or the groups given one get it back; with
        keep, every group's own configuration again."""
        rows = []
        for g in gs:
            meta = int(c.meta[g])
            inc = meta & 0xFF if keep else 0x1F if (meta & 0xFF) == 0x3F else 0x3F
            out = (meta >> 8) & 0xFF if keep else 0
            learn = (meta >> 16) & 0xFF & ~(inc | out)
            s = (meta >> 24) & 7 if meta & O.META_HAS_SELF and ((inc | out | learn) >> ((meta >> 24) & 7)) & 1 \
                else B.CTL_NO_SELF
            rows.append((B.CTL_SET_CONF, int(g), s, 0, (inc, out, learn, int(c.last_index[g]) + 1)))
        return rows

    def _narrow(self, gs):
        return [int(g) for g in gs if g < self.w.n_narrow]

    def _commit_to(self, w, c, rng, n):
        gs = self.hot(8)
        to = [int(min(c.last_index[g], c.committed[g] + int(rng.integers(0, 4)))) for g in gs]
        st = [int(self._control_list(cmds((B.CTL_COMMIT_TO, int(g), 0, 0, (t,))))["status"][0]) for g, t in zip(gs, to)]
        return {"groups": gs.tolist(), "to": to}, st

    def _set_conf(self, w, c, rng, n):
        """SET_CONF rows that leave the plan want_six asks for: a sixth voter for 24 groups the steps advanced, or back
        to five voters for the groups that have one; when the plan is already right, the groups' own configuration
        again.  Only this single-group call changes the plan of the plain shape, so the plan at every begin is the one
        its last set_conf left."""
        if self.want_six == bool(self.conf_six):
            rows = self._conf_rows([g for g in self._narrow(self.hot(8)) if g not in self.conf_six], c, keep=True)
        elif self.conf_six:
            rows, self.conf_six = self._conf_rows(self.conf_six, c), []
        else:
            self.conf_six = self._narrow(self.hot(24))
            rows = self._conf_rows(self.conf_six, c)
        st = [int(self._control_list(cmds(r))["status"][0]) for r in rows]
        return {"rows": rows}, st

    def _control(self, w, c, rng, n):
        rows = []
        gs = self.hot(6)
        for g in gs.tolist():
            top = int(c.last_index[g]) + 2
            rows += [(B.CTL_SET_LOG_BOUNDS, g, 0, 0, (int(c.term_start[g]), top)),
                     (B.CTL_COMMIT_TO, g, 0, 0, (min(top, int(c.committed[g]) + 1),)),
                     (B.CTL_RESET_VOTES, g), (B.CTL_RECORD_VOTE, g, 1, 1), (B.CTL_VOTE_RESULT, g)]
        # a sixth voter and back, in one list: the meta mirror follows the list's order
        six = [g for g in self._narrow(gs[:2]) if g not in self.conf_six]
        rows += self._conf_rows(six, c)
        rows += [(op, g, sl, arg, (0x1F,) + tuple(a[1:])) for op, g, sl, arg, a in self._conf_rows(six, c)]
        lst = cmds(*rows)
        return {"cmds": lst}, self._control_list(lst)

    def _heartbeat_resp(self, w, c, rng, n):
        gs = self.hot(64, lows_only=False)
        g = np.repeat(gs, 2)
        s = np.concatenate([rng.permutation(np.arange(1, 5))[:2] for _ in gs])
        recs = np.zeros(len(g), B.APPEND_RESP_DTYPE)
        recs["group"], recs["peer_slot"], recs["flags"] = g, s, B.REC_HEARTBEAT
        recs["commit"] = c.committed[g]
        return {"recs": recs}, O.arena_apply_heartbeat(c, recs)

    def _update_state(self, w, c, rng, n):
        bm = self.last.bitmap if self.last is not None else self.pending[-1].bitmap if self.pending else None
        if bm is None:
            bm = group_bitmap(self.hot(64), n)
        e = O.arena_send_list(c, bm)
        e = np.ascontiguousarray(e[rng.permutation(len(e))[:512]])
        e = e[np.lexsort((e["peer_slot"], e["group"]))].astype(B.SEND_ENTRY_DTYPE)
        e["next_idx"] = c.last_index[e["group"]] + rng.integers(0, 3, len(e)).astype(np.uint64)
        return {"entries": e}, O.arena_update_state(c, e)

    def _read_index_request(self, w, c, rng, n):
        gs = np.sort(np.concatenate([self.hot(200), rng.integers(0, n, 200)]))
        reqs = np.zeros(len(gs), B.READ_REQ_DTYPE)
        reqs["group"], reqs["ctx"] = gs, rng.integers(1, 12, len(gs))
        return {"reqs": reqs}, w.q.request(c, reqs)

    def _read_index_ack(self, w, c, rng, n):
        recs = R.random_acks(rng, w.q, c.meta, n, 1500, w.hi_half)
        return {"recs": np.ascontiguousarray(recs)}, w.q.ack_seq(c, recs)

    def _read_index_recheck(self, w, c, rng, n):
        gs = self.hot(64).astype(np.uint32)
        return {"groups": gs}, w.q.recheck(c, gs)

    def _pending_ctx(self, g):
        q = self.w.q
        k = int(q.count[g])
        return int(q.ctx[g, int(self.rng.integers(0, k))]) if k else int(self.rng.integers(1, 12))

    def _heartbeat_wire(self, w, c, rng, n):
        frames = []
        for g in self.hot(96).tolist():
            for s in rng.permutation(np.arange(1, 5))[:2].tolist():
                frames.append(F.frame(g, s, F.message(F.HEARTBEAT_RESPONSE, term=int(c.term[g]),
                                                      commit=int(c.committed[g]), context=F.ctx_bytes(self._pending_ctx(g)))))
        blob, off = F.batch(frames)
        return {"frames": frames}, HW.apply(c, w.q, blob, off, c.term)

    def _heartbeat_frames(self, w, c, rng, n):
        gs = self.hot(32, lows_only=False)
        first = int(max(0, min(gs.min() - 64, n - 2048)))
        k = min(2048, n - first)
        ids = rng.integers(1, 1 << 62, (O.SLOTS + 1, k), dtype=np.uint64)
        sel = np.zeros(side_len(n), bool)
        sel[gs] = True
        sel[first + np.flatnonzero(rng.random(k) < 0.3)] = True
        select = V.bitmap(sel)
        return {"first": first, "n": k, "ids": ids, "select": select}, HF.bcast_heartbeats(c, w.q, first, k, ids, select)

    def _follower_heartbeat(self, w, c, rng, n):
        gs = self.hot(64)
        frames = [F.frame(g, 0, F.message(8, term=int(c.term[g]), commit=int(min(c.last_index[g], c.committed[g] + 2)), frm=2))
                  for g in gs.tolist()]
        sel = np.zeros(side_len(n), bool)
        sel[gs] = True
        select, ids = V.bitmap(sel), np.arange(1, side_len(n) + 1, dtype=np.uint64)
        blob, off = F.batch(frames)
        return ({"frames": frames, "select": select, "ids": ids},
                HL.follower_heartbeats(c, w.q, blob, off, select, ids))

    def _vote_wire(self, w, c, rng, n):
        gs = self.hot(48)
        frames = []
        for g in gs.tolist():
            for s in range(1, 1 + int(rng.integers(1, 5))):
                frames.append(F.frame(g, s, V.message(V.VOTE_RESPONSE, term=int(c.term[g]), reject=bool(rng.random() < 0.3))))
        frames = [frames[i] for i in rng.permutation(len(frames))]
        sel = np.zeros(side_len(n), bool)
        sel[gs] = True
        select = V.bitmap(sel)
        blob, off = F.batch(frames)
        st, out, tallied = VW.batch(c, w.votes, blob, off, select)
        self.totals["votes_tallied"] += int(tallied)
        return {"frames": frames, "select": select}, (st, out)

    def _vote_request_wire(self, w, c, rng, n):
        gs = self.hot(48)
        table = np.zeros(side_len(n), B.VOTER_DTYPE)
        frames = []
        for g in gs.tolist():
            t = table[g]
            t["id"], t["flags"] = 7, B.VOTER_SELECT
            t["last_term"], t["persisted"] = int(c.term[g]), int(c.last_index[g])
            frames.append(F.frame(g, 0, Q.request(Q.VOTE, int(c.term[g]) + 1, int(c.term[g]), int(c.last_index[g]),
                                                  to=7, frm=int(rng.integers(1, 6)))))
        blob, off = F.batch(frames)
        return {"frames": frames, "table": table}, VR.batch(c, w.q, w.votes, blob, off, table)

    def _step_send_list(self, w, c, rng, n):
        return {}, None if self.last is None else O.arena_send_list(c, self.last.bitmap)

    def _step_results(self, w, c, rng, n):
        return {}, self.last

    def _slot_results(self, w, c, rng, n):
        return {}, self.last

    def _column_read(self, w, c, rng, n):
        return {}, (c.committed[:n].copy(), c.matched[1, :n].copy())

    def _counters_read(self, w, c, rng, n):
        return {}, dict(self.totals)

    def _read_index_get(self, w, c, rng, n):
        gs = self.hot(4)
        return {"groups": gs.tolist()}, [tuple(np.asarray(x).copy() for x in w.q.pending(int(g))) for g in gs]

    def _read_index_read(self, w, c, rng, n):
        first = int(max(0, min(self.hot(1)[0] - 512, n - 2048)))
        return {"first": first, "n": min(2048, n - first)}, queue_view(w.q, first, min(2048, n - first))


def group_bitmap(groups, n):
    bm = np.zeros((n + 31) // 32, np.uint32)
    for g in np.asarray(groups, dtype=np.int64).tolist():
        bm[g >> 5] |= np.uint32(1 << (g & 31))
    return bm


def queue_view(q, first, n):
    """(counts, ctx, index, acks) of queues [first, first + n), entries past the count zeroed (raftgpu_read_index_read)."""
    sl = slice(first, first + n)
    k = np.arange(q.max_pending)[None, :] < q.count[sl, None]
    return (q.count[sl].copy(), np.where(k, q.ctx[sl], 0).astype(np.uint64), np.where(k, q.index[sl], 0).astype(np.uint64),
            np.where(k, q.acks[sl], 0).astype(np.uint16))


def schedule(m: Model, rounds: int):
    """The events of one schedule on the model m, generated lazily (each built from the model's state at its place).  A
    round is calls, begin, calls, begin, calls, wait, calls, wait: every call kind at every point of POINTS, in a
    shuffled order; two forms per round, all of FORMS in four rounds.  The set_conf of the first block leaves the plain
    5-voter plan for the first begin of the round and the one of the second block gives 24 groups a sixth voter for
    the second begin (a plan change between two steps in flight); in the second half of the rounds the other way
    round, so that in eight rounds every form begins once on each plan."""
    rng = m.rng
    forms = list(FORMS)

    def calls():
        for kind in rng.permutation(CALLS).tolist():
            yield m.call(kind)

    for r in range(rounds):
        late = r >= rounds // 2
        m.want_six = late
        yield from calls()
        yield m.begin(forms[(2 * r) % len(forms)])
        m.want_six = not late
        yield from calls()
        yield m.begin(forms[(2 * r + 1) % len(forms)])
        yield from calls()
        yield m.wait()
        yield from calls()
        yield m.wait()
    yield from calls()
