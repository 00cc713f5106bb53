"""Followers with earlier term runs for the follower-runs tests (DESIGN 3.22, oracle/follower_runs_oracle.c): literal
logs of several term runs, the table and the rows they imply (at 0, 1 or 2 stated runs, some compacted or stale), and
MsgAppend frames that match in, reject from and truncate into every stated segment."""
import numpy as np

from helpers import B
from oracle import app_follow_oracle as AL
from oracle import follower_runs_oracle as FR
import app_follow as A


def random_log(rng, n_runs, max_len=6, log_cap=64):
    """A literal log of n_runs term runs (terms strictly increasing), entry 0 the dummy: u64[log_cap], last index."""
    terms = np.zeros(log_cap, np.uint64)
    at, t = 1, 0
    for _ in range(n_runs):
        t += int(rng.integers(1, 4))
        k = int(rng.integers(1, max_len + 1))
        terms[at:at + k] = t
        at += k
    return terms, at - 1


class Followers:
    """n followers with literal logs (the literal oracle's groups and terms), and the table and rows they state."""

    def __init__(self, rng, n, log_cap=64, max_runs=6):
        self.n, self.log_cap = n, log_cap
        self.groups = np.zeros(n, AL.GROUP_DTYPE)
        self.terms = np.zeros((n, log_cap), np.uint64)
        last = np.zeros(n, np.int64)
        for g in range(n):
            self.terms[g], last[g] = random_log(rng, int(rng.integers(1, max_runs + 1)), log_cap=log_cap)
        self.groups["last_index"] = last
        self.groups["term"] = self.terms[np.arange(n), last] + rng.integers(0, 3, n).astype(np.uint64)
        self.groups["committed"] = [int(rng.integers(0, max(1, A.run_of(self.terms[g], int(last[g]))[0]))) // 2
                                    for g in range(n)]
        self.groups["id"] = rng.integers(1, 1 << 63, n, dtype=np.uint64)
        self.groups["flags"] = AL.FOLLOWER

    def last(self, g):
        return int(self.groups["last_index"][g])

    def segments(self, g, first_index=1):
        return FR.segments(self.terms[g, :self.last(g) + 1], first_index)

    def columns(self):
        c = A.O.new_columns(self.n + 8, self.n)
        c.term_start[:] = A.NO_TERM_START
        for k in ("committed", "last_index", "term"):
            getattr(c, k)[: self.n] = self.groups[k]
        return c

    def state(self, n_runs, first_index=None, rng=None, stale=0.0):
        """(table, rows): the table states each log's last run, the row up to n_runs runs below it (each at or above
        first_index[g] - 1); with rng a fraction `stale` of the rows is anchored elsewhere (another start or term)."""
        table = np.zeros(self.n, AL.LOG_DTYPE)
        table["id"], table["flags"] = self.groups["id"], AL.SELECT
        rows = FR.rows_for(self.n)
        for g in range(self.n):
            segs = self.segments(g, 1 if first_index is None else min(int(first_index[g]), self.last(g)))
            s, t = segs[0]
            table["run_start"][g], table["run_term"][g] = s, t
            runs = segs[1:1 + n_runs]
            rows[g] = FR.row(g, s, t, runs)
            if rng is not None and rng.random() < stale:
                if rng.random() < 0.5:
                    rows["anchor_start"][g] = s + 1 if s + 1 <= self.last(g) else max(1, s - 1)
                else:
                    rows["anchor_term"][g] = t + 1
        return table, rows


def term_at(terms, last, i):
    return 0 if i > last else int(terms[i])


def probe(rng, f, g, kind=None):
    """One MsgAppend body for follower g at its term: 'match' (entry-less, in a random segment), 'reject' (random index
    and log_term), 'append' (matching in a random segment, then entries that keep some of the log and bring 1-3 new
    terms)."""
    last, terms, term = f.last(g), f.terms[g], int(f.groups["term"][g])
    kind = kind or rng.choice(["match", "reject", "append", "append"])
    committed = int(f.groups["committed"][g])
    frm = int(rng.integers(1, 1 << 40))
    if kind == "reject":
        index = int(rng.integers(committed, last + 3))
        return A.message(3, term=term, log_term=int(rng.integers(0, term + 1)), index=index,
                         commit=int(rng.integers(0, index + 1)), frm=frm)
    segs = f.segments(g)
    k = int(rng.integers(0, len(segs)))
    lo, hi = max(segs[k][0], committed), last if k == 0 else segs[k - 1][0] - 1
    index = min(int(rng.integers(lo, hi + 1)) if lo <= hi else lo, last)
    lt = term_at(terms, last, index)
    if kind == "match":
        return A.message(3, term=term, log_term=lt, index=index, commit=int(rng.integers(0, index + 1)), frm=frm)
    n = int(rng.integers(1, 9))
    keep = int(rng.integers(0, min(n, last - index) + 1))
    ents = [(term_at(terms, last, index + 1 + k), index + 1 + k) for k in range(keep)]
    floor = ents[-1][0] if ents else lt
    new_terms = sorted(int(x) for x in rng.integers(max(floor, 1), term + 1, int(rng.integers(1, 4))))
    per = np.sort(rng.integers(0, len(new_terms), n - keep)) if n > keep else []
    ents += [(new_terms[int(p)], index + 1 + keep + k) for k, p in enumerate(per)]
    return A.message(3, term=term, log_term=lt, index=index, commit=int(rng.integers(0, index + n + 1)), frm=frm,
                     entries=ents)


def responses_by_frame(status, blob, roff):
    """{frame: response bytes} of the frames a batch answered (status low nibble RES_OK)."""
    out, k = {}, 0
    for i, st in enumerate(np.asarray(status).tolist()):
        if st >> 4 == 0 and st & 1:
            out[i] = bytes(blob[roff[k]:roff[k + 1]])
            k += 1
    return out


def literal_by_frame(outcome, blob, roff):
    out, k = {}, 0
    for i, o in enumerate(np.asarray(outcome).tolist()):
        if o == AL.ANSWERED:
            out[i] = bytes(blob[roff[k]:roff[k + 1]])
            k += 1
    return out


def truncate(rng, f, table, frac):
    """A fraction frac of the followers whose table run starts above 1 lose their log from a random index below the run
    on (the host truncated it without restating the table or the row): the table's run is then empty and the row
    stays anchored to it.  Changes f's literal logs in place; returns those groups."""
    rs = table["run_start"][: f.n].astype(np.int64)
    cut = np.flatnonzero((rs > 1) & (rng.random(f.n) < frac))
    for g in cut.tolist():
        last = int(rng.integers(max(1, int(rs[g]) - 3), int(rs[g])))
        f.terms[g, last + 1:] = 0
        f.groups["last_index"][g] = last
        f.groups["committed"][g] = min(int(f.groups["committed"][g]), last)
    return cut


# ----------------------------------------------------------------------------- the election dialogue at both ends

def follower_of(rng, leader, ts):
    """A follower of a leader whose log is `leader` (terms, entry 0 first; become_leader's entry at ts): it holds the
    leader's log up to an index inside the leader's last or second-last earlier term run (at least one entry of that
    run), then, half of the time, a divergent tail at a term the leader never had."""
    starts = [i for i in range(1, ts) if leader[i] != leader[i - 1]]
    k = int(rng.integers(max(0, len(starts) - 2), len(starts)))
    end = starts[k + 1] - 1 if k + 1 < len(starts) else ts - 1
    out = list(leader[: int(rng.integers(starts[k], end + 1)) + 1])
    if rng.random() < 0.6:
        free = [t for t in range(out[-1] + 1, leader[ts]) if t not in set(leader)]
        if free:
            out += [int(rng.choice(free))] * int(rng.integers(1, 5))
    return out


class Dialogue:
    """A store-wide election on n groups x `peers` slots: each leader (slot 0, its last two earlier runs stated) probes
    its followers (slots 1..peers - 1, each slot a follower arena whose rows state two runs below the table's run when
    follower_runs is set) until every follower's log is its leader's.  Each round: the probes of the cells not done go
    through the entries pass; its NEEDS_LOG frames are stepped on the host from the literal logs (which also step every
    decided frame and must answer it byte for byte as the pass did), and those followers' table rows and rows are
    restated; every response goes to the leader as one wire batch, whose NEEDS_LOG frames the host resolves from the
    leader's literal log as REJECT + EXT records.  The oracles (oracle/follower_runs_oracle.c, leader_runs_oracle.c) run
    every round; with `device` = (leader arena factory, follower arena factory) the arenas run alongside and must equal
    them.  host_follower / host_leader count the frames the host resolved."""

    def __init__(self, rng, n, follower_runs, peers=5, device=None):
        from oracle import leader_runs_oracle as LR
        import append_reject as R
        self.LR, self.R = LR, R
        self.n, self.P, self.runs, self.dev = n, peers, follower_runs, device is not None
        self.leaders = []
        for _ in range(n):
            t = R.random_log(rng, int(rng.integers(2, 7)))
            self.leaders.append(t + [t[-1] + int(rng.integers(1, 4))])
        self.term = np.array([t[-1] for t in self.leaders], np.uint64)
        self.ts = np.array([len(t) - 1 for t in self.leaders], np.int64)
        c = A.O.new_columns(n, n)
        c.term[:n], c.term_start[:n], c.last_index[:n] = self.term, self.ts, self.ts
        c.meta[:n] = A.O.make_meta((1 << peers) - 1, self_slot=0)
        c.next_idx[:, :n] = self.ts
        c.matched[0, :n] = self.ts
        self.ref = c
        self.lrows = R.rows_for(self.leaders, np.ones(n), 2)
        self.ids = rng.integers(1, 1 << 40, (peers, n), dtype=np.uint64)
        self.slots = []
        for sl in range(1, peers):
            f = Followers.__new__(Followers)
            f.n, f.log_cap = n, 64
            f.terms = np.zeros((n, 64), np.uint64)
            f.groups = np.zeros(n, AL.GROUP_DTYPE)
            for g in range(n):
                lg = follower_of(rng, self.leaders[g], int(self.ts[g]))
                f.terms[g, : len(lg)] = lg
                f.groups["last_index"][g] = len(lg) - 1
            f.groups["term"], f.groups["id"], f.groups["flags"] = self.term, self.ids[sl], AL.FOLLOWER
            table, rows = f.state(2)
            self.slots.append({"f": f, "c": f.columns(), "table": table, "rows": rows if follower_runs else None})
        self.host_follower = self.host_leader = self.rounds = 0
        if device:
            make_leader, make_follower = device
            self.la = make_leader(c, n, self.lrows)
            for s in self.slots:
                s["a"] = make_follower(s["c"], n, follower_runs, s["rows"])
                s["dtable"] = A.full_table(s["a"], s["table"])

    def done(self, s, g):
        f, ts = s["f"], int(self.ts[g])
        return f.last(g) == ts and list(f.terms[g, : ts + 1]) == self.leaders[g]

    def round(self, PF):
        LR, R, O, n = self.LR, self.R, A.O, self.n
        resp = []
        for sl, s in enumerate(self.slots, start=1):
            f = s["f"]
            cells = [g for g in range(n) if not self.done(s, g)]
            if not cells:
                continue
            probes = []
            for g in cells:
                i = int(self.ref.next_idx[sl, g]) - 1
                ld = self.leaders[g]
                probes.append(A.frame(g, sl, A.message(3, term=int(self.term[g]), log_term=ld[i], index=i,
                                                       frm=int(self.ids[0, g]), to=int(self.ids[sl, g]),
                                                       entries=[(ld[j], j) for j in range(i + 1, int(self.ts[g]) + 1)])))
            blob, off = A.batch(probes)
            want = FR.batch(s["c"], None, s["table"], s["rows"], blob, off, True)
            if self.dev:
                got = PF.run(s["a"], "follower_append_entries", blob, off, s["dtable"], device=False)
                PF.equal(want, tuple(got[:2]) + (got[2].view(want[2].dtype),) + tuple(got[3:]),
                         ("status", "from", "appended", "response bytes", "response offsets", "totals"), ("slot", sl))
            groups, terms = f.groups, f.terms
            outcome, lb, lo, _ = AL.literal(groups, terms, blob, off)
            assert (outcome == AL.ANSWERED).all()
            mine, lit = responses_by_frame(want[0], want[3], want[4]), literal_by_frame(outcome, lb, lo)
            st = want[0] >> 4
            assert set(np.unique(st).tolist()) <= {B.WIRE_OK, B.WIRE_NEEDS_LOG}
            restate = []
            for k, g in enumerate(cells):
                if st[k] == B.WIRE_OK:
                    assert mine[k] == lit[k] and int(s["c"].last_index[g]) == f.last(g)
                    assert FR.stated_ok(terms[g], s["table"][g], s["rows"][g] if self.runs else None, f.last(g))
                else:
                    restate.append(g)
            self.host_follower += len(restate)
            for g in restate:  # the host stepped the frame: its log moved, the table's row and the row are stated again
                segs = f.segments(g)
                s["table"]["run_start"][g], s["table"]["run_term"][g] = segs[0]
                s["c"].last_index[g] = f.last(g)
                if self.runs:
                    s["rows"][g] = FR.row(g, segs[0][0], segs[0][1], segs[1:3])
            if self.dev:
                s["a"].column_write(B.COL_LAST_INDEX, 0, 0, s["c"].last_index[:n].copy())
                s["dtable"][:n] = s["table"]
                if self.runs:
                    if restate:
                        assert not s["a"].follower_runs_set(s["rows"][restate]).any()
                    assert np.array_equal(s["a"].follower_runs_get(0, n), s["rows"])
            resp += [bytes(lb[a:b]) for a, b in zip(lo[:-1].tolist(), lo[1:].tolist())]
        if not resp:
            return False
        blob, off = A.batch(resp)
        want = R.oracle_step(self.ref, self.lrows, blob, off)
        O.arena_recompute(self.ref)
        undecided = np.flatnonzero((want >> 4) == B.WIRE_NEEDS_LOG).tolist()
        self.host_leader += len(undecided)
        lst, lrecs, lhint, lsnap = LR.literal_batch(self.leaders, np.ones(n), self.term, blob, off)
        recs = []
        for i in undecided:
            recs.append(tuple(lrecs[i]))
            recs.append((lrecs["group"][i], lrecs["peer_slot"][i], B.REC_EXT, 0, lhint[i], lsnap[i]))
        recs = np.array(recs, B.APPEND_RESP_DTYPE) if recs else np.zeros(0, B.APPEND_RESP_DTYPE)
        if len(recs):
            O.arena_apply(self.ref, recs, mode=0)
        if self.dev:
            self.la.step_begin_wire(PF.host_batch(blob, off, len(blob)), B.STEP_READ_COMMITTED)
            self.la.step_wait()
            assert np.array_equal(self.la.wire_status(), want)
            if len(recs):
                rb = PF.host_batch(np.zeros(0, np.uint8), np.zeros(1, np.uint32), 0)
                rb.records, rb.n_records = recs, len(recs)
                self.la.step_begin_wire(rb, B.STEP_READ_COMMITTED)
                self.la.step_wait()
            lc = self.la.read_columns(n)
            assert np.array_equal(lc.next_idx[:, :n], self.ref.next_idx[:, :n])
            assert np.array_equal(lc.matched[:, :n], self.ref.matched[:, :n])
        self.rounds += 1
        return True

    def run(self, PF, max_rounds=16):
        while self.round(PF):
            assert self.rounds <= max_rounds
        for sl, s in enumerate(self.slots, start=1):
            assert all(self.done(s, g) for g in range(self.n))
            assert (self.ref.matched[sl, : self.n] == self.ts).all()
