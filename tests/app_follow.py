"""Followers for the MsgAppend-at-the-follower tests (raftgpu_follower_append, oracle/app_follow_oracle.c): literal logs
(a term per index, the dummy entry at 0), the run table derived from them -- the longest last-term run, or a shortened
one -- the arena columns they imply, MsgAppend frames built field by field, and which terms the reference's decision
reads."""
import numpy as np

from helpers import B, O
import pass_forms as PF
from oracle import app_follow_oracle as AL

U64 = (1 << 64) - 1
NO_TERM_START = U64


def varint(v: int) -> bytes:
    out = bytearray()
    while v >= 0x80:
        out.append((v & 0x7F) | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


def entry(term=0, index=0) -> bytes:
    return b"".join(varint(no << 3) + varint(v) for no, v in ((2, term), (3, index)) if v)


def message(msg_type=3, term=0, log_term=0, index=0, commit=0, frm=0, entries=None, to=1) -> bytes:
    """eraftpb.Message in field-number order, zero scalars omitted; entries: [(term, index)] (an Entry each, (0, 0) an
    empty one)."""
    out = b""
    for no, v in ((1, msg_type), (2, to), (3, frm), (4, term), (5, log_term), (6, index)):
        if v:
            out += varint(no << 3) + varint(v)
    for t, i in entries or ():
        e = entry(t, i)
        out += varint(7 << 3 | 2) + varint(len(e)) + e
    if commit:
        out += varint(8 << 3) + varint(commit)
    return out


def frame(group, x, body: bytes) -> bytes:
    return np.array([group << 4 | x], dtype="<u4").tobytes() + body


def batch(frames):
    blob = np.frombuffer(b"".join(frames), dtype=np.uint8).copy()
    offsets = np.concatenate([[0], np.cumsum([len(f) for f in frames])]).astype(np.uint32)
    return blob, offsets


def run_of(row, last):
    """The longest last-term run of a log: (run_start, run_term) with term(i) == run_term on [run_start, last]."""
    t = row[last]
    s = last
    while s > 0 and row[s - 1] == t:
        s -= 1
    return s, int(t)


class World:
    """n followers with literal logs (the literal oracle's groups and terms) and the arena / run table they imply."""

    def __init__(self, rng, n, log_cap=64, max_last=30):
        self.n, self.log_cap = n, log_cap
        self.groups = np.zeros(n, AL.GROUP_DTYPE)
        self.terms = np.zeros((n, log_cap), np.uint64)
        last = rng.integers(0, max_last + 1, n)
        for g in range(n):
            steps = rng.choice([0, 0, 0, 1, 2], int(last[g]))
            self.terms[g, 1:last[g] + 1] = 1 + np.cumsum(steps)
        self.groups["last_index"] = last
        self.groups["term"] = self.terms[np.arange(n), last] + rng.integers(0, 2, n).astype(np.uint64)
        self.groups["term"][self.groups["term"] == 0] = 1
        self.groups["committed"] = (last * rng.random(n)).astype(np.uint64)
        self.groups["id"] = rng.integers(1, 1 << 63, n, dtype=np.uint64)
        self.groups["flags"] = AL.FOLLOWER

    def copy(self):
        w = object.__new__(World)
        w.n, w.log_cap, w.groups, w.terms = self.n, self.log_cap, self.groups.copy(), self.terms.copy()
        return w

    def runs(self, rng=None, shorten=0.0):
        """(run_start, run_term) per group; with rng, a fraction `shorten` of the runs cut to a random suffix (an empty
        one included)."""
        out = [run_of(self.terms[g], int(self.groups["last_index"][g])) for g in range(self.n)]
        if rng is not None:
            for g in np.flatnonzero(rng.random(self.n) < shorten):
                s, t = out[g]
                out[g] = (int(rng.integers(s, int(self.groups["last_index"][g]) + 2)), t)
        return out

    def columns(self):
        c = O.new_columns(self.n + 8, self.n)
        c.term_start[:] = NO_TERM_START
        for k in ("committed", "last_index", "term"):
            getattr(c, k)[: self.n] = self.groups[k]
        return c

    def table(self, runs):
        t = np.zeros(self.n, AL.LOG_DTYPE)
        t["id"] = self.groups["id"]
        t["run_start"] = [s for s, _ in runs]
        t["run_term"] = [r for _, r in runs]
        t["flags"] = AL.SELECT
        return t


def reads_outside(row, last, committed, run_start, index, log_term) -> bool:
    """Whether handle_append_entries without entries reads a term the run does not state (term(i) is known above last
    and on [run_start, last])."""
    if index < committed:
        return False
    known = lambda i: i > last or run_start <= i <= last
    term = lambda i: 0 if i > last else int(row[i])
    if not known(index):
        return True
    if term(index) == log_term:
        return False
    h = min(index, last)
    while True:
        if not known(h):
            return True
        if term(h) <= log_term:
            return False
        h -= 1


def random_append(rng, w, g, entries_p=0.1, safe=False):
    """A MsgAppend to follower g at its term, near its log's end: matching, mismatching, stale, above the log.  safe: no
    frame the reference would panic on (commit <= index, entries that follow index)."""
    last, term = int(w.groups["last_index"][g]), int(w.groups["term"][g])
    index = int(rng.integers(0, last + 3))
    if index <= last and rng.random() < 0.6:
        log_term = int(w.terms[g, index])
    elif index > last and not safe and rng.random() < 0.5:
        log_term = 0                                                  # term(i) above last_index: a match
    else:
        log_term = int(rng.integers(1, term + 2))
    commit = int(rng.integers(0, index + 1)) if safe or rng.random() < 0.9 else int(rng.integers(0, last + 6))
    ents = None
    if rng.random() < entries_p:
        k = int(rng.integers(1 if safe else 0, 4))
        ents = [(int(rng.integers(min(max(log_term, 1), term), term + 1)), index + j + 1) for j in range(k)] or [(0, 0)]
    return message(3, term=term, log_term=log_term, index=index, commit=commit, frm=int(rng.integers(1, 1 << 40)),
                   entries=ents)


def split_responses(blob, offsets):
    """[(header, body)] of a response blob."""
    return [(int.from_bytes(bytes(blob[a:a + 4]), "little"), bytes(blob[a + 4:b]))
            for a, b in zip(np.asarray(offsets[:-1]).tolist(), np.asarray(offsets[1:]).tolist())]


def state(c, n):
    return {k: getattr(c, k)[:n].copy() for k in ("committed", "last_index", "term", "term_start", "meta")}


LOG_STATUS_OK = B.WIRE_OK << 4 | B.RES_OK


NAMES = ("status", "from", "response bytes", "response offsets", "totals")


def host_form(a, blob, off, table, n_bytes=None):
    """raftgpu_follower_append's host form over the batch, with the table extended to the arena's highest group."""
    return a.follower_append(PF.host_batch(blob, off, n_bytes), full_table(a, table))


def full_table(a, table):
    """table cut or zero-extended to the arena's highest group."""
    t = np.zeros(a.get_info().hi, AL.LOG_DTYPE)
    t[: min(len(t), len(table))] = table[: len(t)]
    return t


def follower_arena(n_narrow, n_wide, cols, reads=False, extra=64):
    """An arena of n_narrow groups then n_wide pairs, its group columns written from cols (name -> u64[n]) -> (arena, host
    columns with c.term, read queues or None)."""
    n = n_narrow + 2 * n_wide
    a = B.Arena(n + extra)
    if reads:
        a.enable_read_index(8)
    assert a.group_alloc_range(n_narrow) == 0
    for k in range(n_wide):
        assert a.group_alloc_wide() == n_narrow + 2 * k
    for col, arr in cols.items():
        a.column_write(col, 0, 0, np.ascontiguousarray(arr[:n], np.uint64))
    c = a.read_columns(n)
    c.term = a.column_read(B.COL_TERM, 0, 0, n, np.uint64)
    q = None
    if reads:
        from oracle import read_oracle as RO
        q = RO.ReadQueues(c.cap, 8)
        q.allocated[:n] = 1
    return a, c, q


def hostile(rng, terms, k):
    """k frames that must not pass or that go back to the host: garbage, unknown groups, truncations, other types,
    frames with entries, term 0, stale and future terms, a commit out of range."""
    out, n_f = [], len(terms)
    for j in range(k):
        g, x = int(rng.integers(0, n_f)), int(rng.integers(16))
        t = int(terms[g])
        kind = j % 9
        if kind == 0:
            out.append(frame(g, x, rng.integers(0, 256, int(rng.integers(0, 24)), dtype=np.uint8).tobytes()))
        elif kind == 1:
            out.append(frame(n_f + int(rng.integers(0, 100)), x, message(3, term=t, index=1)))
        elif kind == 2:
            out.append(frame(g, x, message(3, term=t, index=5, commit=1 << 40, frm=3)[:-1]))
        elif kind == 3:
            out.append(frame(g, x, message(int(rng.choice([4, 8, 9, 17])), term=t, index=1)))
        elif kind == 4:
            out.append(frame(g, x, message(3, term=t, index=1, frm=2, entries=[(t, 2)] * int(rng.integers(1, 3)))))
        elif kind == 5:
            out.append(frame(g, x, message(3, term=0, index=1)))
        elif kind == 6:
            out.append(frame(g, x, message(3, term=max(1, t + int(rng.choice([-1, 1]))), index=1)))
        elif kind == 7:                                                # matches above last_index, commit_to out of range
            out.append(frame(g, x, message(3, term=t, log_term=0, index=U64 - 1, commit=U64 - 1, frm=2)))
        else:
            out.append(np.array([g << 4 | x], "<u4").tobytes()[: int(rng.integers(0, 4))])
    return out
