"""MsgAppend frames with entries for the follower tests (raftgpu_follower_append_entries, oracle/app_entries_oracle.c):
eraftpb.Entry records with every field, Messages built from them (hostile layouts included), and random frames for a
follower whose log, run and committed index are known."""
import numpy as np

from helpers import B
from oracle import app_follow_oracle as AL
import app_follow as A

varint = A.varint
U64 = A.U64


def entry(term=0, index=0, data=b"", context=b"", entry_type=0, sync_log=False) -> bytes:
    """eraftpb.Entry in field-number order, zero / empty fields omitted: 1 entry_type, 2 term, 3 index, 4 data,
    5 sync_log, 6 context."""
    out = b""
    if entry_type:
        out += varint(1 << 3) + varint(entry_type)
    for no, v in ((2, term), (3, index)):
        if v:
            out += varint(no << 3) + varint(v)
    if data:
        out += varint(4 << 3 | 2) + varint(len(data)) + data
    if sync_log:
        out += varint(5 << 3) + b"\x01"
    if context:
        out += varint(6 << 3 | 2) + varint(len(context)) + context
    return out


def record(e: bytes) -> bytes:
    """One field-7 record: tag, length, Entry."""
    return varint(7 << 3 | 2) + varint(len(e)) + e


def message(term=0, log_term=0, index=0, commit=0, frm=0, records=(), to=1, msg_type=3, split_at=None) -> bytes:
    """eraftpb.Message in field-number order (zero scalars omitted) with the field-7 records as given; split_at: a
    reject_hint field between records[split_at - 1] and records[split_at]."""
    out = b""
    for no, v in ((1, msg_type), (2, to), (3, frm), (4, term), (5, log_term), (6, index)):
        if v:
            out += varint(no << 3) + varint(v)
    for k, r in enumerate(records):
        if split_at is not None and k == split_at:
            out += varint(11 << 3) + varint(7)
        out += r
    if commit:
        out += varint(8 << 3) + varint(commit)
    return out


PAYLOADS = (0, 1, 16, 127, 128, 1000, 20_000)


def random_frame(rng, last, run_start, run_term, term, committed, big=False, hostile=0.0):
    """A MsgAppend at term to a follower whose log ends at last with the run [run_start, last] of run_term: most often a
    match inside the run with 0-64 entries (overlapping, truncating inside the run, or past last_index), else stale,
    rejected or a gap; hostile: the fraction of frames with a term-0 entry, wrong indexes, a split span, a scalar
    field 7 or a truncated Entry.  big: payloads up to past the 16 KiB stage."""
    kind = rng.random()
    lo = max(run_start, committed)
    if kind < 0.7 and lo <= last:
        index = int(rng.integers(lo, last + 1))
        log_term = run_term
    elif kind < 0.8 and committed > 0:
        index = int(rng.integers(0, committed))
        log_term = int(rng.integers(0, term + 1))
    elif kind < 0.9:
        index = int(rng.integers(0, last + 3))
        log_term = int(rng.integers(run_term + 1, term + 2))
    else:
        index = last + int(rng.integers(1, 3))
        log_term = 0
    n = int(rng.choice([0, 1, 2, 3, 8, 64], p=[0.1, 0.4, 0.2, 0.15, 0.1, 0.05]))
    terms = []
    t = run_term
    for j in range(n):
        i = index + 1 + j
        if i <= last and rng.random() < 0.85 and (not terms or terms[-1] == run_term):
            terms.append(run_term)                                        # overlap: matches the run
        else:
            if rng.random() < 0.3:
                t = int(rng.integers(max(t, 1), term + 1))
            terms.append(max(t, 1))
    sizes, p = (PAYLOADS, [0.3, 0.2, 0.2, 0.1, 0.1, 0.09, 0.01]) if big else (PAYLOADS[:4], None)
    ents = [entry(tt, index + 1 + j, data=bytes(int(rng.choice(sizes, p=p)) * [0x5A]) if rng.random() < 0.5 else b"",
                  context=b"ctx" if rng.random() < 0.1 else b"", entry_type=int(rng.random() < 0.1))
            for j, tt in enumerate(terms)]
    split = None
    if n and rng.random() < hostile:
        h = int(rng.integers(0, 5))
        j = int(rng.integers(0, n))
        if h == 0:
            ents[j] = entry(0, index + 1 + j)
        elif h == 1:
            ents[j] = entry(terms[j], index + 2 + j)
        elif h == 2 and n > 1:
            split = int(rng.integers(1, n))
        elif h == 3:
            recs = [record(e) for e in ents]
            recs.insert(j, varint(7 << 3) + varint(5))
            return message(term, log_term, index, int(rng.integers(0, index + n + 2)), int(rng.integers(1, 1 << 40)), recs)
        else:
            ents[j] = ents[j] + b"\x10"                                   # a tag without its value
    commit = int(rng.integers(0, index + n + 1)) if rng.random() < 0.95 else int(rng.integers(0, last + n + 5))
    return message(term, log_term, index, commit, int(rng.integers(1, 1 << 40)), [record(e) for e in ents], split_at=split)


WIDE_LO = 0x20000000  # RAFTGPU_META_WIDE_LO


NAMES = ("status", "from", "appended", "response bytes", "response offsets", "totals")


def world(rng, n_narrow, n_wide, reads):
    """A follower arena of n_narrow groups then n_wide pairs at random terms and logs, and its log table with random runs
    -> (arena, host columns, read queues or None, table)."""
    n = n_narrow + 2 * n_wide
    terms = rng.integers(2, 1000, n).astype(np.uint64)
    last = rng.integers(0, 1 << 20, n).astype(np.uint64)
    committed = last - np.minimum(last, rng.integers(0, 40, n).astype(np.uint64))
    hi = np.arange(n_narrow + 1, n, 2)
    terms[hi] = terms[hi - 1]
    term_start = np.where(rng.random(n) < 0.03, np.uint64(1), np.uint64(A.NO_TERM_START))
    cols = {B.COL_TERM: terms, B.COL_LAST_INDEX: last, B.COL_COMMITTED: committed, B.COL_TERM_START: term_start}
    a, c, q = A.follower_arena(n_narrow, n_wide, cols, reads)
    table = np.zeros(a.get_info().hi, AL.LOG_DTYPE)
    table["id"][:n] = rng.integers(1, 1 << 63, n, dtype=np.uint64)
    table["flags"][:n] = np.where(rng.random(n) < 0.97, AL.SELECT, 0)
    top = np.maximum(c.last_index[:n], np.concatenate([c.last_index[1:n], [0]]))
    table["run_start"][:n] = np.where(rng.random(n) < 0.95, top - np.minimum(top, rng.integers(0, 50, n).astype(np.uint64)),
                                      top + 1)
    table["run_term"][:n] = terms - rng.integers(0, 2, n).astype(np.uint64)
    return a, c, q, table


N_NARROW, N_WIDE = 99_000, 500
