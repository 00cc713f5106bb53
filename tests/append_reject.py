"""Leaders for the rejection tests of the wire step with leader runs (raftgpu_leader_runs_set, oracle/leader_runs_oracle.c):
literal leader logs (a term per index, the dummy entry at 0), the rows they imply, MsgAppendResponse frames built field by
field, and the oracle's step: the batch form's statuses and hints applied through the records every wire test uses."""
import numpy as np

from helpers import B, O
from oracle import leader_runs_oracle as LR
import app_follow as A


def response(term, index=0, reject=False, hint=0, log_term=0, commit=0, snap=0, frm=2) -> bytes:
    """A MsgAppendResponse (msg_type 4) in field-number order, zero scalars omitted."""
    out = b""
    for no, v in ((1, 4), (2, 1), (3, frm), (4, term), (5, log_term), (6, index), (8, commit), (10, int(reject)),
                  (11, hint), (13, snap)):
        if v:
            out += A.varint(no << 3) + A.varint(v)
    return out


def random_log(rng, n_runs, leader_term=None):
    """A leader's log with n_runs term runs, the last one its own term: terms[i] of entry i, terms[0] = 0."""
    terms = sorted(rng.choice(np.arange(1, 40), size=n_runs, replace=False).tolist())
    if leader_term is not None:
        terms[-1] = leader_term
    out = [0]
    for t in terms:
        out += [t] * int(rng.integers(1, 6))
    return out


def rows_for(logs, first_index, n_runs, cap=None):
    """ROW_DTYPE rows for every group's log (runs_of_log with n_runs runs)."""
    rows = np.zeros(cap or len(logs), LR.ROW_DTYPE)
    for g, t in enumerate(logs):
        term, ts, runs = LR.runs_of_log(t, int(first_index[g]), n_runs)
        rows[g] = LR.row(g, term, ts, runs)
    return rows


def leader_columns(logs, cap, n_peers=5, seed=0):
    """Columns of leaders with these logs: term = the last term, term_start / last_index from the log, every peer
    probing at next_idx = last_index + 1 (matched 0)."""
    n = len(logs)
    c = O.new_columns(cap, n)
    rng = np.random.default_rng(seed)
    for g, t in enumerate(logs):
        term, ts, _ = LR.runs_of_log(t, 1, 0)
        c.term[g], c.term_start[g], c.last_index[g] = term, ts, len(t) - 1
        c.committed[g] = int(rng.integers(0, ts))
    c.meta[:n] = O.make_meta((1 << n_peers) - 1, self_slot=0)
    for s in range(n_peers):
        c.next_idx[s, :n] = c.last_index[:n] + 1
        c.pflags[s, :n] = B.STATE_PROBE
    return c


def oracle_step(ref, rows, blob, offsets, n_bytes=None):
    """The wire step on the oracle's columns (changed in place): lro_decode_batch, then every WIRE_OK frame's record (and
    a REJECT's EXT with its hint) through ro_arena_apply, in frame order.  Returns the status bytes."""
    status, recs, hint, snap = LR.decode_batch(ref, rows, blob, offsets, n_bytes)
    ok = np.nonzero(status == O.WIRE_OK)[0]
    rws = []
    for i in ok:
        rws.append(tuple(recs[i]))
        if recs["flags"][i] & B.REC_REJECT:
            rws.append((recs["group"][i], recs["peer_slot"][i], B.REC_EXT, 0, hint[i], snap[i]))
    seq = np.array(rws, dtype=B.APPEND_RESP_DTYPE) if rws else np.zeros(0, dtype=B.APPEND_RESP_DTYPE)
    res = O.arena_apply(ref, seq, mode=0)
    main = (seq["flags"] & B.REC_EXT) == 0
    want = (status.astype(np.uint32) << 4).astype(np.uint8)
    want[ok] |= res[main] & 0xF
    return want
