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


def leader_arena(c, n, runs):
    """An arena of n groups loaded from the oracle columns c (terms included), with leader runs when runs is set."""
    a = B.Arena(n)
    if runs:
        a.enable_leader_runs()
    assert a.group_alloc_range(n) == 0
    a.load_columns(c)
    a.column_write(B.COL_TERM, 0, 0, c.term[:n].copy())
    return a


def leader_frames(rng, c, groups, peers, per_cell, needs_log=0.0, stale=0.2):
    """1..per_cell MsgAppendResponse frames per (group, peer) cell, the cells interleaved in a random arrival order (a
    cell's frames keep theirs): accepts at increasing indexes (a fraction `stale` at an index already matched),
    rejections with log_term 0 at the probe's index, and a fraction needs_log of rejections with log_term > 0."""
    cells = []
    for g in groups:
        last = int(c.last_index[g])
        for s in peers:
            k = int(rng.integers(1, per_cell + 1))
            idx = sorted(rng.integers(0, last + 1, k).tolist())
            fr = []
            for j in range(k):
                if rng.random() < 0.25:
                    lt = int(rng.integers(1, 40)) if rng.random() < needs_log else 0
                    body = response(int(c.term[g]), index=int(rng.integers(0, last + 1)), reject=True,
                                      hint=int(rng.integers(0, last + 2)), log_term=lt)
                else:
                    i = idx[j] if rng.random() >= stale else int(rng.integers(0, idx[j] + 1))
                    body = response(int(c.term[g]), index=i, commit=int(rng.integers(0, last + 1)))
                fr.append(A.frame(g, s, body))
            cells.append(fr)
    order = rng.permutation(sum(len(f) for f in cells))
    owner = np.repeat(np.arange(len(cells)), [len(f) for f in cells])[order]
    pos = [0] * len(cells)
    out = []
    for cell in owner.tolist():       # each cell's frames in their order, cells interleaved
        out.append(cells[cell][pos[cell]])
        pos[cell] += 1
    return out


def pipelined_appends(rng, last, run_term, term, committed, k, entries=True):
    """k pipelined MsgAppend bodies to a follower whose log ends at `last` with term run_term: frame j's entries (1-3
    at `term`) start at frame j-1's last index + 1; without entries, k heartbeat-like appends at `last` with rising
    commits.  -> [(body, last index after it)]."""
    out, idx, lt = [], last, run_term
    for _ in range(k):
        if entries:
            cnt = int(rng.integers(1, 4))
            ents = [(term, idx + j + 1) for j in range(cnt)]
        else:
            cnt, ents = 0, None
        top = idx + cnt
        commit = int(rng.integers(min(committed, top), top + 1))
        out.append((A.message(3, term=term, log_term=lt, index=idx, commit=commit, frm=int(rng.integers(1, 1 << 40)),
                              entries=ents), top))
        if entries:
            idx, lt = top, term
    return out


def interleave(rng, per_group):
    """[(group, [frames])] -> one batch order: every group's frames in their order, the groups interleaved."""
    owner = np.repeat(np.arange(len(per_group)), [len(f) for _, f in per_group])
    owner = owner[rng.permutation(len(owner))]
    pos = [0] * len(per_group)
    out = []
    for k in owner.tolist():
        out.append(per_group[k][1][pos[k]])
        pos[k] += 1
    return out
