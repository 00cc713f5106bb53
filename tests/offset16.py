"""The edges of the 16-bit offset window of next_idx and peer_committed, for the tests.

On the device both are int16 offsets from the cell's matched; an offset outside (INT16_MIN, INT16_MAX] is stored
as the escape code INT16_MIN with the exact value in the u64 column beside it (k_common.cuh).  helpers.py keeps the
generators of the wider window the codec had before (edge_state, random_batch(edge=True)); these are the same
generators at this window: states with cells exactly on either side of both bounds, and batches that land cells on
the bounds and move them across, both ways, through the records the fused fast path takes and through the others."""
import numpy as np

from helpers import O, offset_of, random_batch

I16_MIN, I16_MAX = -(2 ** 15), 2 ** 15 - 1
EDGE16_FITS = (0, 1, -1, I16_MAX, I16_MIN + 1)                                  # distances stored as offsets
EDGE16_ESCAPES = (I16_MAX + 1, I16_MIN, I16_MIN - 1, 1 << 31, -(1 << 40))       # and distances that escape
EDGE16_D = np.array(EDGE16_FITS + EDGE16_ESCAPES)
RESET16_LAST = (2 ** 15 - 2, 2 ** 15 - 1, 2 ** 15, 2 ** 32 + 5)                   # last indexes of the Raft::reset shape
_BELOW = np.array([I16_MIN + 1, I16_MIN, I16_MIN - 1])                           # landing distances at the lower bound
_ABOVE = np.array([I16_MAX, I16_MAX + 1, I16_MAX - 1])                           # and at the upper one
_STEP = 1 << 15
_INDEX_LIMIT = 1 << 48   # as in helpers: the compact stream's run headers hold 48-bit bases

# record kinds of edge_batch
(K_RANDOM, K_LOCAL_JUMP, K_PROBE_REJECT, K_WIDE_RAISE, K_COMMIT_UP, K_RESET_RETURN, K_ESCAPED, K_PAIR) = range(8)


def fits16(value, matched):
    """The host model of off_encode: True where `value` is stored as an offset from `matched`."""
    d = offset_of(value, matched)
    return (d > I16_MIN) & (d <= I16_MAX)


def escaped16(c, n=None):
    """[SLOTS][n] bool: cells whose next_idx or peer_committed escapes."""
    n = c.n_groups if n is None else n
    m = c.matched[:, :n]
    return ~fits16(c.next_idx[:, :n], m) | ~fits16(c.peer_committed[:, :n], m)


def edge_state16(c, rng, frac=0.3, n=None, escape_groups=None):
    """helpers.edge_state at this window: next_idx and peer_committed of a fraction `frac` of the cells of groups
    [0, n) at distances from EDGE16_FITS + EDGE16_ESCAPES, a fifth of those in the Raft::reset shape (matched 0,
    next_idx = last_index + 1, Probe); every peer cell of the groups `escape_groups` selects escaped.  In place."""
    n = c.n_groups if n is None else n
    shape = (O.SLOTS, n)
    m = c.matched[:, :n].astype(np.int64)
    pick = rng.random(shape) < frac
    esc_d = np.array(EDGE16_ESCAPES)

    def place(full):
        d = np.where(full, esc_d[rng.integers(0, len(esc_d), shape)], EDGE16_D[rng.integers(0, len(EDGE16_D), shape)])
        v = m + d
        return np.where((v < 0) | (v >= _INDEX_LIMIT), m - d, v)

    full = np.zeros(shape, dtype=bool) if escape_groups is None else np.broadcast_to(escape_groups[:n], shape)
    pick |= full
    nx, pc = place(full), place(full)
    c.next_idx[:, :n] = np.where(pick, nx, c.next_idx[:, :n])
    c.peer_committed[:, :n] = np.where(pick, pc, c.peer_committed[:, :n])
    reset = pick & (rng.random(shape) < 0.2)
    last = np.array(RESET16_LAST)[rng.integers(0, len(RESET16_LAST), shape)]
    c.matched[:, :n][reset] = 0
    c.next_idx[:, :n][reset] = last[reset] + 1
    c.pflags[:, :n][reset] = O.STATE_PROBE
    c.pending_snapshot[:, :n][reset] = 0
    c.pending_request_snapshot[:, :n][reset] = 0
    return c


def edge_batch(ref, rng, per_cell, keep=None, with_kinds=False):
    """random_batch(ref, rng, per_cell, keep), then some of its records rewritten -- each keeping its kind (LOCAL,
    accept, REJECT with its EXT hint) -- to land a cell on either side of a bound of the window:
    - K_LOCAL_JUMP: a LOCAL record raising the self slot's matched so that peer_committed - matched lands at
      -(2^15 - 1), -2^15 or -2^15 - 1 (or next_idx - matched at 2^15 - 1, 2^15 or 2^15 - 2); the fast path takes it.
    - K_PROBE_REJECT: a REJECT of a Probe-state peer at next_idx - 1 whose hint lands next_idx at matched - 2^15 + 1,
      matched - 2^15 or one below (the fast path takes these too).
    - K_WIDE_RAISE: an accept raising matched like the LOCAL jumps, with a commit below.
    - K_COMMIT_UP: an accept whose commit is 2^15 - 1, 2^15 or 2^15 - 2 above the new matched.
    - K_RESET_RETURN: an accept at last_index of a peer in the reset shape.
    - K_ESCAPED: the records left on cells that are escaped already.
    - K_PAIR: the first two accepts of a cell with several: escape, then return (or the reverse), in one batch.
    With `with_kinds` the result is (records, kind of every record)."""
    out = random_batch(ref, rng, per_cell, keep=keep)
    main = np.flatnonzero((out["flags"] & O.REC_EXT) == 0)
    r = len(main)
    g, s = out["group"][main].astype(np.int64), out["peer_slot"][main].astype(np.int64)
    local = (out["flags"][main] & O.REC_LOCAL) != 0
    reject = (out["flags"][main] & O.REC_REJECT) != 0
    accept = ~local & ~reject
    nxt = np.minimum(main + 1, len(out) - 1)
    hinted = reject & (main + 1 < len(out)) & ((out["flags"][nxt] & O.REC_EXT) != 0)
    index, commit = out["index"][main].astype(np.int64), out["commit"][main].astype(np.int64)
    ext_index, ext_snap = out["index"][nxt].astype(np.int64), out["commit"][nxt].astype(np.int64)
    cell = g * 8 + s
    first = np.r_[True, cell[1:] != cell[:-1]] if r else np.zeros(0, dtype=bool)
    rank = np.arange(r) - np.maximum.accumulate(np.where(first, np.arange(r), 0))
    m = ref.matched[s, g].astype(np.int64)
    nx = ref.next_idx[s, g].astype(np.int64)
    pc = ref.peer_committed[s, g].astype(np.int64)
    state = ref.pflags[s, g] & O.PF_STATE_MASK
    esc = ~fits16(nx, m) | ~fits16(pc, m)
    u = rng.random(r)
    free = np.ones(r, dtype=bool)
    kind = np.zeros(r, dtype=np.uint8)

    def take(mask, k, new_index=None):
        mask &= free
        if new_index is not None:
            mask &= (new_index >= 0) & (new_index < _INDEX_LIMIT)
        free[mask] = False
        kind[mask] = k
        return mask

    # escape and return within one batch: a cell's first two records, both accepts
    second = (rank == 1) & accept & np.r_[False, accept[:-1]] & (rng.random(r) < 0.6)
    pc_up = rng.integers(0, 2, r)
    x = np.maximum(np.maximum(m, pc), nx - 1) + 1
    for lead, back in ((~esc, m + 6 + _STEP), (esc, x + 1)):
        sel = second & lead & (back < _INDEX_LIMIT)
        sel[1:] &= free[:-1]
        a1 = take(sel.copy(), K_PAIR)
        a0 = np.r_[a1[1:], False]
        free[a0], kind[a0] = False, K_PAIR
        if lead is esc:                                                     # return, then escape
            index[a0], commit[a0] = x[a0], x[a0]
            index[a1], commit[a1] = (x + 1)[a1], (x + 1 + _STEP + pc_up)[a1]
        else:                                                               # escape (commit 2^15 + above), then return
            index[a0], commit[a0] = (m + 1)[a0], (m + 1 + _STEP + pc_up)[a0]
            index[a1], commit[a1] = (m + 6 + _STEP)[a1], (m + 5 + _STEP)[a1]

    below = _BELOW[rng.integers(0, 3, r)]
    above = _ABOVE[rng.integers(0, 3, r)]
    lift_pc = pc - m - below                                           # raise matched by this: pc lands at `below`
    lift_nx = nx - above                                               # matched to land next_idx at `above`
    to_nx = (lift_nx > m) & (local | (state == O.STATE_REPLICATE)) & (rng.random(r) < 0.7)
    lifted = np.where(to_nx, lift_nx, m + lift_pc)
    ok = to_nx | (lift_pc > 0)
    a = take(local & ok & (u < 0.7), K_LOCAL_JUMP, new_index=lifted)
    index[a] = lifted[a]
    commit[a] = np.where(rng.random(r) < 0.4, 0, lifted + rng.integers(0, 1000, r))[a]

    a = take(hinted & (state == O.STATE_PROBE) & (m >= _STEP + 4) & (nx >= 1) & (u < 0.35), K_PROBE_REJECT)
    index[a] = (nx - 1)[a]
    commit[a] = np.maximum(0, nx - 1 - rng.integers(0, 4, r))[a]
    ext_index[a], ext_snap[a] = (m + below - 1)[a], 0

    a = take(accept & ok & (u < 0.5), K_WIDE_RAISE, new_index=lifted)
    index[a], commit[a] = lifted[a], np.maximum(0, np.minimum(pc, m) - 1 - rng.integers(0, 4, r))[a]

    a = take(accept & (m == 0) & (nx >= 1) & (u < 0.8), K_RESET_RETURN)
    li = nx - 1
    index[a] = li[a]
    commit[a] = np.where(rng.random(r) < 0.5, 0, li - rng.integers(0, 3, r).clip(0, li))[a]

    top = m + rng.integers(0, 3, r)
    a = take(accept & (u < 0.65), K_COMMIT_UP, new_index=top + above)
    index[a], commit[a] = top[a], (top + above)[a]

    kind[free & esc] = K_ESCAPED
    # (random_batch's hostile values, such as a rejection at next_idx - 1 of a next_idx 0, went through int64 above
    # and come back unchanged)
    out["index"][main], out["commit"][main] = index.astype(np.uint64), commit.astype(np.uint64)
    h = main[hinted]
    out["index"][h + 1], out["commit"][h + 1] = ext_index[hinted].astype(np.uint64), ext_snap[hinted].astype(np.uint64)
    if not with_kinds:
        return out
    kinds = np.zeros(len(out), dtype=np.uint8)
    kinds[main] = kind
    kinds[h + 1] = kind[hinted]
    return out, kinds


def self_behind16(c, rng, n, frac=0.5):
    """Groups whose leader's matched lies 2^15 - 1, 2^15 or 2^15 + 1 below the index every other voter has
    acknowledged (and the group can commit): the recompute raises the leader's peer_committed to it
    (hot_update_committed), landing it on, or just past, the upper bound.  Returns the groups chosen."""
    meta = c.meta[:n].astype(np.int64)
    has = ((meta & O.META_HAS_SELF) != 0) & (c.term_start[:n] != O.U64_MAX) & (rng.random(n) < frac)
    own = (meta >> 24) & 7
    x = c.last_index[:n].astype(np.int64) + (1 << 20)
    gap = np.array([I16_MAX, I16_MAX + 1, I16_MAX + 2])[rng.integers(0, 3, n)]
    g = np.flatnonzero(has)
    c.matched[:, g] = x[g]
    c.next_idx[:, g] = x[g] + 1
    c.peer_committed[:, g] = x[g] - 3
    c.matched[own[g], g] = x[g] - gap[g]
    c.next_idx[own[g], g] = x[g] - gap[g] + 1
    c.peer_committed[own[g], g] = x[g] - gap[g]
    c.committed[g] = x[g] - 10
    c.term_start[g] = x[g] - 20
    c.last_index[g] = x[g] + 5
    return has
