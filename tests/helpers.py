"""Shared test glue: product binding + oracle side by side, the random states and batches of the
differential tests, and one checked step of each device-resident fused tile kernel."""
import importlib
from dataclasses import dataclass

import numpy as np

from oracle import datadriven as dd
from oracle import oracle as O

B = importlib.import_module("raft-rs_b200").binding

COMPARE_COLUMNS = ("matched", "next_idx", "peer_committed", "pending_snapshot",
                   "pending_request_snapshot", "commit_group_id", "pflags", "meta", "committed",
                   "term_start", "last_index")


def assert_columns_equal(got, want, n, what=""):
    for name in COMPARE_COLUMNS:
        a, b = getattr(got, name)[..., :n], getattr(want, name)[..., :n]
        if not np.array_equal(a, b):
            bad = np.argwhere(a != b)[:5]
            raise AssertionError(f"{what}: column {name} differs at {bad.tolist()}: "
                                 f"got {a[tuple(bad[0])]} want {b[tuple(bad[0])]}")


def bitmap_to_bool(bm, n):
    return np.unpackbits(np.ascontiguousarray(bm).view(np.uint8), bitorder="little")[:n].astype(bool)


def checksum(arr) -> int:
    """Order-sensitive 64-bit checksum (wrapping multiply-add) for full-size comparisons."""
    a = np.ascontiguousarray(arr).astype(np.uint64).ravel()
    w = (np.arange(a.size, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15)) | np.uint64(1)
    with np.errstate(over="ignore"):
        return int((a * w).sum(dtype=np.uint64))


# --------------------------------------------------------------------------- random states and batches

@dataclass(frozen=True)
class Shape:
    """A family of group configurations for random_state.

    Every group draws one (incoming, outgoing, learner_pool) mask triple from `confs`; half of the groups
    then get learners, a random subset of learner_pool outside the group's voters.  `confs=None` draws
    arbitrary masks instead: any incoming set, an outgoing half in 30 % of the groups, learners in 40 %.
    With `group_commit`, 15 % of the groups use group commit.  The leader's own slot is absent in 10 % of
    the groups; otherwise it is one of the group's voters, or with `self_any_peer` any of its peers."""
    confs: tuple = None
    group_commit: bool = False
    self_any_peer: bool = False


# The configurations the fused tile kernels are tested at: name -> (shape, the union of its groups' voter
# masks = the voter hint of an arena holding them, RAFTGPU_FORCE_GENERAL, seed).  The two v5 cases hold the
# same groups and batches; only the kernel instantiation differs.
_V5 = Shape(((0x1f, 0, 0xe0),))
TILE_SHAPES = {
    "v1": (Shape(((0x01, 0, 0xfe),), group_commit=True), 0x01, False, 101),
    "v3": (Shape(((0x07, 0, 0xf8),), group_commit=True), 0x07, False, 103),
    "v4": (Shape(((0x0f, 0, 0xf0),), group_commit=True), 0x0f, False, 104),
    "v5_simple": (_V5, 0x1f, False, 105),
    "v5_general": (_V5, 0x1f, True, 105),
    "v6": (Shape(((0x38, 0x07, 0xc0), (0x07, 0x38, 0xc0)), group_commit=True), 0x3f, False, 106),
    "joint7": (Shape(((0x1f, 0x67, 0x80),), group_commit=True), 0x7f, False, 107),
    "any8": (Shape(None, group_commit=True), 0xff, False, 108),
    # 3-subsets of {1, 2, 5, 7}: learners anywhere else, the leader sometimes a learner outside the hint
    "sparse_a": (Shape(((0x26, 0, 0xd9), (0x86, 0, 0x79), (0xa2, 0, 0x5d), (0xa4, 0, 0x5b)), group_commit=True,
                       self_any_peer=True), 0xa6, False, 109),
    "sparse_b": (Shape(((0xe0, 0, 0x1f),), group_commit=True), 0xe0, False, 110),
}


def is_simple5(meta):
    """The plain 5-voter configuration the kSimple5 kernels are specialised for (is_simple5, arena.cu)."""
    return (np.asarray(meta, dtype=np.uint32) & np.uint32(0xffff | O.META_GROUP_COMMIT | 0x60000000)) == 0x1f


def _random_bit(mask, rng):
    """One set bit (slot number) of every mask, uniformly; 0 for an empty mask."""
    bits = (mask[:, None] >> np.arange(8)) & 1
    return (rng.random((len(mask), 8)) * bits).argmax(axis=1)


def random_state(n, shape, rng):
    """Host columns of n groups: configurations from `shape`; per-peer states in Probe, Replicate and
    Snapshot, paused and inflights-full flags, pending snapshots and snapshot requests, commit group ids;
    term_start = u64::MAX (not the leader of its term) in 5 % of the groups.  1 % of the groups have
    indexes around 2^32 or 2^48, beyond what a compact run header's 48-bit base holds."""
    c = O.new_columns(n, n)
    if shape.confs is None:
        inc = rng.integers(1, 256, n)
        out = np.where(rng.random(n) < 0.3, rng.integers(0, 256, n), 0)
        lrn = np.where(rng.random(n) < 0.4, rng.integers(0, 256, n), 0) & ~(inc | out)
    else:
        confs = np.array(shape.confs, dtype=np.int64)
        pick = confs[rng.integers(0, len(confs), n)]
        inc, out = pick[:, 0], pick[:, 1]
        lrn = np.where(rng.random(n) < 0.5, pick[:, 2] & rng.integers(0, 256, n), 0) & ~(inc | out)
    peers = inc | out | (lrn if shape.self_any_peer else 0)
    has_self = rng.random(n) < 0.9
    gc = shape.group_commit & (rng.random(n) < 0.15)
    meta = inc | (out << 8) | (lrn << 16) | np.where(has_self, (_random_bit(peers, rng) << 24) | O.META_HAS_SELF, 0) | \
        np.where(gc, O.META_GROUP_COMMIT, 0)
    c.meta[:] = meta.astype(np.uint32)

    base = rng.integers(100, 1 << 40, n)
    edge = rng.random(n) < 0.01
    base = np.where(edge, np.where(rng.random(n) < 0.5, 1 << 32, 1 << 48) + rng.integers(-20, 30, n), base)
    c.last_index[:] = base + rng.integers(0, 10, n)
    c.term_start[:] = np.maximum(1, base - rng.integers(0, 30, n))
    c.term_start[rng.random(n) < 0.05] = np.uint64(O.U64_MAX)
    c.committed[:] = base - rng.integers(0, 40, n)
    c.term[:] = rng.integers(1, 1000, n)

    m = base - rng.integers(0, 50, (O.SLOTS, n))
    c.matched[:] = m
    c.next_idx[:] = m + 1 + rng.integers(0, 5, (O.SLOTS, n))
    c.peer_committed[:] = m - rng.integers(0, 5, (O.SLOTS, n))
    state = np.array([O.STATE_PROBE, O.STATE_REPLICATE, O.STATE_REPLICATE, O.STATE_SNAPSHOT])[rng.integers(0, 4, (O.SLOTS, n))]
    c.pflags[:] = state | np.where(rng.random((O.SLOTS, n)) < 0.3, O.PF_PAUSED, 0) | \
        np.where(rng.random((O.SLOTS, n)) < 0.2, O.PF_INS_FULL, 0) | np.where(rng.random((O.SLOTS, n)) < 0.5, O.PF_RECENT_ACTIVE, 0)
    c.pending_snapshot[:] = np.where(state == O.STATE_SNAPSHOT, m + rng.integers(0, 6, (O.SLOTS, n)), 0)
    c.pending_request_snapshot[:] = np.where(rng.random((O.SLOTS, n)) < 0.05, rng.integers(1, 100, (O.SLOTS, n)), 0)
    c.commit_group_id[:] = rng.integers(0, 4, (O.SLOTS, n))
    return c


def random_batch(ref, rng, per_cell, keep=None, edge=False, with_kinds=False):
    """A batch in group order for the groups of `ref`: 70 % of the groups (of those `keep` selects) get
    records for 1-5 random peer slots, the group's peers or not, each cell up to `per_cell` records.  The
    leader's own slot gets LOCAL records; other slots accepts (stale ones, commits above the index, commits
    far below it) or rejections, 85 % of them with a hint (EXT), a fifth of those with a snapshot request.

    With `edge`, records are drawn from the state to put cells exactly on either side of the offset window of
    next_idx and peer_committed (_edge_records; groups whose eight cells are all escaped get records on all eight
    slots).  With `with_kinds` the result is (records, kind of every record: K_*)."""
    n = ref.n_groups
    on = rng.random(n) >= 0.3
    if keep is not None:
        on &= keep
    k = rng.integers(1, 6, n)
    if edge:
        crowd = (escaped_cells(ref).sum(axis=0) == O.SLOTS) & (True if keep is None else keep)
        on |= crowd
        k = np.where(crowd, O.SLOTS, k)
    perm = rng.random((n, O.SLOTS)).argsort(axis=1)           # every group's peer slots in a random order
    g, j = np.nonzero(on[:, None] & (np.arange(O.SLOTS) < k[:, None]))
    cnt = rng.integers(1, per_cell + 1, len(g))
    g, s = np.repeat(g, cnt), np.repeat(perm[g, j], cnt)
    r = len(g)
    m = ref.matched[s, g].astype(np.int64)
    nx = ref.next_idx[s, g].astype(np.int64)
    meta = ref.meta[g].astype(np.int64)
    local = ((meta & O.META_HAS_SELF) != 0) & (((meta >> 24) & 7) == s)
    accept = ~local & (rng.random(r) < 0.7)
    reject = ~local & ~accept

    index, commit = np.zeros(r, dtype=np.int64), np.zeros(r, dtype=np.int64)
    li = m + rng.integers(0, 8, r)
    index[local] = li[local]
    commit[local] = np.where(rng.random(r) < 0.2, 0, li + rng.integers(0, 5, r))[local]
    ai = np.maximum(0, m + rng.integers(-6, 12, r))
    drop = np.where(rng.random(r) < 0.05, rng.integers(0, 300, r), rng.integers(0, 6, r))
    index[accept] = ai[accept]
    commit[accept] = np.where(rng.random(r) < 0.03, ai + 3, np.maximum(0, ai - drop))[accept]
    ri = np.stack([nx - 1, m, m + 1, m + 3, np.maximum(0, m - 2)])[rng.integers(0, 5, r), np.arange(r)]
    index[reject] = ri[reject]
    commit[reject] = np.maximum(0, m - rng.integers(0, 4, r))[reject]
    ext = reject & (rng.random(r) < 0.85)
    ext_index = np.maximum(0, ri + rng.integers(-5, 3, r))
    ext_snapshot = np.where(rng.random(r) < 0.2, rng.integers(1, 1 << 30, r), 0)
    kind = np.zeros(r, dtype=np.uint8)
    if edge:
        rank = np.arange(r) - np.repeat(np.cumsum(cnt) - cnt, cnt)    # a record's place among its cell's
        _edge_records(ref, rng, g, s, rank, local, accept, reject, ext, index, commit, ext_index, ext_snapshot, kind)

    pos = np.arange(r) + np.cumsum(ext) - ext                 # each EXT right behind its REJECT
    out = np.zeros(r + int(ext.sum()), dtype=O.APPEND_RESP_DTYPE)
    out["group"][pos], out["peer_slot"][pos] = g, s
    out["flags"][pos] = np.where(local, O.REC_LOCAL, np.where(reject, O.REC_REJECT, 0))
    out["index"][pos], out["commit"][pos] = index, commit
    pe = pos[ext] + 1
    out["group"][pe], out["peer_slot"][pe], out["flags"][pe] = g[ext], s[ext], O.REC_EXT
    out["index"][pe], out["commit"][pe] = ext_index[ext], ext_snapshot[ext]
    if not with_kinds:
        return out
    kinds = np.zeros(len(out), dtype=np.uint8)
    kinds[pos], kinds[pe] = kind, kind[ext]
    return out, kinds


# --------------------------------------------------------------------------- the offset window of next_idx / peer_committed
# On the device next_idx and peer_committed are int32 offsets from the cell's matched; an offset outside
# (INT32_MIN, INT32_MAX] is stored as the escape code INT32_MIN with the exact value beside it (k_common.cuh).

I32_MIN, I32_MAX = -(2 ** 31), 2 ** 31 - 1
EDGE_FITS = (0, 1, -1, I32_MAX, I32_MIN + 1)                         # distances value - matched stored as offsets
EDGE_ESCAPES = (I32_MAX + 1, I32_MIN, I32_MIN - 1, 1 << 40, -(1 << 40))  # and the ones that escape
RESET_LAST = (2 ** 31 - 2, 2 ** 31 - 1, 2 ** 31, 2 ** 32 + 5, 2 ** 48 + 3)  # last indexes of the Raft::reset shape
_BELOW = np.array([I32_MIN + 1, I32_MIN, I32_MIN - 1])             # landing distances at the lower bound
_ABOVE = np.array([I32_MAX, I32_MAX + 1, I32_MAX - 1])             # and at the upper one
# indexes the edge records stay below: a compact run header holds a 48-bit base, and a batch must stay tileable for
# the fused compact kernels to take it (one with several records per cell has no other way in)
_INDEX_LIMIT = 1 << 48

# record kinds of random_batch(edge=True)
(K_RANDOM, K_LOCAL_JUMP, K_PROBE_REJECT, K_WIDE_RAISE, K_COMMIT_UP, K_RESET_RETURN, K_ESCAPED, K_PAIR) = range(8)


def offset_of(value, matched):
    """value - matched as a signed 64-bit distance (mod 2^64)."""
    return (np.asarray(value, dtype=np.uint64) - np.asarray(matched, dtype=np.uint64)).view(np.int64)


def fits(value, matched):
    """The host model of off_encode: True where `value` is stored as an offset from `matched`, False where it
    escapes."""
    d = offset_of(value, matched)
    return (d > I32_MIN) & (d <= I32_MAX)


def escaped_cells(c, n=None):
    """[SLOTS][n] bool: cells whose next_idx or peer_committed escapes."""
    n = c.n_groups if n is None else n
    m = c.matched[:, :n]
    return ~fits(c.next_idx[:, :n], m) | ~fits(c.peer_committed[:, :n], m)


def edge_state(c, rng, frac=0.3, n=None, escape_groups=None):
    """Moves next_idx and peer_committed of a fraction `frac` of the cells of groups [0, n) to the edges of the
    offset window, in place.  A chosen cell gets both values at distances from EDGE_FITS + EDGE_ESCAPES (drawn
    independently); a fifth of the chosen cells instead get the shape Raft::reset leaves (matched 0, next_idx =
    last_index + 1 for a last index from RESET_LAST, Probe, peer_committed kept).  Cells are drawn from every
    slot alike, so hinted slots, learners outside the hint, the self slot and Snapshot-state peers all get them.
    Every peer cell of the groups `escape_groups` selects gets escaping distances for both values (whole tiles of
    them overflow the fused kernels' per-warp lists of deferred records).  Values stay in [0, 2^63)."""
    n = c.n_groups if n is None else n
    shape = (O.SLOTS, n)
    m = c.matched[:, :n].astype(np.int64)
    pick = rng.random(shape) < frac
    all_d, esc_d = np.array(EDGE_FITS + EDGE_ESCAPES), np.array(EDGE_ESCAPES)

    def place(full):
        d = np.where(full, esc_d[rng.integers(0, len(esc_d), shape)], all_d[rng.integers(0, len(all_d), shape)])
        v = m + d
        return np.where((v < 0) | (v >= _INDEX_LIMIT), m - d, v)

    full = np.zeros(shape, dtype=bool) if escape_groups is None else np.broadcast_to(escape_groups[:n], shape)
    pick |= full
    nx, pc = place(full), place(full)
    c.next_idx[:, :n] = np.where(pick, nx, c.next_idx[:, :n])
    c.peer_committed[:, :n] = np.where(pick, pc, c.peer_committed[:, :n])
    reset = pick & (rng.random(shape) < 0.2)
    last = np.array(RESET_LAST)[rng.integers(0, len(RESET_LAST), shape)]
    c.matched[:, :n][reset] = 0
    c.next_idx[:, :n][reset] = last[reset] + 1
    c.pflags[:, :n][reset] = O.STATE_PROBE
    c.pending_snapshot[:, :n][reset] = 0
    c.pending_request_snapshot[:, :n][reset] = 0
    return c


def _edge_records(ref, rng, g, s, rank, local, accept, reject, ext, index, commit, ext_index, ext_snapshot, kind):
    """random_batch(edge=True): overwrites some of the drawn records (arrays edited in place) with records that land
    a cell on either side of a bound of the offset window, from the cell's state in `ref`:
    - K_LOCAL_JUMP: a LOCAL record raising the self slot's matched so that peer_committed - matched lands at
      -(2^31 - 1), -2^31 or -2^31 - 1 (or next_idx - matched at 2^31 - 1, 2^31 or 2^31 - 2 under a high next_idx);
      no commit or one within the packed 24-bit delta, so the fused fast path takes it.
    - K_PROBE_REJECT: a REJECT of a Probe-state peer at next_idx - 1 with an EXT hint landing next_idx at matched -
      2^31 + 1, matched - 2^31 or one below (the fast path takes these too).
    - K_WIDE_RAISE: an accept raising matched by 2^31 or more with a commit far below (packed WIDE), landing
      peer_committed (or next_idx of a Replicate peer) like the LOCAL jumps.
    - K_COMMIT_UP: an accept whose commit is 2^31 - 1, 2^31 or 2^31 + 1 above the new matched.
    - K_RESET_RETURN: an accept at last_index of a peer in the reset shape, with and without a commit.
    - K_ESCAPED: the ordinary records left on cells that are escaped already (the fast path must decline them).
    - K_PAIR: the first two records of a cell with several: escape, then return (or the reverse for a cell that
      is escaped), within one batch."""
    r = len(g)
    m = ref.matched[s, g].astype(np.int64)
    nx = ref.next_idx[s, g].astype(np.int64)
    pc = ref.peer_committed[s, g].astype(np.int64)
    state = ref.pflags[s, g] & O.PF_STATE_MASK
    esc = ~fits(nx, m) | ~fits(pc, m)
    u = rng.random(r)
    free = np.ones(r, dtype=bool)

    def take(mask, k, is_accept, is_reject=False, new_index=None):
        mask &= free
        if new_index is not None:
            mask &= new_index < _INDEX_LIMIT
        free[mask] = False
        kind[mask] = k
        accept[mask], reject[mask] = is_accept, is_reject
        ext[mask] = is_reject
        return mask

    # escape and return within one batch (several records per cell)
    step = 1 << 31
    cell = g.astype(np.int64) * 8 + s
    coin = rng.random(r)[np.arange(r) - rank]                          # one draw per cell
    pair = ~local & (rank <= 1) & np.isin(cell, cell[rank == 1]) & (coin < 0.6)
    pair &= np.where(esc, np.maximum(np.maximum(m, pc), nx - 1) + 2, m + 6 + step)[np.arange(r) - rank] < _INDEX_LIMIT
    pc_up = rng.integers(0, 2, r)
    x = np.maximum(np.maximum(m, pc), nx - 1) + 1
    a = take(pair & ~esc & (rank == 0), K_PAIR, True, new_index=m + 6 + step)                 # escape (commit 2^31 + above), then return
    index[a], commit[a] = (m + 1)[a], (m + 1 + step + pc_up)[a]
    a = take(pair & ~esc & (rank == 1), K_PAIR, True, new_index=m + 6 + step)
    index[a], commit[a] = (m + 6 + step)[a], (m + 5 + step)[a]
    a = take(pair & esc & (rank == 0), K_PAIR, True, new_index=x + 1)                  # return, then escape
    index[a], commit[a] = x[a], x[a]
    a = take(pair & esc & (rank == 1), K_PAIR, True, new_index=x + 1)
    index[a], commit[a] = (x + 1)[a], (x + 1 + step + pc_up)[a]

    below = _BELOW[rng.integers(0, 3, r)]
    above = _ABOVE[rng.integers(0, 3, r)]
    lift_pc = pc - m - below                                           # raise matched by this: pc lands at `below`
    lift_nx = nx - above                                               # matched to land next_idx at `above`
    to_nx = (lift_nx > m) & (local | (state == O.STATE_REPLICATE)) & (rng.random(r) < 0.7)
    lifted = np.where(to_nx, lift_nx, m + lift_pc)
    ok = to_nx | (lift_pc > 0)
    a = take(local & ok & (u < 0.7), K_LOCAL_JUMP, False, new_index=lifted)
    index[a] = lifted[a]
    commit[a] = np.where(rng.random(r) < 0.4, 0, lifted + rng.integers(0, 1000, r))[a]

    a = take(~local & (state == O.STATE_PROBE) & (m >= step + 4) & (nx >= 1) & (u < 0.35), K_PROBE_REJECT, False, True,
             new_index=nx)
    index[a] = (nx - 1)[a]
    commit[a] = np.maximum(0, nx - 1 - rng.integers(0, 4, r))[a]
    ext_index[a], ext_snapshot[a] = (m + below - 1)[a], 0

    a = take(~local & ok & (u < 0.5), K_WIDE_RAISE, True, new_index=lifted)
    index[a], commit[a] = lifted[a], np.maximum(0, np.minimum(pc, m) - 1 - rng.integers(0, 4, r))[a]

    a = take(~local & (m == 0) & (nx >= 1) & (u < 0.8), K_RESET_RETURN, True)
    li = nx - 1
    index[a] = li[a]
    commit[a] = np.where(rng.random(r) < 0.5, 0, li - rng.integers(0, 3, r).clip(0, li))[a]

    a = take(~local & (u < 0.65), K_COMMIT_UP, True)
    top = m + rng.integers(0, 3, r)
    index[a], commit[a] = top[a], (top + above)[a]

    kind[free & esc] = K_ESCAPED


# --------------------------------------------------------------------------- checked fused steps

_UNWRITTEN = np.uint64(0xDEADBEEFDEADBEEF)   # commit_out is filled with this before a step: every group must overwrite it


def _check_outputs(arena, n, ref, want_adv, want_bm, bm, com, before, what):
    words = (n + 31) // 32
    assert np.array_equal(bm[:words], want_bm[:words]), f"{what}: advanced bitmap differs"
    if not np.array_equal(com, ref.committed[:n]):
        g = int(np.flatnonzero(com != ref.committed[:n])[0])
        raise AssertionError(f"{what}: commit_out of group {g} is {com[g]}, want {ref.committed[g]}")
    after = arena.counters()
    assert after["recomputes"] - before["recomputes"] == arena.get_info().hi, f"{what}: recompute count"
    assert after["advanced"] - before["advanced"] == want_adv, f"{what}: advanced count"
    assert_columns_equal(arena.read_columns(n), ref, n, what)


def fused_round(arena, n, recs, ref, pk, d_bufs):
    """One fused step (raftgpu_step_sorted_device) on `recs` (group order) checked against the oracle: the
    result byte of every record, the advanced bitmap, the commit index of every group in [0, n), the
    recompute / advanced counters and every column.  Returns (groups advanced, result bytes of the records
    that are not EXT payloads)."""
    k = arena.pack_records(recs, pk)
    off = B.tile_index(pk, k, n)
    d_pk, d_off, d_res, d_bm, d_com = d_bufs
    arena.h2d(d_pk, pk[:k])
    arena.h2d(d_off, off)
    arena.h2d(d_bm, np.zeros(arena.cap // 32, dtype=np.uint32))   # bits past n_groups are left untouched
    arena.h2d(d_com, np.full(arena.cap, _UNWRITTEN, dtype=np.uint64))
    before = arena.counters()
    arena.step_sorted_device(d_pk, k, d_off, d_results=d_res, d_adv=d_bm, d_commit=d_com)
    res = np.zeros(k, dtype=np.uint8)
    bm = np.zeros(arena.cap // 32, dtype=np.uint32)
    com = np.zeros(n, dtype=np.uint64)
    arena.d2h(res, d_res)
    arena.d2h(bm, d_bm)
    arena.d2h(com, d_com)
    want_res = O.arena_apply(ref, recs, mode=0)
    want_adv, want_bm, _, _ = O.arena_recompute(ref)
    main_pk = (pk[:k, 0] & np.uint64(1 << 37)) == 0           # packed records that are not EXT payloads
    main_orig = (recs["flags"] & B.REC_EXT) == 0
    if not np.array_equal(res[main_pk], want_res[main_orig]):
        i = int(np.flatnonzero(res[main_pk] != want_res[main_orig])[0])
        raise AssertionError(f"per-record results differ: record {recs[main_orig][i]} got {res[main_pk][i]} "
                             f"want {want_res[main_orig][i]}")
    assert not res[~main_pk].any()
    _check_outputs(arena, n, ref, want_adv, want_bm, bm, com, before, "fused step")
    return want_adv, res[main_pk]


def compact_round(arena, n, recs, ref, blob, d_bufs, ordered=False):
    """One fused compact step (raftgpu_step_compact_device) on `recs` (group order), checked against the
    oracle like fused_round.  Returns (groups advanced, result bytes of the records that are not EXT payloads)."""
    nb, units = B.pack_compact(recs, blob, want_units=True)
    hdr = blob[:64].view(B.COMPACT_HDR_DTYPE)[0]
    assert hdr["flags"] & B.COMPACT_TILEABLE
    d_blob, d_off, d_res, d_bm, d_com, d_bad = d_bufs
    nu = int(hdr["n_units"])
    arena.h2d(d_blob, blob[:nb])
    arena.h2d(d_bm, np.zeros(arena.cap // 32, dtype=np.uint32))
    arena.h2d(d_com, np.full(arena.cap, _UNWRITTEN, dtype=np.uint64))
    arena.h2d(d_res, np.zeros(max(nu, 1), dtype=np.uint8))
    arena.h2d(d_bad, np.zeros(1, dtype=np.uint32))
    before = arena.counters()
    arena.compact_tile_index_device(d_blob, blob, d_off, d_bad)
    arena.step_compact_device(d_blob, blob, d_off, d_results=d_res, d_adv=d_bm, d_commit=d_com, d_dup=d_bad,
                              ordered=ordered)
    res = np.zeros(max(nu, 1), dtype=np.uint8)
    bm = np.zeros(arena.cap // 32, dtype=np.uint32)
    com = np.zeros(n, dtype=np.uint64)
    bad = np.zeros(1, dtype=np.uint32)
    arena.d2h(res, d_res)
    arena.d2h(bm, d_bm)
    arena.d2h(com, d_com)
    arena.d2h(bad, d_bad)
    assert bad[0] == 0
    want_res = O.arena_apply(ref, recs, mode=0)
    want_adv, want_bm, _, _ = O.arena_recompute(ref)
    main = (recs["flags"] & B.REC_EXT) == 0
    assert np.array_equal(res[units[main]], want_res[main]), "per-record results differ"
    other = np.ones(len(res), dtype=bool)
    other[units[main]] = False
    assert not res[other].any()
    _check_outputs(arena, n, ref, want_adv, want_bm, bm, com, before, "fused compact step")
    return want_adv, res[units[main]]


def compact_bufs(arena, n, per_group):
    """Host blob and device buffers (blob, tile table, results, bitmap, commit_out, duplicate count) for
    compact_round on batches of up to per_group records per group."""
    cap_b = B.compact_bound(per_group * n + 64)
    blob = np.zeros(cap_b, dtype=np.uint8)
    d = (arena.device_alloc(cap_b), arena.device_alloc(4 * (3 * (arena.cap // B.tile_groups() + 2) + 2)),
         arena.device_alloc(3 * per_group * n + 64), arena.device_alloc(arena.cap // 8),
         arena.device_alloc(8 * arena.cap), arena.device_alloc(4))
    return blob, d


# --------------------------------------------------------------------------- every way into the fused kernels

def ring_wrapping_groups():
    """A group count at which the fused kernels' stage ring wraps: 18 tiles per SM plus a ragged one: the grid is one CTA per SM (fewer only with fewer tiles), and consumer
    group cg of a CTA takes the CTA's tiles cg, cg + 3, ...; a stage is used again n_stages tiles later."""
    a = B.Arena(256)
    sm = a.info.sm_count
    a.close()
    tg = B.tile_groups()
    n = 18 * sm * tg + 77
    tiles = -(-n // tg)
    assert tiles > sm and n % tg
    assert tiles // sm >= 2 * 8 + 1       # every CTA wraps an 8-stage ring twice
    assert tiles // sm // 3 >= 5          # every consumer group gets at least 5 tiles
    return n


class Paths:
    """One arena per way into the fused kernels, loaded with the same state, each with its oracle copy."""

    def __init__(self, n, init, records_api):
        self.n = n
        names = ["packed", "compact", "ordered"] + (["records"] if records_api else [])
        self.arenas, self.refs = {}, {}
        for name in names:
            a = B.Arena(n)
            assert a.group_alloc_range(n) == 0
            a.load_columns(init)
            self.arenas[name], self.refs[name] = a, O.copy_columns(init)
        pa = self.arenas["packed"]
        self.pk = np.zeros((16 * n, 2), dtype=np.uint64)
        self.d_packed = (pa.device_alloc(self.pk.nbytes), pa.device_alloc(4 * (n // B.tile_groups() + 2)),
                         pa.device_alloc(8 * n), pa.device_alloc(pa.cap // 8), pa.device_alloc(8 * pa.cap))
        self.blob, self.d_compact = compact_bufs(self.arenas["compact"], n, 12)
        _, self.d_ordered = compact_bufs(self.arenas["ordered"], n, 12)

    def round(self, recs, per_cell, what):
        """One batch through every path that takes it; returns the per-record result bytes of each."""
        assert len(recs) <= 6 * self.n
        out = {}
        B.pack_compact(recs, self.blob)
        if not self.blob[:64].view(B.COMPACT_HDR_DTYPE)[0]["flags"] & B.COMPACT_TILEABLE:
            # a unit block of the compact stream holds runs of groups at most 4095 past its first: a batch spread
            # thinner than that is not tileable (the library steps it with the scatter kernel)
            out["packed"] = fused_round(self.arenas["packed"], self.n, recs, self.refs["packed"], self.pk, self.d_packed)[1]
            for name in self.arenas:
                if name != "packed":
                    self.arenas[name].load_columns(self.refs["packed"])
                    self.refs[name] = O.copy_columns(self.refs["packed"])
            return out
        if per_cell == 1:
            out["packed"] = fused_round(self.arenas["packed"], self.n, recs, self.refs["packed"], self.pk, self.d_packed)[1]
            out["compact"] = compact_round(self.arenas["compact"], self.n, recs, self.refs["compact"], self.blob,
                                           self.d_compact)[1]
        out["ordered"] = compact_round(self.arenas["ordered"], self.n, recs, self.refs["ordered"], self.blob,
                                       self.d_ordered, ordered=True)[1]
        if "records" in self.arenas:
            records_round(self.arenas["records"], self.n, recs, self.refs["records"], what)
        if per_cell > 1:       # the packed and per-unit kernels promise one record per cell: catch them up
            for name in ("packed", "compact"):
                self.arenas[name].load_columns(self.refs["ordered"])
                self.refs[name] = O.copy_columns(self.refs["ordered"])
        return out

    def reload(self, state):
        """Every arena and oracle copy to `state` (host columns)."""
        for name, a in self.arenas.items():
            a.load_columns(state)
            self.refs[name] = O.copy_columns(state)

    def close(self):
        for a in self.arenas.values():
            a.close()


def records_round(arena, n, recs, ref, what):
    """raftgpu_step_begin_records: the library packs the batch and picks the kernel and its plan itself."""
    arena.step_begin_records(recs, B.STEP_READ_COMMITTED)
    r = arena.step_wait()
    O.arena_apply(ref, recs, mode=0)
    want_adv, want_bm, _, _ = O.arena_recompute(ref)
    assert r.n_advanced == want_adv and r.n_duplicates == 0, what
    # the fused kernel counts records without their EXT payloads (the scatter fallback counts both)
    assert r.n_records == np.count_nonzero((recs["flags"] & B.REC_EXT) == 0), what
    bm, com = arena.step_results(n)
    assert np.array_equal(bm, want_bm[: len(bm)]), what
    adv = bitmap_to_bool(bm, n)
    assert np.array_equal(com[adv], ref.committed[:n][adv]), what
    assert_columns_equal(arena.read_columns(n), ref, n, f"records API, {what}")


# --------------------------------------------------------------------------- arenas set up like a wire-pass scenario

ARENA_COLUMNS = ("term_start", "committed", "last_index", "matched", "next_idx", "peer_committed", "pflags")


def votes(a, n):
    """The arena's votes of groups [0, n): u8 [SLOTS][n]."""
    return np.stack([a.column_read(B.COL_VOTES, s, 0, n, np.uint8) for s in range(O.SLOTS)])


def check_columns(a, c, vt, n, ins=False):
    """The arena's ARENA_COLUMNS, terms and votes (and Inflights metas with ins) of groups [0, n) against the oracle's
    columns c and votes vt."""
    cols = a.read_columns(n)
    for name in ARENA_COLUMNS:
        assert np.array_equal(getattr(cols, name), getattr(c, name)[..., :n]), name
    assert np.array_equal(a.column_read(B.COL_TERM, 0, 0, n, np.uint64), c.term[:n])
    assert np.array_equal(votes(a, n), vt[:, :n])
    if ins:
        for s in range(O.SLOTS):
            assert np.array_equal(a.column_read(B.COL_INS_META, s, 0, n, np.uint32), c.ins_meta[s, :n]), s


def arena_of(s, read_index=False, inflights=0, leader_runs=False):
    """An arena of s.n + 64 group slots set up like scenario s (vote_request_frames.Scenario, follow_term.scenario,
    vote_frames.Election): s.n_narrow narrow groups from slot 0, then s.n_wide wide pairs, then the control list
    s.setup and, where s has one, s.campaign."""
    a = B.Arena(s.n + 64)
    if read_index:
        a.enable_read_index()
    if inflights:
        a.enable_inflights(inflights)
    if leader_runs:
        a.enable_leader_runs()
    if s.n_narrow:
        assert a.group_alloc_range(s.n_narrow) == 0
    for k in range(s.n_wide):
        assert a.group_alloc_wide() == s.n_narrow + 2 * k
    assert np.all(a.control(s.setup)["status"] == 0)
    if getattr(s, "campaign", None) is not None:
        a.control(s.campaign)
    return a


def oracle_wire_step(ref, wb, n_groups, terms):
    """What the step must do: local records first, then every frame the decoder accepts, in frame order (the first
    frame of a cell; later ones are DUP), then Raft::maybe_commit for every group.  Returns (status bytes, adv bitmap)."""
    res_local = O.arena_apply(ref, wb.records[: wb.n_records].copy(), mode=0) if wb.n_records else None
    status, recs, hint, snap = O.wire_decode_batch(wb.bytes[: wb.n_bytes], wb.offsets[: wb.n + 1], n_groups, terms)
    ok = np.nonzero(status == O.WIRE_OK)[0]
    rows = []
    for i in ok:
        rows.append(tuple(recs[i]))
        if recs["flags"][i] & B.REC_REJECT:
            rows.append((recs["group"][i], recs["peer_slot"][i], B.REC_EXT, 0, hint[i], snap[i]))
    seq = np.array(rows, dtype=B.APPEND_RESP_DTYPE) if rows else np.zeros(0, dtype=B.APPEND_RESP_DTYPE)
    res = O.arena_apply(ref, seq, mode=0)
    main = (seq["flags"] & B.REC_EXT) == 0
    want = (status.astype(np.uint32) << 4).astype(np.uint8)
    want[ok] |= res[main] & 0xF
    adv, bm, _, _ = O.arena_recompute(ref)
    return want, bm, adv, res_local


def oracle_wire_apply(c, blob, offsets, n, terms, n_bytes=None):
    """raftgpu_wire_apply_device: the AppendResponse frames, first of every cell, in frame order."""
    status, recs, hint, snap = O.wire_decode_batch(blob, offsets, n, terms, n_bytes)
    ok = np.nonzero(status == O.WIRE_OK)[0]
    rows = []
    for i in ok:
        rows.append(tuple(recs[i]))
        if recs["flags"][i] & B.REC_REJECT:
            rows.append((recs["group"][i], recs["peer_slot"][i], B.REC_EXT, 0, hint[i], snap[i]))
    seq = np.array(rows, dtype=B.APPEND_RESP_DTYPE) if rows else np.zeros(0, dtype=B.APPEND_RESP_DTYPE)
    res = O.arena_apply(c, seq, mode=0)
    want = (status.astype(np.uint32) << 4).astype(np.uint8)
    want[ok] |= res[(seq["flags"] & B.REC_EXT) == 0] & 0xF
    return want


def full_state(arena, n, inflights=False):
    """Every column of groups [0, n): the host-column set, votes, term and (with inflights) the Inflights meta."""
    c = arena.read_columns(n)
    votes = np.stack([arena.column_read(B.COL_VOTES, s, 0, n, np.uint8) for s in range(B.SLOTS)])
    c.term[:] = arena.column_read(B.COL_TERM, 0, 0, n, np.uint64)
    ins = None
    if inflights:
        ins = np.stack([arena.column_read(B.COL_INS_META, s, 0, n, np.uint32) for s in range(B.SLOTS)])
    return c, votes, ins


def assert_state_equal(a, b, n, what):
    ca, va, ia = a
    cb, vb, ib = b
    assert_columns_equal(ca, cb, n, what)
    assert np.array_equal(ca.term[:n], cb.term[:n]), f"{what}: term"
    assert np.array_equal(va[:, :n], vb[:, :n]), f"{what}: votes"
    if ia is not None or ib is not None:
        assert np.array_equal(ia[:, :n], ib[:, :n]), f"{what}: ins_meta"


def records_step(arena, n, recs, ref, what):
    """raftgpu_step_begin_records (the library picks the kernel from its launch plan), checked against the oracle."""
    arena.step_begin_records(recs, B.STEP_READ_COMMITTED)
    r = arena.step_wait()
    O.arena_apply(ref, recs, mode=0)
    want_adv, want_bm, _, _ = O.arena_recompute(ref)
    assert r.n_advanced == want_adv, what
    bm, com = arena.step_results(n)
    assert np.array_equal(bm, want_bm[: len(bm)]), what
    adv = bitmap_to_bool(bm, n)
    assert np.array_equal(com[adv], ref.committed[:n][adv]), what
    assert_columns_equal(arena.read_columns(n), ref, n, what)


def scatter_step(arena, n, recs, ref, what):
    """Enqueued records and raftgpu_step, checked against the oracle."""
    arena.enqueue(recs)
    r = arena.step(B.STEP_READ_COMMITTED)
    O.arena_apply(ref, recs, mode=0)
    want_adv, _, _, _ = O.arena_recompute(ref)
    assert r.n_advanced == want_adv, what
    assert_columns_equal(arena.read_columns(n), ref, n, what)


def several_tiles():
    """Seven full tiles and a ragged eighth."""
    return 7 * B.tile_groups() + 77


def escape_tiles(n):
    """Every ninth tile: each of its cells escaped."""
    return (np.arange(n) // B.tile_groups()) % 9 == 4


def storm(c, rng, n):
    """The state right after an election at a last index past 2^31 (Raft::reset, then become_leader): every peer
    cell but the leader's own has matched 0 and next_idx = last_index + 1, both escaped."""
    last = np.array(RESET_LAST[1:])[rng.integers(0, len(RESET_LAST) - 1, n)]
    meta = c.meta[:n].astype(np.int64)
    own = ((meta & O.META_HAS_SELF) != 0)[None, :] & (((meta >> 24) & 7)[None, :] == np.arange(O.SLOTS)[:, None])
    follower = ~own
    c.last_index[:n] = last
    c.term_start[:n] = last
    c.committed[:n] = np.minimum(c.committed[:n], last - 1)
    c.matched[:, :n] = np.where(follower, 0, last)                 # the leader: persisted = last_index
    c.peer_committed[:, :n] = np.where(follower, c.peer_committed[:, :n], c.committed[:n])
    c.next_idx[:, :n] = last + 1
    c.pflags[:, :n] = np.where(follower, O.STATE_PROBE, c.pflags[:, :n])
    c.pending_snapshot[:, :n] = np.where(follower, 0, c.pending_snapshot[:, :n])
    c.pending_request_snapshot[:, :n] = np.where(follower, 0, c.pending_request_snapshot[:, :n])
    assert not fits(c.next_idx[:, :n][follower], 0).any()
    return c


def as_set(e):
    return sorted(zip(e["group"].tolist(), e["peer_slot"].tolist(), e["flags"].tolist(), e["next_idx"].tolist()))


class GpuQuorum:
    """Evaluates the quorum functions on the GPU: voter ids are mapped to peer slots of one
    arena group, acked indexes become its matched / commit_group_id columns."""

    def __init__(self, arena):
        self.a = arena
        self.g = arena.group_alloc()

    def _setup(self, incoming, outgoing, lookup, gc):
        ids = []
        for i in list(incoming) + list(outgoing):
            if i not in ids:
                ids.append(i)
        assert len(ids) <= B.SLOTS
        slot = {i: s for s, i in enumerate(ids)}
        m_in = sum(1 << slot[i] for i in set(incoming))
        m_out = sum(1 << slot[i] for i in set(outgoing))
        self.a.group_set_conf(self.g, 0, 0, 0, None, 1)            # drop every Progress
        self.a.group_set_conf(self.g, m_in, m_out, 0, None, 1)
        self.a.set_group_commit(self.g, gc)
        for i, s in slot.items():
            p = self.a.progress_get(self.g, s)
            p.matched, p.commit_group_id = lookup.get(i, (0, 0))   # missing voter == (0, 0)
            self.a.progress_set(self.g, s, p)
        return slot

    def joint(self, incoming, outgoing, lookup, gc):
        self._setup(incoming, outgoing, lookup, gc)
        return self.a.maximal_committed_index(self.g)

    def majority(self, voters, lookup, gc):
        return self.joint(voters, [], lookup, gc)

    def joint_vote(self, incoming, outgoing, votes):
        slot = self._setup(incoming, outgoing, {}, False)
        self.a.reset_votes(self.g)
        for i, v in votes.items():
            if i in slot:
                self.a.record_vote(self.g, slot[i], v)
        return self.a.vote_result(self.g)[2]

    def majority_vote(self, voters, votes):
        return self.joint_vote(voters, [], votes)

    def impl(self):
        return dd.Impl(self.majority, self.joint, self.majority_vote, self.joint_vote)


def random_config_state(n, rng):
    """Arbitrary configurations (joint, learners, group commit, no self) and per-peer states."""
    c = O.new_columns(n, n)
    for g in range(n):
        inc = int(rng.integers(1, 256))
        out = int(rng.integers(0, 256)) if rng.random() < 0.3 else 0
        learners = int(rng.integers(0, 256)) & ~(inc | out) if rng.random() < 0.4 else 0
        voters = [s_ for s_ in range(8) if (inc | out) >> s_ & 1]
        self_slot = int(rng.choice(voters)) if rng.random() < 0.9 else None
        c.meta[g] = O.make_meta(inc, out, learners, self_slot, group_commit=bool(rng.random() < 0.15))
        base = int(rng.integers(100, 1 << 40))
        c.last_index[g] = base + int(rng.integers(0, 10))
        c.term_start[g] = (1 << 64) - 1 if rng.random() < 0.05 else max(1, base - int(rng.integers(0, 30)))
        c.committed[g] = base - int(rng.integers(0, 40))
        c.term[g] = int(rng.integers(1, 1000))
        for s_ in range(8):
            m = base - int(rng.integers(0, 50))
            c.matched[s_, g] = m
            c.next_idx[s_, g] = m + 1 + int(rng.integers(0, 5))
            c.peer_committed[s_, g] = m - int(rng.integers(0, 5))
            state = int(rng.choice([O.STATE_PROBE, O.STATE_REPLICATE, O.STATE_REPLICATE, O.STATE_SNAPSHOT]))
            c.pflags[s_, g] = state | (O.PF_PAUSED if rng.random() < 0.3 else 0) | (O.PF_INS_FULL if rng.random() < 0.2 else 0) | \
                (O.PF_RECENT_ACTIVE if rng.random() < 0.5 else 0)
            c.pending_snapshot[s_, g] = m + int(rng.integers(0, 6)) if state == O.STATE_SNAPSHOT else 0
            c.pending_request_snapshot[s_, g] = int(rng.integers(1, 100)) if rng.random() < 0.05 else 0
            c.commit_group_id[s_, g] = int(rng.integers(0, 4))
    return c


def random_cell_batch(ref, n, rng, per_cell):
    """Group-ordered batch; `per_cell` > 1 lets a (group, peer) cell receive several records."""
    rows = []
    for g in range(n):
        if rng.random() < 0.3:
            continue
        meta = int(ref.meta[g])
        has_self, self_slot = bool(meta & O.META_HAS_SELF), (meta >> 24) & 7
        slots = rng.permutation(8)[: int(rng.integers(1, 6))]
        for s_ in slots:
            s_ = int(s_)
            for _ in range(int(rng.integers(1, per_cell + 1))):
                m, nx = int(ref.matched[s_, g]), int(ref.next_idx[s_, g])
                kind = rng.random()
                if has_self and s_ == self_slot:
                    idx = m + int(rng.integers(0, 8))
                    rows.append((g, s_, B.REC_LOCAL, 0, idx, 0 if rng.random() < 0.2 else idx + int(rng.integers(0, 5))))
                elif kind < 0.7:
                    idx = max(0, m + int(rng.integers(-6, 12)))
                    commit = idx + 3 if rng.random() < 0.03 else max(0, idx - int(rng.integers(0, 300 if rng.random() < 0.05 else 6)))
                    rows.append((g, s_, 0, 0, idx, commit))
                else:
                    idx = int(rng.choice([nx - 1, m, m + 1, m + 3, max(0, m - 2)]))
                    rows.append((g, s_, B.REC_REJECT, 0, idx, max(0, m - int(rng.integers(0, 4)))))
                    if rng.random() < 0.85:
                        rows.append((g, s_, B.REC_EXT, 0, max(0, idx + int(rng.integers(-5, 3))),
                                     int(rng.integers(1, 1 << 30)) if rng.random() < 0.2 else 0))
    return np.array(rows, dtype=B.APPEND_RESP_DTYPE) if rows else np.zeros(0, dtype=B.APPEND_RESP_DTYPE)


# k_tile.cuh: tile geometry and shared memory of the fused tile kernels
TILE, GROUPS, MAX_STAGES = 256, 3, 8


ROW64, ROW8 = (TILE + 2) * 8, TILE + 16


SMEM = 227 * 1024 - 5 * 1024


UNIT_CAP = 1536


KERNELS = {"packed": (0, 0), "compact": (4 * UNIT_CAP, GROUPS * TILE * 4)}   # (payload bytes, extra bytes)


def stage_bytes(h, payload):
    return 3 * h * ROW64 + 3 * ROW64 + TILE * 4 + h * ROW8 + payload


def stages(h, kernel):
    payload, extra = KERNELS[kernel]
    return min(MAX_STAGES, (SMEM - extra) // stage_bytes(h, payload))


def plan(meta, force_general, kernel):
    """tile_plan (arena.cu): (simple5 instantiation, hint, stages) of an arena whose groups hold `meta`."""
    simple5 = not force_general and bool(is_simple5(meta).all())
    hint = 0x1f if simple5 else int(np.bitwise_or.reduce((meta & 0xff) | ((meta >> 8) & 0xff)))
    return simple5, hint, stages(bin(hint).count("1"), kernel)
