"""Shared test glue: product binding + oracle side by side, the random states and batches of the
differential tests, and one checked step of each device-resident fused tile kernel."""
import importlib
from dataclasses import dataclass

import numpy as np

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


def random_batch(ref, rng, per_cell, keep=None):
    """A batch in group order for the groups of `ref`: 70 % of the groups (of those `keep` selects) get
    records for 1-5 random peer slots, the group's peers or not, each cell up to `per_cell` records.  The
    leader's own slot gets LOCAL records; other slots accepts (stale ones, commits above the index, commits
    far below it) or rejections, 85 % of them with a hint (EXT), a fifth of those with a snapshot request."""
    n = ref.n_groups
    on = rng.random(n) >= 0.3
    if keep is not None:
        on &= keep
    k = rng.integers(1, 6, n)
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

    pos = np.arange(r) + np.cumsum(ext) - ext                 # each EXT right behind its REJECT
    out = np.zeros(r + int(ext.sum()), dtype=O.APPEND_RESP_DTYPE)
    out["group"][pos], out["peer_slot"][pos] = g, s
    out["flags"][pos] = np.where(local, O.REC_LOCAL, np.where(reject, O.REC_REJECT, 0))
    out["index"][pos], out["commit"][pos] = index, commit
    pe = pos[ext] + 1
    out["group"][pe], out["peer_slot"][pe], out["flags"][pe] = g[ext], s[ext], O.REC_EXT
    out["index"][pe], out["commit"][pe] = ext_index[ext], ext_snapshot[ext]
    return out


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
    assert np.array_equal(res[main_pk], want_res[main_orig]), "per-record results differ"
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
