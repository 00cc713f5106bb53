"""step_tile_kernel's record buffers: each consumer group copies up to REC_CAP packed records of its next tile into
shared memory and reads the rest of a crowded tile from HBM (k_tile.cuh, kRecCap).

Batches whose tiles hold exactly REC_CAP - 1, REC_CAP and REC_CAP + 1 packed records; a REJECT at position
REC_CAP - 1, so that its EXT record (the hint, and a snapshot request) is the first record past the copy; crowded tiles
beside record-less ones in a random order, so that both buffers of a consumer group and empty fills follow each other;
at a size where the stage ring wraps.  Both instantiations (kSimple5, and the general one with
RAFTGPU_FORCE_GENERAL=1) run the same state and batches; every round is compared with the oracle (result bytes,
advanced bitmap, commit_out, counters, every column).  Run with -m gpu."""
import numpy as np
import pytest

from helpers import B, O, TILE_SHAPES, fused_round, random_state, ring_wrapping_groups

pytestmark = pytest.mark.gpu

REC_CAP = 4 * B.tile_groups()          # kRecCap
PK_REJECT, PK_EXT = 1 << 35, 1 << 37   # wire_format.h
EDGE = "edge"                          # the kind of a tile whose REJECT sits at REC_CAP - 1

# the kinds of tile a batch mixes: name -> the tile's plan, a list of either an exact number of packed records of
# random kinds, or ("reject", packed records of that REJECT: 2 with a hint, 3 with a snapshot request as well)
PLANS = {
    "empty": [],
    "light": [137],
    "cap - 1": [REC_CAP - 1],
    "cap": [REC_CAP],
    "cap + 1": [REC_CAP + 1],
    EDGE: [REC_CAP - 1, ("reject", 2)],
    "edge with a snapshot request": [REC_CAP - 1, ("reject", 3), 211],
    "snapshot request past the cap": [REC_CAP - 2, ("reject", 3), 95],
    "crowded": [3 * REC_CAP // 2],
}


def tile_sizes(rng, self_slot, plan):
    """The packed size of the record of each cell of one tile (group order, each group's slots in a random order;
    0: no record) so that the tile packs to exactly what `plan` says.  A leader's own slot only takes size 1."""
    ng = len(self_slot)
    slots = rng.random((ng, O.SLOTS)).argsort(axis=1)
    g = np.repeat(np.arange(ng), O.SLOTS)
    s = slots.ravel()
    own = s == np.repeat(self_slot, O.SLOTS)
    size = np.zeros(len(s), dtype=np.int64)
    at = 0
    for step in plan:
        if isinstance(step, tuple):
            at += int(np.argmax(~own[at:]))          # a REJECT: not on a leader's own slot
            size[at] = step[1]
            at += 1
            continue
        want = np.where(own[at:], 1, rng.choice([1, 2, 3], p=[0.6, 0.3, 0.1], size=len(s) - at))
        cum = np.cumsum(want)
        last = int(np.searchsorted(cum, step))       # the first cell at which the tile reaches `step`
        want[last] -= cum[last] - step
        size[at:at + last + 1] = want[:last + 1]
        at += last + 1
    return g, s, size


def records(ref, rng, g, s, size):
    """One record per cell of packed size `size`, never WIDE: 1 an accept, or a LOCAL record on the leader's own
    slot; 2 a REJECT with a hint (EXT); 3 the same with a snapshot request."""
    r = len(g)
    m = ref.matched[s, g].astype(np.int64)
    nx = ref.next_idx[s, g].astype(np.int64)
    meta = ref.meta[g].astype(np.int64)
    local = ((meta & O.META_HAS_SELF) != 0) & (((meta >> 24) & 7) == s)
    reject = size >= 2
    index, commit = np.maximum(0, m + rng.integers(-6, 12, r)), np.zeros(r, dtype=np.int64)
    commit[:] = np.maximum(0, index - np.where(rng.random(r) < 0.05, rng.integers(0, 300, r), rng.integers(0, 6, r)))
    li = m + rng.integers(0, 8, r)
    index[local] = li[local]
    commit[local] = np.where(rng.random(r) < 0.2, 0, li + rng.integers(0, 5, r))[local]
    ri = np.stack([nx - 1, m, m + 1, m + 3, np.maximum(0, m - 2)])[rng.integers(0, 5, r), np.arange(r)]
    index[reject] = ri[reject]
    commit[reject] = np.minimum(ri, np.maximum(0, m - rng.integers(0, 4, r)))[reject]
    pos = np.arange(r) + np.cumsum(reject) - reject          # each EXT right behind its REJECT
    out = np.zeros(r + int(reject.sum()), dtype=O.APPEND_RESP_DTYPE)
    out["group"][pos], out["peer_slot"][pos] = g, s
    out["flags"][pos] = np.where(local, O.REC_LOCAL, np.where(reject, O.REC_REJECT, 0))
    out["index"][pos], out["commit"][pos] = index, commit
    pe = pos[reject] + 1
    out["group"][pe], out["peer_slot"][pe], out["flags"][pe] = g[reject], s[reject], O.REC_EXT
    out["index"][pe] = np.maximum(0, ri + rng.integers(-5, 3, r))[reject]
    out["commit"][pe] = np.where(size == 3, rng.integers(1, 1 << 30, r), 0)[reject]
    return out


def batch(ref, rng, n):
    """A batch in group order whose tiles take the plans of PLANS in a random order -> (records, kind of every tile).
    The ragged last tile stays light."""
    tg = B.tile_groups()
    n_tiles = -(-n // tg)
    names = sorted(PLANS)
    kinds = [names[i] for i in rng.integers(0, len(names), n_tiles - 1)] + ["light"]
    meta = ref.meta[:n].astype(np.int64)
    self_slot = np.where(meta & O.META_HAS_SELF, (meta >> 24) & 7, O.SLOTS)
    gs, ss, sizes = [], [], []
    for t, kind in enumerate(kinds):
        g0 = t * tg
        g, s, size = tile_sizes(rng, self_slot[g0:g0 + tg], PLANS[kind])
        on = size > 0
        gs.append(g[on] + g0)
        ss.append(s[on])
        sizes.append(size[on])
    return records(ref, rng, np.concatenate(gs), np.concatenate(ss), np.concatenate(sizes)), kinds


def packed_size(plan):
    return sum(step[1] if isinstance(step, tuple) else step for step in plan)


@pytest.mark.parametrize("name", ["v5_simple", "v5_general"])
def test_record_buffers_at_their_edges(name, monkeypatch):
    shape, _, force_general, seed = TILE_SHAPES[name]
    if force_general:
        monkeypatch.setenv("RAFTGPU_FORCE_GENERAL", "1")     # read when an arena is created
    else:
        monkeypatch.delenv("RAFTGPU_FORCE_GENERAL", raising=False)
    n = ring_wrapping_groups()
    rng = np.random.default_rng(seed)
    ref = random_state(n, shape, rng)
    arena = B.Arena(n)
    assert arena.group_alloc_range(n) == 0
    arena.load_columns(ref)
    tg = B.tile_groups()
    pk = np.zeros((2 * REC_CAP * (n // tg + 1), 2), dtype=np.uint64)
    d_bufs = (arena.device_alloc(pk.nbytes), arena.device_alloc(4 * (n // tg + 2)), arena.device_alloc(pk.shape[0]),
              arena.device_alloc(arena.cap // 8), arena.device_alloc(8 * arena.cap))
    rng = np.random.default_rng(seed + 1)        # the same batches for both instantiations
    for rnd in range(3):
        recs, kinds = batch(ref, rng, n)
        # the batch is what the plans say: every tile's packed size, and a REJECT at REC_CAP - 1 of every edge tile
        k = arena.pack_records(recs, pk)
        off = B.tile_index(pk, k, n).astype(np.int64)
        assert [int(c) for c in np.diff(off)] == [packed_size(PLANS[kind]) for kind in kinds]
        for t in np.flatnonzero(np.array(kinds) == EDGE):
            w0, w1 = int(pk[off[t] + REC_CAP - 1, 0]), int(pk[off[t] + REC_CAP, 0])
            assert w0 & PK_REJECT and not w0 & PK_EXT and w1 & PK_EXT
        assert {"empty", "cap", EDGE, "crowded"} <= set(kinds)
        fused_round(arena, n, recs, ref, pk, d_bufs)
    arena.close()
