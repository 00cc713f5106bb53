"""The fused tile kernels' launch plan, restated, and the shape matrix of test_gpu_tile_shapes.py checked
on the CPU: that it reaches every stage count of both kernels, and that its states and batches exercise
every apply path (through the oracle only, so the GPU tests cannot go vacuous unnoticed)."""
import numpy as np
import pytest

from helpers import B, O, TILE_SHAPES, is_simple5, random_batch, random_state

# k_tile.cuh: tile geometry and shared memory of the fused tile kernels
TILE, GROUPS, MAX_STAGES = 256, 3, 8
ROW64, ROW8 = (TILE + 2) * 8, TILE + 16
SMEM = 227 * 1024 - 5 * 1024
UNIT_CAP = 1536
KERNELS = {"packed": (0, 0), "compact": (4 * UNIT_CAP, GROUPS * TILE * 4)}   # (payload bytes, extra bytes)

# stage counts per number of hinted slots H = 1..8
WANT_STAGES = {"packed": (8, 8, 8, 6, 5, 4, 4, 3), "compact": (8, 8, 6, 5, 4, 4, 3, 3)}


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


needs_256 = pytest.mark.skipif(B.tile_groups() != 256, reason="the stage table is for 256-group tiles")


@needs_256
def test_stage_counts_restated():
    assert stage_bytes(5, 0) == 39536 and stage_bytes(5, 4 * UNIT_CAP) == 45680
    for kernel, want in WANT_STAGES.items():
        assert tuple(stages(h, kernel) for h in range(1, 9)) == want, kernel
        assert min(want) >= GROUPS        # wait_stage needs a stage per consumer group


@needs_256
def test_shape_matrix_covers_every_stage_count():
    reachable = {(k, s) for k, want in WANT_STAGES.items() for s in want}
    covered, at_h5 = set(), set()
    for name, (shape, hint, force_general, seed) in TILE_SHAPES.items():
        meta = random_state(3000, shape, np.random.default_rng(seed)).meta
        for kernel in KERNELS:
            simple5, h, n_stages = plan(meta, force_general, kernel)
            assert n_stages == WANT_STAGES[kernel][bin(hint).count("1") - 1], (name, kernel)
            covered.add((kernel, n_stages))
            if h == 0x1f:
                at_h5.add(simple5)
    assert covered == reachable
    assert at_h5 == {True, False}
    assert {h for _, h, _, _ in TILE_SHAPES.values()} >= {0xa6, 0xe0}    # hints that are not a prefix of the slots


@pytest.mark.parametrize("name", sorted(TILE_SHAPES))
def test_shape_states_and_batches_take_every_path(name):
    shape, hint, force_general, seed = TILE_SHAPES[name]
    rng = np.random.default_rng(seed)
    n = 3000
    ref = random_state(n, shape, rng)
    meta = ref.meta[:n].astype(np.int64)
    voters = (meta & 0xff) | ((meta >> 8) & 0xff)
    assert int(np.bitwise_or.reduce(voters)) == hint
    assert is_simple5(meta).all() == name.startswith("v5_")
    assert (ref.committed[:n] >> np.uint64(48)).any() and (ref.committed[:n] >> np.uint64(32) == 1).any()

    recs = random_batch(ref, rng, 1)
    assert np.all(np.diff(recs["group"].astype(np.int64)) >= 0)
    main = (recs["flags"] & O.REC_EXT) == 0
    g, s, f = recs["group"].astype(np.int64), recs["peer_slot"].astype(np.int64), recs["flags"]
    present = ((meta[g] | meta[g] >> 8 | meta[g] >> 16) >> s) & 1 == 1
    learner = (meta[g] >> 16 >> s) & 1 == 1
    snapshot = (ref.pflags[s, g] & O.PF_STATE_MASK) == O.STATE_SNAPSHOT
    nxt = np.append(recs[1:], recs[:1])
    snap_req = ((f & O.REC_REJECT) != 0) & ((nxt["flags"] & O.REC_EXT) != 0) & (nxt["commit"] != 0)
    res = O.arena_apply(ref, recs, mode=0)
    adv, _, _, _ = O.arena_recompute(ref)
    accept, reject = main & (f == 0), (f & O.REC_REJECT) != 0
    paths = {
        "update": accept & ((res & O.RES_OK) != 0),
        "stale accept": accept & present & (res == 0),
        "decrement": reject & ((res & O.RES_OK) != 0),
        "stale decrement": reject & present & (res == 0),
        "snapshot request": snap_req & present,
        "Snapshot-state peer": main & present & snapshot,
        "learner": main & learner,
        "absent peer": main & (res == O.RES_NO_PROGRESS),
        "LOCAL": (f & O.REC_LOCAL) != 0,
        "RES_OLD_PAUSED": (res & O.RES_OLD_PAUSED) != 0,
    }
    missing = [p for p, hit in paths.items() if not hit.any()]
    assert not missing, f"{name}: the batch never takes {missing}"
    assert adv > 0
    if name == "sparse_a":     # learners in hinted slots, and leaders outside the hint
        assert (main & learner & ((hint >> s) & 1 == 1)).any()
        has_self = (meta & O.META_HAS_SELF) != 0
        assert (has_self & ((hint >> ((meta >> 24) & 7)) & 1 == 0)).any()
