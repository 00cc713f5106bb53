"""The fused tile kernels' launch plan, restated, and the shape matrix of test_gpu_tile_shapes.py checked
on the CPU: that it reaches every stage count of both kernels, and that its states and batches exercise
every apply path (through the oracle only, so the GPU tests cannot go vacuous unnoticed)."""
import numpy as np
import pytest

from helpers import (B, GROUPS, KERNELS, O, TILE_SHAPES, UNIT_CAP, is_simple5, plan, random_batch, random_state,
                     stage_bytes, stages)


# stage counts per number of hinted slots H = 1..8
WANT_STAGES = {"packed": (8, 8, 8, 6, 5, 4, 4, 3), "compact": (8, 8, 6, 5, 4, 4, 3, 3)}


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
