"""The fused tile kernels (step_tile_kernel, step_tile_compact_kernel) at a size where their stage ring
wraps, for every voter-slot layout the launch plan distinguishes.

The stage count depends on how many slots the arena's voter hint covers (TILE_SHAPES and
test_tile_shapes.py), the stage rows map to the hinted slots, and the kSimple5 instantiation runs only
while every group is the plain 5-voter configuration.  Each shape gets fresh arenas (the hint never
shrinks), one per way into the kernels, all loaded with the same random state; every step is compared
with the oracle: result bytes, advanced bitmap, commit_out, counters and every column.  Run with -m gpu.
"""
import numpy as np
import pytest

from helpers import (B, O, TILE_SHAPES, Paths, compact_bufs, compact_round, fused_round, is_simple5, random_batch,
                     random_state, ring_wrapping_groups)

pytestmark = pytest.mark.gpu

RECORDS_API_SHAPES = ("v3", "sparse_a", "joint7")


@pytest.fixture(scope="module")
def n_groups():
    return ring_wrapping_groups()


def run_shape(name, n, monkeypatch):
    """Every round of one shape on fresh arenas; the per-record result bytes of every round and path."""
    shape, hint, force_general, seed = TILE_SHAPES[name]
    if force_general:
        monkeypatch.setenv("RAFTGPU_FORCE_GENERAL", "1")     # read when an arena is created
    else:
        monkeypatch.delenv("RAFTGPU_FORCE_GENERAL", raising=False)
    rng = np.random.default_rng(seed)
    init = random_state(n, shape, rng)
    assert int(np.bitwise_or.reduce(init.meta[:n] & 0xff | (init.meta[:n] >> 8) & 0xff)) == hint
    paths = Paths(n, init, name in RECORDS_API_SHAPES)
    g = np.arange(n)
    tg = B.tile_groups()
    # light (record-less) tiles finish early and the loads of the next ones land out of order; the first two
    # partial batches are too thin for the compact stream, the next two are not
    thin = ("every seventh tile", "random 2 %")
    rounds = [("one wave", None, 1),
              ("every seventh tile", (g // tg) % 7 == 0, 1),
              ("random 2 %", rng.random(n) < 0.02, 1),
              ("every third tile", (g // tg) % 3 == 0, 1),
              ("random 25 %", rng.random(n) < 0.25, 1),
              ("suffix", g >= n - n // 50, 1),
              ("three records per cell", None, 3)]
    results = []
    for what, keep, per_cell in rounds:
        recs = random_batch(paths.refs["ordered"], rng, per_cell, keep)
        results.append(paths.round(recs, per_cell, f"{name}, {what}"))
        assert (list(results[-1]) == ["packed"]) == (what in thin), what
    paths.close()
    return results


@pytest.mark.parametrize("name", [s for s in sorted(TILE_SHAPES) if not s.startswith("v5_")])
def test_fused_kernels_at_ring_wrapping_size(name, n_groups, monkeypatch):
    run_shape(name, n_groups, monkeypatch)


def test_simple5_and_general_instantiations_agree(n_groups, monkeypatch):
    """The plain 5-voter store (self in slots 0-4 or none, learners in 5-7, adversarial peer states) through the
    kSimple5 kernels, then the same state and batches with RAFTGPU_FORCE_GENERAL=1 through the general ones."""
    simple = run_shape("v5_simple", n_groups, monkeypatch)
    general = run_shape("v5_general", n_groups, monkeypatch)
    for i, (a, b) in enumerate(zip(simple, general)):
        assert a.keys() == b.keys()
        for path in a:
            assert np.array_equal(a[path], b[path]), (i, path)


def test_tile_plan_changes_between_steps(n_groups):
    """One fused step through each kernel after every control-plane call that changes the launch plan of an
    arena that starts all plain 5-voter: the oracle state is read back from the arena after the call."""
    n = n_groups
    rng = np.random.default_rng(77)
    init = random_state(n, TILE_SHAPES["v5_simple"][0], rng)
    arena = B.Arena(n)
    assert arena.group_alloc_range(n) == 0
    arena.load_columns(init)
    tg = B.tile_groups()
    pk = np.zeros((8 * n, 2), dtype=np.uint64)
    d_packed = (arena.device_alloc(pk.nbytes), arena.device_alloc(4 * (arena.cap // tg + 2)), arena.device_alloc(8 * n),
                arena.device_alloc(arena.cap // 8), arena.device_alloc(8 * arena.cap))
    blob, d_compact = compact_bufs(arena, arena.cap, 12)

    def steps(simple5, what):
        hi = arena.get_info().hi
        ref = arena.read_columns(hi)
        assert is_simple5(ref.meta[:hi]).all() == simple5, what
        fused_round(arena, hi, random_batch(ref, rng, 1), ref, pk, d_packed)
        compact_round(arena, hi, random_batch(ref, rng, 1), ref, blob, d_compact)

    steps(True, "plain 5-voter")
    g6, gc, gf = 1000, n // 2, n - 300
    arena.group_set_conf(g6, 0x5f, 0, 0x80, 2, 1 << 20)          # slot 6 votes: general kernel, 6 hinted slots
    steps(False, "a sixth voter")
    arena.set_group_commit(gc, True)
    steps(False, "group commit on")
    arena.set_group_commit(gc, False)
    steps(False, "group commit off")
    arena.group_free(gf)                                           # meta 0 inside [0, hi): not simple5
    steps(False, "a free group")
    assert arena.group_alloc() == gf
    arena.group_set_conf(gf, 0x1f, 0, 0, 0, 1 << 20)
    arena.group_set_conf(g6, 0x1f, 0, 0, 2, 1 << 20)
    steps(True, "plain 5-voter again")
    w = arena.group_alloc_wide()
    with pytest.raises(B.RaftGpuError) as e:                      # the fused kernels evaluate 8-slot groups only
        arena.step_sorted_device(d_packed[0], 0, d_packed[1])
    assert e.value.status == B.ERR_INVALID
    B.pack_compact(np.zeros(0, dtype=B.APPEND_RESP_DTYPE), blob)           # a well-formed header
    with pytest.raises(B.RaftGpuError) as e:
        arena.step_compact_device(d_compact[0], blob, d_compact[1])
    assert e.value.status == B.ERR_INVALID
    arena.group_free(w)
    steps(False, "after the wide group")                          # free slots behind the stores' groups
    arena.close()
