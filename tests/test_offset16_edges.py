"""The 16-bit offset window of next_idx and peer_committed on the CPU, against the C oracle.

The edge generators of offset16.py must really move both fields across both bounds of the window, both ways, and
land them exactly on the bounds -- through the records the fused fast path takes as well as through the others --
for the GPU tests that run on them (test_gpu_offset16_edges.py) to mean anything.  And the benchmark's own streams
must never leave the window: a cell that escapes takes the general path, so a benchmark whose cells escaped would be
timing the slow path."""
import importlib

import numpy as np
import pytest

from helpers import O, TILE_SHAPES, offset_of, random_state
from offset16 import (I16_MAX, I16_MIN, K_LOCAL_JUMP, K_PROBE_REJECT, edge_batch, edge_state16, escaped16, fits16)

B = importlib.import_module("raft-rs_b200").binding
FLOOR = 50


def transitions(before, after, field, n):
    mb, ma = before.matched[:, :n], after.matched[:, :n]
    vb, va = getattr(before, field)[:, :n], getattr(after, field)[:, :n]
    fb, fa = fits16(vb, mb), fits16(va, ma)
    moved = (mb != ma) | (vb != va)
    d = offset_of(va, ma)
    return {"to escape": fb & ~fa, "back": ~fb & fa, "escaped, new value": ~fb & ~fa & (vb != va),
            "at INT16_MAX": moved & (d == I16_MAX), "at INT16_MIN + 1": moved & (d == I16_MIN + 1),
            "at INT16_MIN": moved & (d == I16_MIN)}


def test_edge_state16_covers_every_kind_of_cell():
    shape, hint = TILE_SHAPES["sparse_a"][:2]
    n = 20_000
    rng = np.random.default_rng(13)
    c = random_state(n, shape, rng)
    before = O.copy_columns(c)
    edge_state16(c, rng, n=n)
    m = c.matched[:, :n]
    moved = (c.next_idx[:, :n] != before.next_idx[:, :n]) | (m != before.matched[:, :n])
    meta = c.meta[:n].astype(np.int64)
    slot = np.arange(O.SLOTS)[:, None]
    learner = ((meta >> 16) >> slot) & 1 == 1
    is_self = ((meta & O.META_HAS_SELF) != 0) & (((meta >> 24) & 7) == slot)
    hinted = ((hint >> slot) & 1 == 1) & np.ones((1, n), dtype=bool)
    snapshot = (c.pflags[:, :n] & O.PF_STATE_MASK) == O.STATE_SNAPSHOT
    for what, sel in (("hinted slots", hinted), ("learners outside the hint", learner & ~hinted),
                      ("self slots", is_self), ("Snapshot-state peers", snapshot)):
        assert np.count_nonzero(moved & sel) >= FLOOR, what
        for field in ("next_idx", "peer_committed"):
            d = offset_of(getattr(c, field)[:, :n], m)
            for want in (0, 1, -1, I16_MAX, I16_MIN + 1, I16_MAX + 1, I16_MIN, I16_MIN - 1):
                assert np.count_nonzero(moved & sel & (d == want)) >= 5, (what, field, want)
    reset = (m == 0) & (before.matched[:, :n] != 0)
    assert np.count_nonzero(reset & ~fits16(c.next_idx[:, :n], 0)) >= FLOOR
    assert np.count_nonzero(reset & fits16(c.next_idx[:, :n], 0)) >= FLOOR     # last_index 2^15 - 2


def test_edge16_batches_cross_both_bounds_both_ways():
    """Per round, per field: cells that escape, return, stay escaped with a new value, or end exactly at INT16_MAX,
    INT16_MIN + 1 or INT16_MIN (the escape code's own value); and the same classes reached by the records the fused
    fast path takes (LOCAL jumps, hinted Probe rejections) from cells that fit."""
    rng = np.random.default_rng(15)
    n = 20_000
    for name in ("any8", "sparse_a", "v5_simple"):
        c = random_state(n, TILE_SHAPES[name][0], rng)
        edge_state16(c, rng, n=n, escape_groups=(np.arange(n) // 512) % 9 == 4)
        for rnd in range(4):
            per_cell = 3 if rnd == 3 else 1
            before = O.copy_columns(c)
            recs, kinds = edge_batch(c, rng, per_cell, with_kinds=True)
            O.arena_apply(c, recs, mode=0)
            O.arena_recompute(c)
            main = (recs["flags"] & O.REC_EXT) == 0
            sel = main & np.isin(kinds, (K_LOCAL_JUMP, K_PROBE_REJECT))
            gs, ss = recs["group"][sel], recs["peer_slot"][sel]
            fit_before = fits16(before.next_idx[ss, gs], before.matched[ss, gs]) & \
                fits16(before.peer_committed[ss, gs], before.matched[ss, gs])
            fast_cells = np.zeros((O.SLOTS, n), dtype=bool)
            fast_cells[ss[fit_before], gs[fit_before]] = True
            for field in ("next_idx", "peer_committed"):
                for what, cells in transitions(before, c, field, n).items():
                    got = np.count_nonzero(cells)
                    assert got >= FLOOR, f"{name}, round {rnd}, {field}: {got} cells {what}"
                    if per_cell == 1 and what in ("to escape", "at INT16_MIN + 1", "at INT16_MIN"):
                        got = np.count_nonzero(cells & fast_cells)
                        assert got >= FLOOR, f"{name}, round {rnd}, {field}, fast path: {got} cells {what}"


def test_self_update_reaches_the_upper_bound():
    """offset16.self_behind16 puts the leader's own cell 2^15 - 1, 2^15 and 2^15 + 1 below the index the group
    commits: the recompute (hot_update_committed) lands peer_committed on the bound and past it."""
    from offset16 import self_behind16
    n = 20_000
    rng = np.random.default_rng(17)
    c = random_state(n, TILE_SHAPES["v5_simple"][0], rng)
    chosen = self_behind16(c, rng, n)
    O.arena_recompute(c)
    g = np.flatnonzero(chosen)
    own = (c.meta[g].astype(np.int64) >> 24) & 7
    d = offset_of(c.peer_committed[own, g], c.matched[own, g])
    for want in (I16_MAX, I16_MAX + 1, I16_MAX + 2):
        assert np.count_nonzero(d == want) > 50, want


# --------------------------------------------------------------------------- the benchmark's streams

# bench.py's workloads (groups reduced) and the most rounds one of its arenas sees: the e2e arena takes about 400
# rounds over its three legs at --steps 100; 480 leaves room.
BENCH_STREAMS = {"cfg2": (5, False, 0x5EED0002), "cfg3": (5, False, 0x5EED0003),
                 "cfg4": (5, True, 0x5EED0004), "cfg5": (5, False, 0x5EED0005)}
ROUNDS = 480


@pytest.mark.parametrize("workload", sorted(BENCH_STREAMS))
def test_bench_streams_stay_inside_the_16bit_window(workload):
    k_peers, joint, seed = BENCH_STREAMS[workload]
    n = 4096
    for a in (0, 1):                          # the first two device-leg arenas (seed + 0x100 * a); a = 0 is the e2e arena's seed
        s = B.Synth(n, seed + 0x100 * a, k_peers=k_peers, joint=joint)
        c = O.copy_columns(s.initial)
        assert not escaped16(c, n).any(), (workload, a, "initial state")
        worst_nx = worst_pc = 0
        for rnd in range(ROUNDS):
            O.arena_apply(c, s.next_round().copy(), mode=0)
            O.arena_recompute(c)
            esc = escaped16(c, n)
            assert not esc.any(), f"{workload}, arena {a}, round {rnd}: {np.count_nonzero(esc)} cells escape"
            m = c.matched[:, :n]
            worst_nx = max(worst_nx, int(np.abs(offset_of(c.next_idx[:, :n], m)).max()))
            worst_pc = max(worst_pc, int(np.abs(offset_of(c.peer_committed[:, :n], m)).max()))
        # the margin left: a lagging follower's peer_committed - matched grows by some 19 entries a round, so a
        # stream this long stays within half the window (the first cells escape after about 1900 rounds; DESIGN 2)
        assert worst_nx < I16_MAX // 2 and worst_pc < I16_MAX // 2, (workload, worst_nx, worst_pc)
