"""The edge generators of helpers.py (edge_state, random_batch(edge=True)) against the C oracle, on the CPU: the
states and batches the offset-edge GPU tests run on must really move next_idx and peer_committed across both
bounds of the 32-bit offset window, both ways, and land them exactly on the bounds -- through the records the
fused fast path takes as well as through the others."""
import numpy as np

from helpers import (I32_MAX, I32_MIN, K_LOCAL_JUMP, K_PROBE_REJECT, O, TILE_SHAPES, edge_state, fits, offset_of,
                     random_batch, random_state)

FLOOR = 50


def transitions(before, after, field, n):
    """Counts of the transition classes of one field over the cells whose matched or value changed."""
    mb, ma = before.matched[:, :n], after.matched[:, :n]
    vb, va = getattr(before, field)[:, :n], getattr(after, field)[:, :n]
    fb, fa = fits(vb, mb), fits(va, ma)
    moved = (mb != ma) | (vb != va)
    d = offset_of(va, ma)
    return {"to escape": fb & ~fa, "back": ~fb & fa, "escaped, new value": ~fb & ~fa & (vb != va),
            "at INT32_MAX": moved & (d == I32_MAX), "at INT32_MIN + 1": moved & (d == I32_MIN + 1),
            "at INT32_MIN": moved & (d == I32_MIN)}


def test_edge_state_covers_every_kind_of_cell():
    shape, hint = TILE_SHAPES["sparse_a"][:2]
    n = 20_000
    rng = np.random.default_rng(3)
    c = random_state(n, shape, rng)
    before = O.copy_columns(c)
    edge_state(c, rng, n=n)
    moved = (c.next_idx[:, :n] != before.next_idx[:, :n]) | (c.matched[:, :n] != before.matched[:, :n])
    meta = c.meta[:n].astype(np.int64)
    slot = np.arange(O.SLOTS)[:, None]
    learner = ((meta >> 16) >> slot) & 1 == 1
    is_self = ((meta & O.META_HAS_SELF) != 0) & (((meta >> 24) & 7) == slot)
    hinted = ((hint >> slot) & 1 == 1) & np.ones((1, n), dtype=bool)
    snapshot = (c.pflags[:, :n] & O.PF_STATE_MASK) == O.STATE_SNAPSHOT
    for what, sel in (("hinted slots", hinted), ("learners outside the hint", learner & ~hinted),
                      ("self slots", is_self), ("self slots outside the hint", is_self & ~hinted),
                      ("Snapshot-state peers", snapshot)):
        assert np.count_nonzero(moved & sel) >= FLOOR, what
        for field in ("next_idx", "peer_committed"):
            v = getattr(c, field)[:, :n]
            assert np.count_nonzero(moved & sel & ~fits(v, c.matched[:, :n])) >= FLOOR, (what, field)
    reset = (c.matched[:, :n] == 0) & (before.matched[:, :n] != 0)
    assert np.count_nonzero(reset & ~fits(c.next_idx[:, :n], 0)) >= FLOOR
    assert np.count_nonzero(reset & fits(c.next_idx[:, :n], 0)) >= FLOOR      # last_index 2^31 - 2


def test_edge_batches_cross_both_bounds_both_ways():
    """Per round, per field: cells that escape, return, stay escaped with a new value, or end exactly at
    INT32_MAX, INT32_MIN + 1 or INT32_MIN (the escape code's own value).  Then the same classes reached by the
    records the fused fast path takes (LOCAL jumps, hinted Probe rejections) from cells that fit."""
    rng = np.random.default_rng(5)
    n = 20_000
    for name in ("any8", "sparse_a", "v5_simple"):
        c = random_state(n, TILE_SHAPES[name][0], rng)
        edge_state(c, rng, n=n, escape_groups=(np.arange(n) // 512) % 9 == 4)
        for rnd in range(4):
            per_cell = 3 if rnd == 3 else 1
            before = O.copy_columns(c)
            recs, kinds = random_batch(c, rng, per_cell, edge=True, with_kinds=True)
            O.arena_apply(c, recs, mode=0)
            O.arena_recompute(c)
            main = (recs["flags"] & O.REC_EXT) == 0
            fast_cells = np.zeros((O.SLOTS, n), dtype=bool)
            sel = main & np.isin(kinds, (K_LOCAL_JUMP, K_PROBE_REJECT))
            gs, ss = recs["group"][sel], recs["peer_slot"][sel]
            fit_before = fits(before.next_idx[ss, gs], before.matched[ss, gs]) & \
                fits(before.peer_committed[ss, gs], before.matched[ss, gs])
            fast_cells[ss[fit_before], gs[fit_before]] = True
            for field in ("next_idx", "peer_committed"):
                for what, cells in transitions(before, c, field, n).items():
                    got = np.count_nonzero(cells)
                    assert got >= FLOOR, f"{name}, round {rnd}, {field}: {got} cells {what}"
                    if per_cell == 1 and what in ("to escape", "at INT32_MIN + 1", "at INT32_MIN"):
                        # the fast-path records start from cells that fit and land them at the lower bound
                        got = np.count_nonzero(cells & fast_cells)
                        assert got >= FLOOR, f"{name}, round {rnd}, {field}, fast path: {got} cells {what}"
