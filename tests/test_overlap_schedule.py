"""The overlap schedules (tests/overlap_schedule.py) reach what tests/test_gpu_overlap.py is there to check: every call
kind with 0, 1 and 2 steps in flight and right after a wait that left one in flight, every step form, a call that moves
the commit index of a group the step in flight advanced, and a call that changes the launch plan between two steps in
flight.  In the plain 5-voter schedules every form also begins on the kSimple5 plan and off it, and the forms the fused
kernels take begin on the kSimple5 plan with a batch that tiles.  Oracle and the host packer only: no GPU."""
import numpy as np
import pytest

from helpers import B
import overlap_schedule as S


# the forms whose batch the fused kernels take when it tiles (the records API, its hybrid head, the compact and packed
# zero-copy forms, the wire form)
FUSED_FORMS = ("records_sorted", "hybrid", "compact", "packed", "wire")
SMALL = [s for s in S.SCHEDULES if s[2] < 100_000]


def _tileable(recs):
    blob = np.zeros(B.compact_bound(len(recs) + 64), np.uint8)
    B.pack_compact(recs, blob)
    return bool(blob[: B.COMPACT_HDR_DTYPE.itemsize].view(B.COMPACT_HDR_DTYPE)[0]["flags"] & B.COMPACT_TILEABLE)


def _two_on_a_cell(recs):
    main = recs[(recs["flags"] & B.REC_EXT) == 0]
    cells = main["group"].astype(np.int64) * 8 + main["peer_slot"]
    return len(np.unique(cells)) < len(cells)


@pytest.mark.parametrize("name,shape,n,seed,rounds,frac,window", SMALL, ids=[s[0] for s in SMALL])
def test_schedule_reaches_every_cell(name, shape, n, seed, rounds, frac, window):
    w = S.World(shape, n, seed)
    cells, forms, hits, plan_between = set(), set(), 0, 0
    plans, fused, ordered = set(), set(), 0
    events = list(S.schedule(S.Model(w, frac, window), rounds))
    for i, e in enumerate(events):
        if e.op == "call":
            cells.add((e.name, e.point))
            if e.point in ("1", "2", "1w"):
                hits += e.info["commit_hits"]
            # a call that changes the plan while one step is in flight, followed by the next begin
            if e.point in ("1", "1w") and e.info["plan_changed"]:
                nxt = next(x for x in events[i + 1:] if x.op != "call")
                plan_between += nxt.op == "begin"
        elif e.op == "begin":
            forms.add(e.name)
            assert e.want.n_advanced > 0, (name, e.name)
            plans.add((e.name, e.info["plan"]))
            if e.info["plan"] and e.name in FUSED_FORMS and _tileable(e.args["recs"]):
                fused.add(e.name)
                ordered += e.name == "records_sorted" and _two_on_a_cell(e.args["recs"])
    missing = {(k, p) for k in S.CALLS for p in S.POINTS} - cells
    assert not missing, sorted(missing)
    assert forms == set(S.FORMS)
    assert hits > 0
    if shape == "plain":
        assert plan_between > 0
        # every form begins on the kSimple5 plan and off it, and the fused forms on it with a batch that tiles (the
        # group-sorted records API with several records on a cell: the ordered kernel)
        assert plans == {(f, p) for f in S.FORMS for p in (True, False)}, sorted(plans)
        assert fused == set(FUSED_FORMS), sorted(fused)
        assert ordered > 0
    assert sum(e.op == "begin" for e in events) == sum(e.op == "wait" for e in events)


def test_the_long_schedule_covers_the_plans_at_1m():
    """plain_1m: the same coverage of plans and tiling as the small plain schedule (the calls are the same code)."""
    name, shape, n, seed, rounds, frac, window = next(s for s in S.SCHEDULES if s[0] == "plain_1m")
    w = S.World(shape, n, seed)
    plans, fused = set(), set()
    for e in S.schedule(S.Model(w, frac, window), rounds):
        if e.op == "begin":
            plans.add((e.name, e.info["plan"]))
            if e.info["plan"] and e.name in FUSED_FORMS and _tileable(e.args["recs"]):
                fused.add(e.name)
    assert plans == {(f, p) for f in S.FORMS for p in (True, False)}, sorted(plans)
    assert fused == set(FUSED_FORMS), sorted(fused)
