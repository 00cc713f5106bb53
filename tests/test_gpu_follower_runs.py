"""The follower's earlier term runs on the device (DESIGN 3.22): raftgpu_follower_append and
raftgpu_follower_append_entries on an arena with follower runs, both forms, against the batch oracle
(oracle/follower_runs_oracle.py) byte for byte -- statuses, from, appended records, responses, the table, the group
columns and the rows read back through raftgpu_follower_runs_get -- and the setter, the getter and their refusals."""
import numpy as np
import pytest

from helpers import B
from oracle import follower_runs_oracle as FR
import app_follow as A
import append_reject as R
import follower_runs as F
import hb_follow as FL
import pass_forms as PF

pytestmark = pytest.mark.gpu

WIDE_LO, WIDE_HI = 0x20000000, 0x40000000  # RAFTGPU_META_WIDE_LO / _HI


def _world(rng, n_narrow, n_wide):
    """Followers on an arena with follower runs: n_narrow groups then n_wide pairs (a pair's high half mirrors its low
    half's columns) -> (arena, followers, host columns, table, rows as the oracle keeps them, the pairs' low halves)."""
    n = n_narrow + 2 * n_wide
    f = F.Followers(rng, n)
    a = B.Arena(n + 64)
    a.enable_follower_runs()
    assert a.group_alloc_range(n_narrow) == 0
    lo = np.array([a.group_alloc_wide() for _ in range(n_wide)], np.int64)
    cols = {B.COL_TERM: f.groups["term"].copy(), B.COL_LAST_INDEX: f.groups["last_index"].copy(),
            B.COL_COMMITTED: f.groups["committed"].copy(), B.COL_TERM_START: np.full(n, A.NO_TERM_START, np.uint64)}
    for arr in cols.values():
        arr[lo + 1] = arr[lo]
    fi = np.where(rng.random(n) < 0.2, rng.integers(1, 8, n), 1)
    table, rows = f.state(2, fi, rng, stale=0.05)
    F.truncate(rng, f, table, 0.05)   # table runs emptied by a truncation, rows still anchored to them
    for k, arr in ((B.COL_LAST_INDEX, "last_index"), (B.COL_COMMITTED, "committed")):
        cols[k] = f.groups[arr].copy()
        cols[k][lo + 1] = cols[k][lo]
    rows[rng.random(n) < 0.1] = FR.row()          # no row stated
    rows["group"] = np.arange(n)
    for arr in (rows,):
        arr[lo + 1] = FR.row()
        arr["group"][lo + 1] = lo + 1
    table[lo + 1] = 0
    for col, arr in cols.items():
        a.column_write(col, 0, 0, np.ascontiguousarray(arr, np.uint64))
    low = np.setdiff1d(np.arange(n), lo + 1)
    st = a.follower_runs_set(rows[low])
    assert st.tolist() == [FR.row_status(r) for r in rows[low]]
    for g in low[st != 0]:  # refused (no row, or a stale anchor that breaks the order): not stored
        rows[g] = FR.row(g)
    c = a.read_columns(n)
    c.term = a.column_read(B.COL_TERM, 0, 0, n, np.uint64)
    return a, f, c, A.full_table(a, table), rows, lo


def _frames(rng, f, lo, per_group, entries):
    hi = set((lo + 1).tolist())
    kinds = ["match", "reject", "append", "append"] if entries else ["match", "reject"]
    frames = [A.frame(g, int(rng.integers(16)), F.probe(rng, f, g, kinds[int(rng.integers(0, len(kinds)))]))
              for _ in range(per_group) for g in range(f.n) if g not in hi]
    return [frames[i] for i in rng.permutation(len(frames))]


def _compare(a, c, blob, off, table, rows, entries, waves, device, what):
    want_table, n = table.copy(), c.n_groups
    want = FR.waves(c, None, want_table, rows, blob, off, entries, waves)
    name = "follower_append_entries" if entries else "follower_append"
    got = PF.run(a, name, blob, off, table, device=device)
    if entries:
        got = tuple(got[:2]) + (got[2].view(want[2].dtype),) + tuple(got[3:])
    else:
        want = want[:2] + want[3:]
    PF.equal(want, got, ("status", "from", "appended", "response bytes", "response offsets", "totals")[:len(want)]
             if entries else ("status", "from", "response bytes", "response offsets", "totals"), what)
    assert np.array_equal(table, want_table), (what, "table")
    assert np.array_equal(a.follower_runs_get(0, n), rows), (what, "rows")
    for k, col in FL.group_state(a, n).items():
        assert np.array_equal(col, getattr(c, k)[:n]), (what, k)
    return want


@pytest.mark.parametrize("waves", [1, 4])
@pytest.mark.parametrize("entries", [False, True], ids=["entry_less", "entries"])
@pytest.mark.parametrize("device", [True, False], ids=["device", "host"])
def test_device_matches_the_batch_oracle(device, entries, waves):
    """100K followers of 1-6 term runs with rows of up to two runs (some compacted, stale or missing), wide pairs:
    probes that match in every segment, rejections and (the entries pass) appends truncating into every segment, in
    two calls with rows restated between them.  Every output, the table, the columns and the rows equal the oracle's."""
    rng = np.random.default_rng(0xF0 + 2 * entries + waves + 8 * device)
    a, f, c, table, rows, lo = _world(rng, 99_000, 500)
    a.set_wire_waves(waves)
    per = 2 if waves > 1 else 1
    for call in range(2):
        blob, off = A.batch(_frames(rng, f, lo, per, entries))
        want = _compare(a, c, blob, off, table, rows, entries, waves, device, f"call {call}")
        decided = (want[0] >> 4 == B.WIRE_OK).sum()
        assert decided > len(off) // 3, decided
        # the host restates some rows (as after a truncation or a snapshot), others are dropped
        pick = rng.choice(np.setdiff1d(np.arange(c.n_groups), lo + 1), 2000, replace=False)
        new = rows[pick].copy()
        new[: 1000] = [FR.row(int(g)) for g in pick[:1000]]
        new["anchor_start"][:1000], new["anchor_term"][:1000] = 7, 3
        st = a.follower_runs_set(new)
        rows[pick[st == 0]] = new[st == 0]


def test_alloc_and_free_clear_rows_and_the_refusals():
    """Group alloc and free clear a row; enable after alloc, and set or get on an arena without follower runs, are
    refused; the setter's statuses are the oracle's row check."""
    a = B.Arena(64)
    a.enable_follower_runs()
    assert a.group_alloc_range(8) == 0
    r = FR.row(3, 20, 9, [(10, 5), (4, 2)])
    assert a.follower_runs_set(np.array([r], FR.ROW_DTYPE)).tolist() == [0]
    assert a.follower_runs_get(3, 1)[0] == r
    a.group_free(3)
    assert a.follower_runs_get(3, 1)[0] == FR.row(3)
    assert a.follower_runs_set(np.array([r], FR.ROW_DTYPE)).tolist() == [B.ERR_RANGE]
    g = a.group_alloc()
    r["group"] = g
    assert a.follower_runs_set(np.array([r], FR.ROW_DTYPE)).tolist() == [0]
    a.group_free(g)
    g2 = a.group_alloc()
    assert a.follower_runs_get(g2, 1)[0] == FR.row(g2)
    bad = [FR.row(0, 20, 0), FR.row(1, 0, 9), FR.row(2, A.NO_TERM_START, 9), FR.row(4, 20, 9, [(0, 0), (4, 2)]),
           FR.row(5, 20, 9, [(20, 5)]), FR.row(6, 20, 9, [(10, 5), (12, 2)]), FR.row(7, 20, 9, [(10, 9)]),
           FR.row(0, 20, 9, [(10, 5), (4, 5)]), FR.row(40, 20, 9)]
    st = a.follower_runs_set(np.array(bad, FR.ROW_DTYPE))
    assert st.tolist() == [FR.row_status(x, allocated=int(x["group"]) < 8) for x in bad]
    assert a._L.raftgpu_follower_runs_get(a._h, 1 << 31, 1, np.zeros(1, FR.ROW_DTYPE).ctypes.data) == B.ERR_RANGE
    assert a._L.raftgpu_arena_enable_follower_runs(a._h) == B.ERR_INVALID  # already enabled
    b = B.Arena(16)
    assert b.group_alloc_range(2) == 0
    assert b._L.raftgpu_arena_enable_follower_runs(b._h) == B.ERR_INVALID  # after alloc
    rows = np.array([FR.row(0, 20, 9)], FR.ROW_DTYPE)
    st = np.zeros(1, np.int32)
    assert b._L.raftgpu_follower_runs_set(b._h, rows.ctypes.data, 1, st.ctypes.data) == B.ERR_INVALID
    assert b._L.raftgpu_follower_runs_get(b._h, 0, 1, rows.ctypes.data) == B.ERR_INVALID


def _leader(c, n, rows):
    a = R.leader_arena(c, n, True)
    assert not a.leader_runs_set(rows).any()
    return a


def _follower(c, n, runs, rows):
    a = B.Arena(n)
    if runs:
        a.enable_follower_runs()
    assert a.group_alloc_range(n) == 0
    for col, name in ((B.COL_TERM, "term"), (B.COL_LAST_INDEX, "last_index"), (B.COL_COMMITTED, "committed"),
                      (B.COL_TERM_START, "term_start")):
        a.column_write(col, 0, 0, getattr(c, name)[:n].copy())
    if runs:
        assert not a.follower_runs_set(rows).any()
    return a


@pytest.mark.parametrize("follower_runs", [True, False], ids=["follower_runs", "no_follower_runs"])
def test_election_round_trip_with_runs_at_both_ends_100k_x5(follower_runs):
    """100K groups x 5 peers after a store-wide election (follower_runs.Dialogue): leaders with their last two earlier
    runs stated, followers that hold their leader's log into its last or second-last earlier run and may carry a
    divergent tail.  Probe -> raftgpu_follower_append_entries (host form, one follower arena per slot) ->
    raftgpu_step_begin_wire, round after round, each call equal to the oracle's, the follower rows the device
    re-anchored read back every round, the rows of host-stepped followers restated, until every follower's log is its
    leader's.  With follower runs no frame goes to the host at either end; without them the count is reported."""
    d = F.Dialogue(np.random.default_rng(0xE1EC), 100_000, follower_runs, device=(_leader, _follower))
    d.run(PF)
    print(f"\nelection round trip, follower runs {'on' if follower_runs else 'off'}: {d.rounds} rounds, "
          f"{d.host_follower} frames stepped on the host at the followers, {d.host_leader} at the leaders")
    if follower_runs:
        assert (d.host_follower, d.host_leader) == (0, 0)
    else:
        assert d.host_follower > 0
    d.la.close()
    for s in d.slots:
        s["a"].close()
