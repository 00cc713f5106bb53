"""Every kernel that reads or writes next_idx and peer_committed, at the edges of their 32-bit offset window.

On the device both are int32 offsets from the cell's matched, with an escape code for the values outside
(INT32_MIN, INT32_MAX] (k_common.cuh).  These tests put cells exactly on either side of both bounds, escape them
and bring them back -- through the fused kernels' fast and general paths, the scatter kernel and the paths the
library picks, the recompute's self update, heartbeat responses, update_state and the send lists, and the control
lists -- and compare everything with the oracle after every round.  The generators are in helpers.py; that they
reach every transition is checked on the CPU by test_offset_edges.py.  Run with -m gpu."""
import importlib

import numpy as np
import pytest

from oracle import control_oracle as CO
from helpers import (B, EDGE_ESCAPES, EDGE_FITS, I32_MAX, I32_MIN, O, RESET_LAST, TILE_SHAPES, Paths, Shape,
                     assert_columns_equal, bitmap_to_bool, edge_state, escaped_cells, fits, offset_of,
                     random_batch, random_state, ring_wrapping_groups)
from control_cmds import cmds
from test_gpu_control import records_step
from test_gpu_wire import oracle_wire_step

pytestmark = pytest.mark.gpu

W = importlib.import_module("raft-rs_b200.wire")
EDGE_D = np.array(EDGE_FITS + EDGE_ESCAPES)


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


# --------------------------------------------------------------------------- the fused kernels

def run_fused(name, n, monkeypatch, rounds=3, storm_rounds=1):
    shape, _, force_general, seed = TILE_SHAPES[name]
    if force_general:
        monkeypatch.setenv("RAFTGPU_FORCE_GENERAL", "1")     # read when an arena is created
    else:
        monkeypatch.delenv("RAFTGPU_FORCE_GENERAL", raising=False)
    rng = np.random.default_rng(seed + 1000)
    init = edge_state(random_state(n, shape, rng), rng, escape_groups=escape_tiles(n))
    paths = Paths(n, init, records_api=False)
    results = []
    for rnd in range(rounds + 1):
        per_cell = 3 if rnd == rounds else 1
        recs = random_batch(paths.refs["ordered"], rng, per_cell, edge=True)
        results.append(paths.round(recs, per_cell, f"{name}, edge round {rnd}"))
    paths.reload(storm(O.copy_columns(paths.refs["ordered"]), rng, n))
    for rnd in range(storm_rounds):
        recs = random_batch(paths.refs["ordered"], rng, 1, edge=True)
        results.append(paths.round(recs, 1, f"{name}, after an election at a high index, round {rnd}"))
    assert escaped_cells(paths.refs["ordered"]).any()
    paths.close()
    return results


@pytest.mark.parametrize("name", ["sparse_a", "any8"])
def test_fused_kernels_at_the_offset_edges(name, monkeypatch):
    run_fused(name, several_tiles(), monkeypatch)


def test_simple5_and_general_fused_kernels_at_the_offset_edges(monkeypatch):
    """The same edge state and batches through the kSimple5 instantiation and, with RAFTGPU_FORCE_GENERAL, the
    general one: both match the oracle, and each other record for record."""
    n = several_tiles()
    simple = run_fused("v5_simple", n, monkeypatch)
    general = run_fused("v5_general", n, monkeypatch)
    for i, (a, b) in enumerate(zip(simple, general)):
        for path in a:
            assert np.array_equal(a[path], b[path]), (i, path)


def test_fused_kernels_at_the_offset_edges_where_the_ring_wraps(monkeypatch):
    run_fused("any8", ring_wrapping_groups(), monkeypatch, rounds=1, storm_rounds=1)


# --------------------------------------------------------------------------- the recompute's self update

def self_behind(c, rng, n, frac=0.5):
    """Groups whose leader's matched lies 2^31 - 1, 2^31 or 2^31 + 1 below the index every other voter has
    acknowledged (and the group can commit): the recompute raises the leader's peer_committed to it."""
    meta = c.meta[:n].astype(np.int64)
    has = ((meta & O.META_HAS_SELF) != 0) & (c.term_start[:n] != O.U64_MAX) & (rng.random(n) < frac)
    own = (meta >> 24) & 7
    x = c.last_index[:n].astype(np.int64) + (1 << 33)
    gap = np.array([I32_MAX, I32_MAX + 1, I32_MAX + 2])[rng.integers(0, 3, n)]
    g = np.flatnonzero(has)
    c.matched[:, g] = x[g]
    c.next_idx[:, g] = x[g] + 1
    c.peer_committed[:, g] = x[g] - 3
    c.matched[own[g], g] = x[g] - gap[g]
    c.next_idx[own[g], g] = x[g] - gap[g] + 1
    c.peer_committed[own[g], g] = x[g] - gap[g]
    c.committed[g] = x[g] - 10
    c.term_start[g] = x[g] - 20
    c.last_index[g] = x[g] + 5
    return has


@pytest.mark.parametrize("name", ["v5_simple", "sparse_a"])
def test_recompute_moves_the_leaders_peer_committed_across_the_bound(name, monkeypatch):
    """The self slot hinted (v5) and, in sparse_a, also a learner outside the hint: the fused kernels' self update
    (TileRing::finish) and the scatter path's recompute, each against the oracle."""
    monkeypatch.delenv("RAFTGPU_FORCE_GENERAL", raising=False)
    shape, hint, _, seed = TILE_SHAPES[name]
    n = several_tiles()
    rng = np.random.default_rng(seed + 2000)
    init = random_state(n, shape, rng)
    chosen = self_behind(init, rng, n)
    paths = Paths(n, init, records_api=True)
    scatter = B.Arena(n)
    assert scatter.group_alloc_range(n) == 0
    scatter.load_columns(init)
    sref = O.copy_columns(init)
    recs = random_batch(paths.refs["ordered"], rng, 1, keep=~chosen)
    paths.round(recs, 1, f"{name}, self update")
    scatter.enqueue(recs)
    r = scatter.step(B.STEP_READ_COMMITTED)
    O.arena_apply(sref, recs, mode=0)
    want_adv, want_bm, _, _ = O.arena_recompute(sref)
    assert r.n_advanced == want_adv
    assert np.array_equal(scatter.step_results(n)[0], want_bm[: (n + 31) // 32])
    assert_columns_equal(scatter.read_columns(n), sref, n, f"{name}, scatter self update")
    ref = paths.refs["ordered"]
    meta = ref.meta[:n].astype(np.int64)
    g = np.flatnonzero(chosen)
    own = (meta[g] >> 24) & 7
    d = offset_of(ref.peer_committed[own, g], ref.matched[own, g])
    outside = ((hint >> own) & 1) == 0
    for want in (I32_MAX, I32_MAX + 1, I32_MAX + 2):
        assert np.count_nonzero(d == want) > 50, want
        if name == "sparse_a":
            assert np.count_nonzero((d == want) & outside) > 10, want
    paths.close()
    scatter.close()


# --------------------------------------------------------------------------- the scatter kernel and the library's paths

N_NARROW, N_WIDE = 6000, 8


def wide_arena(rng, inflights):
    """An arena of narrow groups in the edge state and wide groups (two slots each) with escaped cells, and its
    oracle copy."""
    init = random_state(N_NARROW, Shape(group_commit=True), rng)
    if inflights:
        init.pflags &= np.uint8(~O.PF_INS_FULL & 0xFF)   # the windows start empty: not full
    a = B.Arena(32 * (N_NARROW + 2 * N_WIDE))       # room for the scatter kernel's later waves
    if inflights:
        a.enable_inflights(8)
    assert a.group_alloc_range(N_NARROW) == 0
    a.load_columns(init)
    for k in range(N_WIDE):
        g = a.group_alloc_wide()
        li = int(rng.integers(1 << 31, 1 << 40))
        a.group_set_conf(g, int(rng.integers(1, 1 << 16)), int(rng.integers(0, 1 << 16)) if k % 2 else 0,
                         int(rng.integers(0, 1 << 16)), int(rng.integers(0, 16)), li)
        a.group_reset(g, li - 3, li, li - 5, li)
    n = N_NARROW + 2 * N_WIDE
    ref = a.read_columns(n)
    ref.n_groups = n
    edge_state(ref, rng, n=N_NARROW)
    a.load_columns(ref)
    if inflights:
        O.enable_inflights(ref, 8)
    return a, ref, n


@pytest.mark.parametrize("inflights", [False, True], ids=["no_windows", "inflights"])
def test_scatter_and_library_paths_at_the_offset_edges(inflights, monkeypatch):
    rng = np.random.default_rng(0x0FF5 + inflights)
    a, ref, n = wide_arena(rng, inflights)
    assert escaped_cells(ref).sum() > n
    buf = a.host_alloc_bytes(24 * (8 * 3 * n + 64)).view(B.APPEND_RESP_DTYPE)      # pinned: RAW and HYBRID
    wb = W.WireBuffers(a, 8 * n + 64)
    for rnd, how in enumerate(["enqueue", "records", "raw", "hybrid", "wire", "enqueue3"]):
        recs = random_batch(ref, rng, 3 if how == "enqueue3" else 1, edge=True)
        what = f"{how}, round {rnd}"
        if how in ("enqueue", "enqueue3"):                     # several records per cell: the scatter waves
            a.enqueue(recs)
            r = a.step(B.STEP_READ_COMMITTED)
        elif how == "records":
            records_step(a, n, recs, ref, what)      # wide groups: the library takes the scatter kernel
            continue
        elif how == "wire":
            wb.encode(recs)
            a.step_begin_wire(wb, B.STEP_READ_COMMITTED)
            r = a.step_wait()
            want, want_bm, want_adv, _ = oracle_wire_step(ref, wb, n, None)
            assert np.array_equal(a.wire_status(), want), what
            assert r.n_advanced == want_adv, what
            assert np.array_equal(a.step_results(n)[0], want_bm[: (n + 31) // 32]), what
            assert_columns_equal(a.read_columns(n), ref, n, what)
            continue
        else:
            buf[: len(recs)] = recs
            flags = B.STEP_READ_COMMITTED | (B.STEP_RAW if how == "raw" else B.STEP_HYBRID)
            if how == "hybrid":
                monkeypatch.setenv("RAFTGPU_HYBRID_PACK_PCT", "50")
            a.step_begin_records(buf[: len(recs)], flags)
            r = a.step_wait()
        O.arena_apply(ref, recs, mode=0)
        want_adv, want_bm, _, _ = O.arena_recompute(ref)
        assert r.n_advanced == want_adv and r.n_duplicates == 0, what
        bm, com = a.step_results(n)
        assert np.array_equal(bm, want_bm[: len(bm)]), what
        adv = bitmap_to_bool(bm, n)
        assert np.array_equal(com[adv], ref.committed[:n][adv]), what
        assert_columns_equal(a.read_columns(n), ref, n, what)
    wb.free()
    a.close()


# --------------------------------------------------------------------------- heartbeat responses

def heartbeat_records(ref, rng, n):
    """One REC_HEARTBEAT record per present cell of a random half of the cells: commits 2^31 - 1 and 2^31 above
    matched, near last_index for the peers in the reset shape, and small ones below (escaped cells must keep
    their exact values)."""
    g, s = np.nonzero((rng.random((n, O.SLOTS)) < 0.5))
    m = ref.matched[s, g].astype(np.int64)
    li = ref.last_index[g].astype(np.int64)
    nx = ref.next_idx[s, g].astype(np.int64)
    kind = rng.integers(0, 4, len(g))
    up = m + np.array([I32_MAX, I32_MAX + 1])[rng.integers(0, 2, len(g))]
    near = np.where(m == 0, np.maximum(nx - 1, 0) + rng.integers(-2, 3, len(g)), li - rng.integers(0, 3, len(g)))
    commit = np.select([kind == 0, kind == 1, kind == 2], [up, near, np.maximum(0, m - rng.integers(0, 5, len(g)))],
                       m + rng.integers(0, 5, len(g)))
    recs = np.zeros(len(g), dtype=B.APPEND_RESP_DTYPE)
    recs["group"], recs["peer_slot"], recs["flags"] = g, s, B.REC_HEARTBEAT
    recs["commit"] = np.maximum(commit, 0)
    return recs


def test_heartbeat_responses_at_the_offset_edges():
    """raftgpu_heartbeat_resp and the tracker part of raftgpu_heartbeat_wire on the edge state, then after an
    election at a high index, against ro_arena_apply_heartbeat."""
    n = 20_000
    rng = np.random.default_rng(0x4EA7)
    init = edge_state(random_state(n, Shape(group_commit=True), rng), rng)
    arenas = {}
    for name in ("resp", "wire"):
        a = B.Arena(n)
        assert a.group_alloc_range(n) == 0
        a.load_columns(init)
        arenas[name] = (a, O.copy_columns(init))
    wa = arenas["wire"][0]
    wb = W.WireBuffers(wa, 8 * n + 64, bytes_per_record=32)
    for rnd in range(3):
        if rnd == 2:
            for a, ref in arenas.values():
                storm(ref, rng, n)
                a.load_columns(ref)
        for name, (a, ref) in arenas.items():
            recs = heartbeat_records(ref, rng, n)
            before = O.copy_columns(ref)
            want = O.arena_apply_heartbeat(ref, recs)
            if name == "resp":
                got = a.heartbeat_resp(recs)
                assert np.array_equal(got, want), rnd
            else:
                st, _ = a.heartbeat_wire(wb.encode_heartbeats(recs))
                assert np.array_equal(st & 0xF, want), rnd
                assert (st >> 4 == B.WIRE_OK).all()
            assert_columns_equal(a.read_columns(n), ref, n, f"heartbeat {name}, round {rnd}")
            if rnd == 2:
                continue
            pc0, pc1 = before.peer_committed[:, :n], ref.peer_committed[:, :n]
            m = ref.matched[:, :n]
            assert np.count_nonzero(fits(pc0, m) & ~fits(pc1, m)) > 100
            assert np.count_nonzero(offset_of(pc1, m)[pc0 != pc1] == I32_MAX) > 100
    wb.free()
    for a, _ in arenas.values():
        a.close()


# --------------------------------------------------------------------------- update_state and the send lists

def as_set(e):
    return sorted(zip(e["group"].tolist(), e["peer_slot"].tolist(), e["flags"].tolist(), e["next_idx"].tolist()))


def test_update_state_and_send_lists_at_the_offset_edges():
    """update_state with last + 1 at each distance from matched, then the send list (bcast_append, and after a step
    over its advanced groups) and the heartbeat commits over escaped cells, as sets against the oracle."""
    n = 20_000
    rng = np.random.default_rng(0x5E4D)
    init = edge_state(random_state(n, Shape(group_commit=True), rng), rng, frac=0.5)
    a = B.Arena(n)
    assert a.group_alloc_range(n) == 0
    a.load_columns(init)
    ref = O.copy_columns(init)
    d_out, d_cnt = a.device_alloc(16 * 8 * n), a.device_alloc(8)
    cnt = np.zeros(1, dtype=np.uint64)

    def send_list():
        a.send_list_device(0, n, None, d_out, 8 * n, d_cnt)
        a.d2h(cnt, d_cnt)
        got = np.zeros(int(cnt[0]), dtype=B.SEND_ENTRY_DTYPE)
        a.d2h(got, d_out)
        want = O.arena_send_list(ref)
        assert as_set(got) == as_set(want)
        return want

    d_hb = a.device_alloc(8 * 8 * n)
    for rnd in range(2):
        entries = send_list()
        assert len(entries) > n // 2
        m = ref.matched[entries["peer_slot"], entries["group"]].astype(np.int64)
        last = m + EDGE_D[rng.integers(0, len(EDGE_D), len(entries))] - 1
        entries["next_idx"] = np.where(last < 0, m, last)
        got = a.update_state(entries)
        want = O.arena_update_state(ref, entries)
        assert np.array_equal(got, want), rnd
        assert_columns_equal(a.read_columns(n), ref, n, f"update_state, round {rnd}")
        nx = ref.next_idx[entries["peer_slot"], entries["group"]]
        sent = offset_of(nx, ref.matched[entries["peer_slot"], entries["group"]])
        for d in (I32_MAX, I32_MIN + 1):
            assert np.count_nonzero(sent == d) > 20, d
        assert np.count_nonzero(~fits(nx, ref.matched[entries["peer_slot"], entries["group"]])) > 200
        a.heartbeat_commits_device(0, n, d_hb)
        hb = np.zeros((8, n), dtype=np.uint64)
        a.d2h(hb, d_hb)
        assert np.array_equal(hb, O.arena_heartbeat_commits(ref, 0, n))
        recs = random_batch(ref, rng, 1, edge=True)
        a.enqueue(recs)
        a.step(0)
        O.arena_apply(ref, recs, mode=0)
        _, want_bm, _, _ = O.arena_recompute(ref)
        got = a.step_send_list(8 * n)
        assert as_set(got) == as_set(O.arena_send_list(ref, want_bm)), rnd
    a.close()


# --------------------------------------------------------------------------- control lists

def test_control_lists_at_the_offset_edges():
    """Every Progress method with its arguments at the bounds, SET_CONF adding peers at next_idx near 2^40, RESET at
    last indexes around 2^31, BECOME_LEADER; every column and result against ro_arena_control, then a records step."""
    n = 6000
    rng = np.random.default_rng(0xC0DE)
    init = edge_state(random_state(n, Shape(group_commit=True), rng), rng)
    a = B.Arena(n)
    assert a.group_alloc_range(n) == 0
    a.load_columns(init)
    ref = O.copy_columns(init)
    votes = np.zeros((O.SLOTS, n), dtype=np.uint8)
    rows = []
    for g in rng.permutation(n)[: n // 2]:
        g = int(g)
        meta = int(ref.meta[g])
        present = [s for s in range(8) if (meta | meta >> 8 | meta >> 16) >> s & 1]
        r = rng.random()
        if r < 0.6:
            for _ in range(int(rng.integers(1, 4))):
                s = int(rng.choice(present))
                m, nx = int(ref.matched[s, g]), int(ref.next_idx[s, g])

                def at(base):
                    v = base + int(EDGE_D[rng.integers(0, len(EDGE_D))])
                    return v if v >= 0 else base
                op = int(rng.integers(0, 14))
                x = [at(m), at(m), 0]
                if op == B.POP_MAYBE_DECR_TO:
                    x = [nx - 1 if rng.random() < 0.6 and nx else at(m), at(m) - 1 if m else 0,
                         0 if rng.random() < 0.8 else at(m)]
                rows.append((B.CTL_PROGRESS_OP, g, s, op, [max(v, 0) for v in x]))
        elif r < 0.75:
            inc = (meta & 0xff) | int(rng.integers(0, 256)) & ~((meta >> 16) & 0xff)
            self_slot = (meta >> 24) & 7 if meta & O.META_HAS_SELF else B.CTL_NO_SELF
            rows.append((B.CTL_SET_CONF, g, self_slot, 0, (inc, (meta >> 8) & 0xff, 0,
                                                           (1 << 40) + int(rng.integers(-3, 4)))))
        elif r < 0.9:
            li = (1 << 31) + int(rng.integers(-2, 2))
            rows.append((B.CTL_RESET, g, 0, 0, (li - 1, li, li - 5, li)))
            if rng.random() < 0.7:
                rows.append((B.CTL_BECOME_LEADER, g))
        else:
            rows.append((B.CTL_BECOME_LEADER, g))
    lst = cmds(*rows)
    assert set(range(14)) <= set(lst["arg"][lst["op"] == B.CTL_PROGRESS_OP].tolist())
    got = a.control(lst)
    want = CO.arena_control(ref, votes, lst)
    assert np.array_equal(got["status"], want["status"]) and np.array_equal(got["value"], want["value"])
    assert (got["status"] == B.OK).mean() > 0.9
    assert_columns_equal(a.read_columns(n), ref, n, "control list")
    assert escaped_cells(ref).sum() > n
    for rnd in range(2):
        records_step(a, n, random_batch(ref, rng, 1, edge=True), ref, f"records step after the list, round {rnd}")
    a.close()
