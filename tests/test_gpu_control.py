"""raftgpu_control (the control plane's list form) on the GPU.  Differential against the single-group calls on twin
arenas and against the oracle's ro_arena_control: every column, every result, the counters, and steps afterwards
(which run on the launch plan the meta mirror gives).  Then the 1M-group election storm in lists longer than the
staging buffer, and the edge cases of the call.  Run with -m gpu."""
import ctypes as C

import numpy as np
import pytest

from oracle import control_oracle as CO
from helpers import (B, O, Shape, assert_columns_equal, assert_state_equal, full_state, random_batch,
                     random_state, records_step, scatter_step)
from control_cmds import NO_TERM_START, cmds, random_list

pytestmark = pytest.mark.gpu


def single(arena, m):
    """One command through its single-group call: (status, value); an op with no call is ERR_INVALID."""
    L, h = arena._L, arena._h
    op, g, s, arg = int(m["op"]), int(m["group"]), int(m["peer_slot"]), int(m["arg"])
    a = [int(x) for x in m["a"]]
    out, gr, rj = C.c_int32(0), C.c_uint32(0), C.c_uint32(0)
    if op == B.CTL_SET_CONF:
        return L.raftgpu_group_set_conf(h, g, a[0], a[1], a[2], -1 if s == B.CTL_NO_SELF else s, a[3]), 0
    if op == B.CTL_RESET:
        return L.raftgpu_group_reset(h, g, *a), 0
    if op == B.CTL_BECOME_LEADER:
        return L.raftgpu_group_become_leader(h, g), 0
    if op == B.CTL_SET_LOG_BOUNDS:
        return L.raftgpu_group_set_log_bounds(h, g, a[0], a[1]), 0
    if op == B.CTL_SET_TERM:
        return L.raftgpu_group_set_term(h, g, a[0]), 0
    if op == B.CTL_COMMIT_TO:
        return L.raftgpu_group_commit_to(h, g, a[0]), 0
    if op == B.CTL_MAYBE_COMMIT_TO:
        return L.raftgpu_group_maybe_commit_to(h, g, a[0], C.byref(out)), out.value
    if op == B.CTL_SET_GROUP_COMMIT:
        return L.raftgpu_set_group_commit(h, g, arg), 0
    if op == B.CTL_ASSIGN_COMMIT_GROUP:
        return L.raftgpu_assign_commit_group(h, g, s, a[0]), 0
    if op == B.CTL_RESET_VOTES:
        return L.raftgpu_reset_votes(h, g), 0
    if op == B.CTL_RECORD_VOTE:
        return L.raftgpu_record_vote(h, g, s, arg), 0
    if op == B.CTL_VOTE_RESULT:
        rc = L.raftgpu_vote_result(h, g, C.byref(out), C.byref(gr), C.byref(rj))
        return rc, (out.value | gr.value << 8 | rj.value << 16) if rc == B.OK else 0
    if op == B.CTL_HAS_QUORUM:
        rc = L.raftgpu_has_quorum(h, g, a[0] & 0xFFFFFFFF, C.byref(out))
        return rc, out.value if rc == B.OK else 0
    if op == B.CTL_QUORUM_RECENTLY_ACTIVE:
        rc = L.raftgpu_quorum_recently_active(h, g, s, C.byref(out))
        return rc, out.value if rc == B.OK else 0
    if op == B.CTL_PROGRESS_OP:
        rc = L.raftgpu_progress_op(h, g, s, arg, a[0], a[1], a[2], C.byref(out))
        return rc, out.value if rc == B.OK else 0
    return B.ERR_INVALID, 0


N_NARROW, N_WIDE = 4088, 4   # 4096 group slots: 4088 narrow groups, then 4 wide pairs


def twin_arenas(rng, inflights):
    """Two arenas with the same state: random narrow groups (joint configurations, learners, group commit) and wide
    groups configured through the single calls."""
    init = random_state(N_NARROW, Shape(group_commit=True), rng)
    if inflights:
        init.pflags &= np.uint8(~O.PF_INS_FULL & 0xFF)   # the windows start empty: not full
    wide_conf = [(int(rng.integers(1, 1 << 16)), int(rng.integers(0, 1 << 16)) if k % 2 else 0,
                  int(rng.integers(0, 16)), int(rng.integers(100, 1 << 30))) for k in range(N_WIDE)]
    arenas = []
    for _ in range(2):
        ar = B.Arena(N_NARROW + 2 * N_WIDE + 64)
        if inflights:
            ar.enable_inflights(8)
        assert ar.group_alloc_range(N_NARROW) == 0
        ar.load_columns(init)
        for k, (inc, out, me, li) in enumerate(wide_conf):
            g = ar.group_alloc_wide()
            assert g == N_NARROW + 2 * k
            ar.group_set_conf(g, inc, out, 0, me, li)
            ar.group_reset(g, li - 3, li, li - 5, li)
        arenas.append(ar)
    return arenas


def plan_cases(rng):
    """The launch-plan changes of the fused kernels' plan test: a sixth voter, group commit on and off, a wide
    group's configuration, each among other commands of the same groups."""
    g5, gc, gw = 17, 33, N_NARROW
    return cmds((B.CTL_SET_CONF, g5, 0, 0, (0x3F, 0, 0, 5)), (B.CTL_PROGRESS_OP, g5, 5, B.POP_MAYBE_UPDATE, (3,)),
                (B.CTL_SET_GROUP_COMMIT, gc, 0, 1), (B.CTL_ASSIGN_COMMIT_GROUP, gc, 1, 0, (2,)),
                (B.CTL_SET_GROUP_COMMIT, gc + 1, 0, 1), (B.CTL_SET_GROUP_COMMIT, gc + 1, 0, 0),
                (B.CTL_SET_CONF, gw, 9, 0, (0x0303, 0x0300, 0xC000, 7)), (B.CTL_PROGRESS_OP, gw, 14, B.POP_BECOME_REPLICATE),
                (B.CTL_HAS_QUORUM, gw, 0, 0, (0x0301,)))


@pytest.mark.parametrize("inflights", [False, True], ids=["no_windows", "inflights"])
def test_control_list_matches_single_calls_and_oracle(inflights):
    rng = np.random.default_rng(0xC7A1 + inflights)
    ar_list, ar_single = twin_arenas(rng, inflights)
    n = N_NARROW + 2 * N_WIDE
    groups = list(range(N_NARROW)) + [N_NARROW + 2 * k for k in range(N_WIDE)]
    wide_lo = set(groups[N_NARROW:])
    lst = np.concatenate([plan_cases(rng), random_list(rng, 20_000, groups, wide_lo, n_alloc=n)])
    # every op, every Progress method, refusals of every kind
    assert set(range(15)) <= set(lst["op"].tolist()) and set(range(19)) <= set(lst["arg"][lst["op"] == B.CTL_PROGRESS_OP].tolist())
    assert np.bincount(lst["group"][lst["group"] < n], minlength=n).max() >= 8

    # the oracle from the same state
    ref, votes, ins = full_state(ar_list, n, inflights)
    ref.n_groups = n
    if inflights:
        O.enable_inflights(ref, 8)
        ref.ins_meta[:] = ins
    want = CO.arena_control(ref, votes, lst)

    c0 = ar_list.counters()
    got = ar_list.control(lst)
    c1 = ar_list.counters()
    s0 = ar_single.counters()
    single_res = np.array([single(ar_single, m) for m in lst], dtype=np.int64)
    s1 = ar_single.counters()

    statuses = set(single_res[:, 0].tolist())
    assert {B.OK, B.ERR_RANGE, B.ERR_PEER_NOT_FOUND, B.ERR_TOO_MANY_PEERS, B.ERR_INVALID, B.ERR_COMMIT_RANGE} <= statuses
    assert np.array_equal(got["status"], single_res[:, 0]), np.flatnonzero(got["status"] != single_res[:, 0])[:5]
    assert np.array_equal(got["value"], single_res[:, 1]), np.flatnonzero(got["value"] != single_res[:, 1])[:5]
    assert np.array_equal(got["status"], want["status"]) and np.array_equal(got["value"], want["value"])
    tallied = int(np.count_nonzero((lst["op"] == B.CTL_VOTE_RESULT) & (got["status"] == B.OK)))
    assert c1["votes_tallied"] - c0["votes_tallied"] == s1["votes_tallied"] - s0["votes_tallied"] == tallied
    assert {k: c1[k] - c0[k] for k in c0} == {k: s1[k] - s0[k] for k in s0}

    st_list, st_single = full_state(ar_list, n, inflights), full_state(ar_single, n, inflights)
    assert_state_equal(st_list, st_single, n, "list vs single calls")
    assert_state_equal(st_list, (ref, votes, ref.ins_meta if inflights else None), n, "list vs oracle")

    # steps on the state the lists left: the launch plan follows the meta mirror
    ref2 = O.copy_columns(ref)
    for k, (ar, r) in enumerate(((ar_list, ref), (ar_single, ref2))):
        recs = random_batch(r, np.random.default_rng(5 + k), 1)
        scatter_step(ar, n, recs, r, f"scatter step after the list ({k})")
        recs = random_batch(r, np.random.default_rng(7 + k), 1)
        records_step(ar, n, recs, r, f"records step after the list ({k})")
    ar_list.close()
    ar_single.close()


def test_control_plan_changes_reach_the_fused_kernel():
    """An arena of plain 5-voter groups runs the kSimple5 fused kernel; a list that gives one group a sixth voter,
    or group commit, must move the next step to the general instantiation, exactly as the single calls do."""
    n = 40_000
    s = B.Synth(n, 0x5EED0003)
    for lst in (cmds((B.CTL_SET_CONF, 11, 0, 0, (0x3F, 0, 0, 9))),
                cmds((B.CTL_SET_GROUP_COMMIT, 12, 0, 1), (B.CTL_ASSIGN_COMMIT_GROUP, 12, 1, 0, (1,)),
                     (B.CTL_ASSIGN_COMMIT_GROUP, 12, 2, 0, (2,))),
                cmds((B.CTL_SET_GROUP_COMMIT, 13, 0, 1), (B.CTL_SET_GROUP_COMMIT, 13, 0, 0))):
        arenas = []
        for via_list in (True, False):
            ar = B.Arena(n)
            ar.group_alloc_range(n)
            ar.load_columns(s.initial)
            if via_list:
                assert (ar.control(lst)["status"] == B.OK).all()
            else:
                assert all(single(ar, m)[0] == B.OK for m in lst)
            arenas.append(ar)
        ref = O.copy_columns(s.initial)
        CO.arena_control(ref, np.zeros((O.SLOTS, ref.cap), dtype=np.uint8), lst)
        assert_columns_equal(arenas[0].read_columns(n), ref, n, "list")
        refs = [ref, O.copy_columns(ref)]
        for k, ar in enumerate(arenas):
            recs = random_batch(refs[k], np.random.default_rng(3), 1)
            records_step(ar, n, recs, refs[k], f"fused step after {lst['op'].tolist()} ({k})")
            ar.close()


def storm_lists(n, init, rng):
    """The store-wide election after a restart (INTEGRATION 6): every group campaigns (reset, the new term, its own
    vote, the tally), the vote responses arrive, the winners become leaders.  Slot 0 is every group's own."""
    li = init.last_index[:n].astype(np.uint64)
    g = np.arange(n, dtype=np.uint32)
    a = np.zeros((n, 5), dtype=B.CTL_CMD_DTYPE)
    a["group"] = g[:, None]
    a["op"] = [B.CTL_RESET, B.CTL_SET_TERM, B.CTL_RESET_VOTES, B.CTL_RECORD_VOTE, B.CTL_VOTE_RESULT]
    a["a"][:, 0, 0], a["a"][:, 0, 1], a["a"][:, 0, 2], a["a"][:, 0, 3] = NO_TERM_START, li, init.committed[:n], li
    a["a"][:, 1, 0] = rng.integers(2, 100, n)
    a["arg"][:, 3] = 1
    b = np.zeros((n, 5), dtype=B.CTL_CMD_DTYPE)    # the responses of peers 1..4, then the tally
    b["group"] = g[:, None]
    b["op"][:, :4], b["op"][:, 4] = B.CTL_RECORD_VOTE, B.CTL_VOTE_RESULT
    b["peer_slot"][:, :4] = np.arange(1, 5)
    b["arg"][:, :4] = rng.random((n, 4)) < 0.6
    order = rng.permutation(n)                     # responses arrive in any group order
    return a.reshape(-1), b[order].reshape(-1)


def test_election_storm_1m_against_oracle():
    n = 1_000_000
    s = B.Synth(n, 0x5EED0003)
    assert ((s.initial.meta[:n] >> 24) & 7 == 0).all() and (s.initial.meta[:n] & O.META_HAS_SELF).all()
    ar = B.Arena(n)
    ar.group_alloc_range(n)
    ar.load_columns(s.initial)
    ref = O.copy_columns(s.initial)
    votes = np.zeros((O.SLOTS, n), dtype=np.uint8)
    rng = np.random.default_rng(0x57041)
    campaign, responses = storm_lists(n, s.initial, rng)
    for what, lst in (("campaign", campaign), ("responses", responses)):
        got = ar.control(lst)
        want = CO.arena_control(ref, votes, lst)
        assert (got["status"] == B.OK).all(), what
        assert np.array_equal(got["value"], want["value"]), what
    tally = got["value"].reshape(n, 5)[:, 4]
    winners = responses["group"].reshape(n, 5)[:, 4][(tally & 0xFF) == B.VOTE_WON]
    assert 0.5 * n < len(winners) < n
    lead = np.zeros((len(winners), 2), dtype=B.CTL_CMD_DTYPE)
    lead["group"] = winners[:, None]
    lead["op"] = [B.CTL_RESET, B.CTL_BECOME_LEADER]
    li = ref.last_index[winners]
    lead["a"][:, 0, 0], lead["a"][:, 0, 1], lead["a"][:, 0, 2], lead["a"][:, 0, 3] = li + 1, li, ref.committed[winners], li
    lead = lead.reshape(-1)
    got = ar.control(lead)
    want = CO.arena_control(ref, votes, lead)
    assert (got["status"] == B.OK).all() and np.array_equal(got["value"], want["value"])
    assert_columns_equal(ar.read_columns(n), ref, n, "after the election")
    for k in range(B.SLOTS):
        assert np.array_equal(ar.column_read(B.COL_VOTES, k, 0, n, np.uint8), votes[k]), f"votes of slot {k}"
    assert np.array_equal(ar.column_read(B.COL_TERM, 0, 0, n, np.uint64), ref.term[:n])
    recs = random_batch(ref, np.random.default_rng(11), 1)
    records_step(ar, n, recs, ref, "step after the election")
    ar.close()


def test_control_edge_cases():
    ar = B.Arena(1024)
    ar.group_alloc_range(16)
    L, h = ar._L, ar._h
    res = np.zeros(4, dtype=B.CTL_RESULT_DTYPE)
    one = cmds((B.CTL_SET_CONF, 0, 0, 0, (0x7, 0, 0, 1)))
    assert L.raftgpu_control(h, None, 0, None) == B.OK
    assert L.raftgpu_control(h, one.ctypes.data, 0, None) == B.OK
    assert ar.control(one[:0]).shape == (0,)
    assert L.raftgpu_control(None, one.ctypes.data, 1, res.ctypes.data) == B.ERR_INVALID
    assert L.raftgpu_control(h, None, 1, res.ctypes.data) == B.ERR_INVALID
    assert L.raftgpu_control(h, one.ctypes.data, 1, None) == B.ERR_INVALID
    # records enqueued for a step: refused until the step, like the other host batch calls
    assert (ar.control(one)["status"] == B.OK).all()
    recs = np.zeros(1, dtype=B.APPEND_RESP_DTYPE)
    recs[0] = (0, 1, 0, 0, 1, 0)
    ar.enqueue(recs)
    with pytest.raises(B.RaftGpuError) as e:
        ar.control(one)
    assert e.value.status == B.ERR_BUSY
    ar.step()
    assert (ar.control(one)["status"] == B.OK).all()
    ar.close()
