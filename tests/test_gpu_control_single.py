"""The single-group control calls on the GPU where they meet the command form they are served through: the C
signatures take wider integers than a raftgpu_ctl_cmd holds, they keep working while records are enqueued for a step
(raftgpu_control refuses then), commit_to names its error, vote_result counts its tally, and group alloc / free of
narrow and wide groups leave the state and the launch plan the steps after them depend on.  Every case is checked
against the arena's state afterwards (every column, votes and term), the expected state from the control oracle's
ro_arena_control.  Run with -m gpu."""
import ctypes as C

import numpy as np
import pytest

from oracle import control_oracle as CO
from helpers import (B, O, Shape, TILE_SHAPES, assert_columns_equal, assert_state_equal, full_state, is_simple5,
                     random_batch, random_state, records_step, scatter_step)
from control_cmds import cmds

pytestmark = pytest.mark.gpu

N_NARROW = 62          # then two wide pairs at 62 and 64
WIDE = (62, 64)
N = N_NARROW + 4
G = 5                  # the narrow group the cases use


class World:
    """An arena of narrow groups with random configurations and two wide groups, and the oracle's copy of it."""

    def __init__(self, seed):
        rng = np.random.default_rng(seed)
        self.rng = rng
        init = random_state(N_NARROW, Shape(group_commit=True), rng)
        init.meta[G] = 0x1F | (0x20 << 16) | O.META_HAS_SELF        # peers 0..5, self 0, slot 6 absent
        self.a = B.Arena(256)
        assert self.a.group_alloc_range(N_NARROW) == 0
        self.a.load_columns(init)
        for k, g in enumerate(WIDE):
            assert self.a.group_alloc_wide() == g
            self.a.group_set_conf(g, 0x0307, 0x0300 if k else 0, 0x0400, 9, 40)
            self.a.group_reset(g, 30, 40, 35, 40)
        self.ref, self.votes, _ = full_state(self.a, N)
        self.L, self.h = self.a._L, self.a._h

    def check(self, what, got, status, cmd=None, value=None):
        """got: the call's (status, value); cmd: the command the oracle applies for it (None: the call changes
        nothing); value: the value the call must report (the oracle's when cmd is given)."""
        assert got[0] == status, f"{what}: status {got[0]}, want {status}"
        if cmd is not None:
            want = CO.arena_control(self.ref, self.votes, cmds(cmd))[0]
            assert want["status"] == status, f"{what}: the oracle's status {want['status']}"
            if value is None and status == B.OK:
                value = int(want["value"])
        if value is not None:
            assert got[1] == value, f"{what}: value {got[1]}, want {value}"
        assert_state_equal(full_state(self.a, N), (self.ref, self.votes, None), N, what)

    def out(self, fn, *args):
        r = C.c_int32(0x5A5A)
        return fn(self.h, *args, C.byref(r)), r.value

    def close(self):
        self.a.close()


@pytest.fixture
def world():
    w = World(0x51A6)
    yield w
    w.close()


def test_set_conf_self_slot_is_resolved_before_narrowing(world):
    w = world
    for g, wide in ((G, False), (WIDE[0], True)):
        inc, out, learn = (0x0307, 0x0300, 0x0400) if wide else (0x1F, 0, 0x20)
        for self_slot in (-7, -1, 8, 16, 255, 256, 0x10000, 2):
            ok = self_slot < 0 or self_slot < (16 if wide else 8)
            rc = w.L.raftgpu_group_set_conf(w.h, g, inc, out, learn, self_slot, 11)
            cmd = (B.CTL_SET_CONF, g, B.CTL_NO_SELF if self_slot < 0 else self_slot, 0, (inc, out, learn, 11))
            w.check(f"set_conf({g}, self {self_slot})", (rc, 0), B.OK if ok else B.ERR_TOO_MANY_PEERS,
                    cmd if ok else None)
        # a mask too wide is refused whatever the self slot
        rc = w.L.raftgpu_group_set_conf(w.h, g, (0x10000 if wide else 0x100) | 1, 0, 0, -1, 11)
        w.check(f"set_conf({g}, wide mask)", (rc, 0), B.ERR_TOO_MANY_PEERS)
    # the high half of a wide group is not a group of its own
    rc = w.L.raftgpu_group_set_conf(w.h, WIDE[0] + 1, 1, 0, 0, 256, 11)
    w.check("set_conf(high half)", (rc, 0), B.ERR_RANGE)


def test_progress_op_code_is_checked_after_the_slot(world):
    w = world
    for g, present, absent in ((G, 1, 6), (WIDE[0], 9, 12)):
        for op in (-1, B.POP_INS_FULL + 1, 0x10000, 0x10000 + B.POP_BECOME_SNAPSHOT):
            # a valid op would change the cell: MAYBE_UPDATE past matched, BECOME_SNAPSHOT
            w.check(f"progress_op({g}, {present}, op {op})",
                    w.out(w.L.raftgpu_progress_op, g, present, op, 1 << 60, 0, 0), B.ERR_INVALID, value=0x5A5A)
            w.check(f"progress_op({g}, absent {absent}, op {op})",
                    w.out(w.L.raftgpu_progress_op, g, absent, op, 1 << 60, 0, 0), B.ERR_PEER_NOT_FOUND, value=0x5A5A)
            w.check(f"progress_op({g}, slot 0x101, op {op})",
                    w.out(w.L.raftgpu_progress_op, g, 0x101, op, 1 << 60, 0, 0), B.ERR_RANGE, value=0x5A5A)
        w.check(f"progress_op({g}, {present}, MAYBE_UPDATE)",
                w.out(w.L.raftgpu_progress_op, g, present, B.POP_MAYBE_UPDATE, 1 << 60, 0, 0), B.OK,
                (B.CTL_PROGRESS_OP, g, present, B.POP_MAYBE_UPDATE, (1 << 60, 0, 0)))
        w.check(f"progress_op({g}, {present}, INS_FULL)",
                w.out(w.L.raftgpu_progress_op, g, present, B.POP_INS_FULL, 0, 0, 0), B.OK,
                (B.CTL_PROGRESS_OP, g, present, B.POP_INS_FULL))


def test_peer_slots_past_sixteen_do_not_wrap(world):
    w = world
    for g in (G, WIDE[0]):
        for slot in (0x101, 0x108, 16, 0xFFFFFFFF):
            w.check(f"assign_commit_group({g}, {slot})",
                    (w.L.raftgpu_assign_commit_group(w.h, g, slot, 77), 0), B.ERR_RANGE)
            w.check(f"record_vote({g}, {slot})", (w.L.raftgpu_record_vote(w.h, g, slot, 1), 0), B.ERR_RANGE)
            w.check(f"quorum_recently_active({g}, {slot})",
                    w.out(w.L.raftgpu_quorum_recently_active, g, slot), B.ERR_RANGE, value=0x5A5A)
            w.check(f"progress_op({g}, {slot})",
                    w.out(w.L.raftgpu_progress_op, g, slot, B.POP_PAUSE, 0, 0, 0), B.ERR_RANGE, value=0x5A5A)
    # slots 8..15 of a narrow group do not exist either; of a wide group they are the high half's
    w.check("record_vote(narrow, 9)", (w.L.raftgpu_record_vote(w.h, G, 9, 1), 0), B.ERR_RANGE)
    w.check("quorum_recently_active(narrow, 8)", w.out(w.L.raftgpu_quorum_recently_active, G, 8), B.ERR_RANGE,
            value=0x5A5A)
    w.check("assign_commit_group(wide, 9)", (w.L.raftgpu_assign_commit_group(w.h, WIDE[0], 9, 77), 0), B.OK,
            (B.CTL_ASSIGN_COMMIT_GROUP, WIDE[0], 9, 0, (77,)))
    w.check("quorum_recently_active(wide, 9)", w.out(w.L.raftgpu_quorum_recently_active, WIDE[0], 9), B.OK,
            (B.CTL_QUORUM_RECENTLY_ACTIVE, WIDE[0], 9))
    # an absent peer: assign_commit_group skips it silently
    w.check("assign_commit_group(absent)", (w.L.raftgpu_assign_commit_group(w.h, G, 6, 77), 0), B.OK,
            (B.CTL_ASSIGN_COMMIT_GROUP, G, 6, 0, (77,)))


def test_vote_and_enable_flags_are_any_nonzero(world):
    w = world
    for g in (G, WIDE[0]):
        w.check(f"reset_votes({g})", (w.L.raftgpu_reset_votes(w.h, g), 0), B.OK, (B.CTL_RESET_VOTES, g))
        no = 3 if g == G else 9                       # a voter's "no" (slot 9: the high half's voter 1)
        for s, vote in ((1, 0x10000), (2, -1), (no, 0), (0, 0x100)):
            w.check(f"record_vote({g}, {s}, {vote})", (w.L.raftgpu_record_vote(w.h, g, s, vote), 0), B.OK,
                    (B.CTL_RECORD_VOTE, g, s, int(vote != 0)))
        before = w.a.counters()["votes_tallied"]
        r, gr, rj = C.c_int32(), C.c_uint32(), C.c_uint32()
        rc = w.L.raftgpu_vote_result(w.h, g, C.byref(r), C.byref(gr), C.byref(rj))
        w.check(f"vote_result({g})", (rc, r.value | gr.value << 8 | rj.value << 16), B.OK, (B.CTL_VOTE_RESULT, g))
        assert (gr.value, rj.value) == (3, 1)
        assert w.a.counters()["votes_tallied"] == before + 1
        for enable in (0, 0x10000, 0, -1, 0, -(1 << 31)):
            w.check(f"set_group_commit({g}, {enable})", (w.L.raftgpu_set_group_commit(w.h, g, enable), 0), B.OK,
                    (B.CTL_SET_GROUP_COMMIT, g, 0, int(enable != 0)))
            on = bool(w.ref.meta[g] & O.META_GROUP_COMMIT)
            assert on == (enable != 0)
    # the mirror follows: a step afterwards runs on the launch plan the metas give
    scatter_step(w.a, N, random_batch(w.ref, w.rng, 1), w.ref, "step after the flags")


def test_has_quorum_mask_is_cut_to_the_group(world):
    w = world
    for g, width in ((G, 8), (WIDE[0], 16)):
        for low in (0b11, 0b111, 0x0107, 0x0307, 0x0F):
            for high in (0, 0xFFFF0000, 0xFFFFFF00):
                mask = (low | high) & 0xFFFFFFFF
                st, val = w.out(w.L.raftgpu_has_quorum, g, mask)
                w.check(f"has_quorum({g}, {mask:#x})", (st, val), B.OK, (B.CTL_HAS_QUORUM, g, 0, 0, (mask,)))
                assert val == w.out(w.L.raftgpu_has_quorum, g, mask & ((1 << width) - 1))[1]


def test_commit_to_out_of_range_names_its_error(world):
    w = world
    for g in (G, WIDE[0]):
        li = int(w.ref.last_index[g])
        before = w.ref.committed[g]
        rc = w.L.raftgpu_group_commit_to(w.h, g, li + 1)
        w.check(f"commit_to({g}, last_index + 1)", (rc, 0), B.ERR_COMMIT_RANGE, (B.CTL_COMMIT_TO, g, 0, 0, (li + 1,)))
        assert w.L.raftgpu_last_error(w.h) == b"to_commit is out of range [last_index]"
        assert w.ref.committed[g] == before
        rc = w.L.raftgpu_group_commit_to(w.h, g, li)
        w.check(f"commit_to({g}, last_index)", (rc, 0), B.OK, (B.CTL_COMMIT_TO, g, 0, 0, (li,)))
        assert w.ref.committed[g] == li
    w.check("commit_to(high half)", (w.L.raftgpu_group_commit_to(w.h, WIDE[0] + 1, 1), 0), B.ERR_RANGE)
    w.check("commit_to(unallocated)", (w.L.raftgpu_group_commit_to(w.h, 200, 1), 0), B.ERR_RANGE)


def test_votes_tallied_counts_each_vote_result(world):
    w = world
    c0 = w.a.counters()
    for g in (G, 0, WIDE[0], WIDE[0] + 1, 200, 3):
        r = C.c_int32()
        rc = w.L.raftgpu_vote_result(w.h, g, C.byref(r), None, None)
        assert rc == (B.ERR_RANGE if g == 200 else B.OK)
    c1 = w.a.counters()
    assert c1["votes_tallied"] - c0["votes_tallied"] == 5
    assert {k: c1[k] - c0[k] for k in c0 if k != "votes_tallied"} == {k: 0 for k in c0 if k != "votes_tallied"}


def test_single_calls_while_records_are_enqueued(world):
    """The single calls use no staging set: they run while records wait for a step, and the step applies the records
    on top of what they did.  raftgpu_control, which stages its list, refuses meanwhile."""
    w = world
    recs = random_batch(w.ref, w.rng, 1)
    w.a.enqueue(recs)
    with pytest.raises(B.RaftGpuError) as e:
        w.a.control(cmds((B.CTL_BECOME_LEADER, G)))
    assert e.value.status == B.ERR_BUSY
    calls = [
        ((B.CTL_SET_TERM, G, 0, 0, (99,)), lambda: (w.L.raftgpu_group_set_term(w.h, G, 99), 0)),
        ((B.CTL_SET_TERM, WIDE[1], 0, 0, (98,)), lambda: (w.L.raftgpu_group_set_term(w.h, WIDE[1], 98), 0)),
        ((B.CTL_SET_GROUP_COMMIT, 7, 0, 1), lambda: (w.L.raftgpu_set_group_commit(w.h, 7, 1), 0)),
        ((B.CTL_PROGRESS_OP, G, 1, B.POP_BECOME_REPLICATE),
         lambda: w.out(w.L.raftgpu_progress_op, G, 1, B.POP_BECOME_REPLICATE, 0, 0, 0)),
        ((B.CTL_SET_CONF, 9, 0, 0, (0x3F, 0, 0, 5)), lambda: (w.L.raftgpu_group_set_conf(w.h, 9, 0x3F, 0, 0, 0, 5), 0)),
        ((B.CTL_BECOME_LEADER, WIDE[0]), lambda: (w.L.raftgpu_group_become_leader(w.h, WIDE[0]), 0)),
        ((B.CTL_HAS_QUORUM, G, 0, 0, (0x7,)), lambda: w.out(w.L.raftgpu_has_quorum, G, 0x7)),
    ]
    for cmd, call in calls:
        got = call()
        want = CO.arena_control(w.ref, w.votes, cmds(cmd))[0]
        assert got == (B.OK, int(want["value"]) if cmd[0] == B.CTL_HAS_QUORUM else 0), cmd
    r = w.a.step(B.STEP_READ_COMMITTED)
    O.arena_apply(w.ref, recs, mode=0)
    want_adv, _, _, _ = O.arena_recompute(w.ref)
    assert r.n_advanced == want_adv
    assert_state_equal(full_state(w.a, N), (w.ref, w.votes, None), N, "step after the single calls")
    assert (w.a.control(cmds((B.CTL_BECOME_LEADER, G)))["status"] == B.OK).all()


def _pair_freed(ref, votes, g, halves):
    """What raftgpu_group_free leaves: no term range, an empty configuration (the removed peers' cells reset), meta 0
    and committed 0 on every half."""
    CO.arena_control(ref, votes, cmds((B.CTL_SET_LOG_BOUNDS, g, 0, 0, (B.NO_TERM_START, 0)),
                                      (B.CTL_SET_CONF, g, B.CTL_NO_SELF, 0, (0, 0, 0, 0))))
    ref.meta[g:g + halves] = 0
    ref.committed[g:g + halves] = 0


def test_group_alloc_free_and_reuse_keep_the_launch_plan():
    """Plain 5-voter groups take the kSimple5 fused kernel; a wide group moves every step to the paths that accept
    one (and the fused device entry points refuse); a freed slot (meta 0 inside [0, hi)) moves them to the general
    kernel; reusing the slots as plain 5-voter groups brings kSimple5 back.  State after every call against the
    oracle, steps after every call against O.arena_apply / O.arena_recompute."""
    n = 4096
    rng = np.random.default_rng(0xA110C)
    init = random_state(n, TILE_SHAPES["v5_simple"][0], rng)
    a = B.Arena(n + 64)
    assert a.group_alloc_range(n) == 0
    a.load_columns(init)
    ref, votes, _ = full_state(a, n + 2)
    alloc = np.arange(n + 2) < n                                # the allocated group slots
    d_pk, d_off = a.device_alloc(256), a.device_alloc(4 * (a.cap // B.tile_groups() + 2))

    def state(what):
        assert_state_equal(full_state(a, n + 2), (ref, votes, None), n + 2, what)

    def step(simple5, wide, what):
        hi = a.get_info().hi
        assert is_simple5(ref.meta[:hi]).all() == simple5, what
        if wide:
            with pytest.raises(B.RaftGpuError) as e:          # the fused device entry points take no wide group
                a.step_sorted_device(d_pk, 0, d_off)
            assert e.value.status == B.ERR_INVALID
        else:
            a.step_sorted_device(d_pk, 0, d_off)                # no records: a recompute of [0, hi)
            O.arena_recompute(ref)
        records_step(a, n + 2, random_batch(ref, rng, 1, keep=alloc), ref, what)
        state(what)

    step(True, False, "plain 5-voter")
    g = a.group_alloc_wide()
    assert g == n
    alloc[g:g + 2] = True
    ref.meta[g], ref.meta[g + 1] = 0x20000000, 0x40000000     # empty halves that know they are halves
    state("alloc_wide")
    a.group_set_conf(g, 0x0F0F, 0, 0x10, 0, 20)
    a.group_reset(g, 15, 20, 12, 20)
    CO.arena_control(ref, votes, cmds((B.CTL_SET_CONF, g, 0, 0, (0x0F0F, 0, 0x10, 20)),
                                      (B.CTL_RESET, g, 0, 0, (15, 20, 12, 20))))
    step(False, True, "a wide group")
    a.group_free(g)
    alloc[g:g + 2] = False
    _pair_freed(ref, votes, g, 2)
    state("free wide")
    step(False, False, "after the wide group")
    gf = 1000
    a.group_free(gf)
    alloc[gf] = False
    _pair_freed(ref, votes, gf, 1)
    state("free narrow")
    step(False, False, "a free narrow slot")
    for want in (gf, g + 1, g):                                 # the free list, last freed first
        assert a.group_alloc() == want
        alloc[want] = True
        a.group_set_conf(want, 0x1F, 0, 0, 0, 30)
        a.group_reset(want, 25, 30, 28, 30)
        CO.arena_control(ref, votes, cmds((B.CTL_SET_CONF, want, 0, 0, (0x1F, 0, 0, 30)),
                                          (B.CTL_RESET, want, 0, 0, (25, 30, 28, 30))))
        state(f"reuse {want}")
    step(True, False, "plain 5-voter again")
    assert_columns_equal(a.read_columns(n + 2), ref, n + 2, "end")
    a.close()
