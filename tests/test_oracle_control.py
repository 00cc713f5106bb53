"""The control plane's list form on the CPU oracle (ro_arena_control, oracle/control_oracle.c): the lifecycle of one group, the reference's
vote golden vectors, the statuses of refused commands, and the C layout of the command and result structs."""
import os
import sys

import numpy as np
import pytest

from oracle import control_oracle as CO
from oracle import datadriven as dd
from oracle import oracle as O
from helpers import B
from control_cmds import cmds, NO_TERM_START, META_WIDE_LO, META_WIDE_HI

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def arena(n_groups, cap=None, wide_pairs=0):
    """Oracle columns of n_groups narrow groups followed by wide_pairs wide groups (two slots each)."""
    n = n_groups + 2 * wide_pairs
    c = O.new_columns(cap or n + 8, n)
    c.term_start[:] = NO_TERM_START
    for k in range(wide_pairs):
        lo = n_groups + 2 * k
        c.meta[lo], c.meta[lo + 1] = META_WIDE_LO, META_WIDE_HI
    return c, np.zeros((O.SLOTS, c.cap), dtype=np.uint8)


def run(c, votes, *rows):
    return CO.arena_control(c, votes, cmds(*rows))


def prog(c, g, s):
    f = int(c.pflags[s, g])
    return (int(c.matched[s, g]), int(c.next_idx[s, g]), int(c.peer_committed[s, g]), f & 3,
            bool(f & O.PF_RECENT_ACTIVE))


def test_lifecycle_mirrors_raft_new_reset_become_leader():
    """The expectations of the single-call lifecycle test, through the list form."""
    c, votes = arena(1)
    # Raft::new: confchange::restore adds three voters with next_idx = last_index + 1 = 1
    r = run(c, votes, (B.CTL_SET_CONF, 0, 0, 0, (0b111, 0, 0, 1)), (B.CTL_PROGRESS_OP, 0, 5, B.POP_IS_PAUSED))
    assert r["status"].tolist() == [B.OK, B.ERR_PEER_NOT_FOUND]
    for s in range(3):
        assert prog(c, 0, s) == (0, 1, 0, B.STATE_PROBE, True)
    # Raft::reset at last_index 7, committed 4, persisted 7 (raft.rs:942-971)
    assert run(c, votes, (B.CTL_RESET, 0, 0, 0, (NO_TERM_START, 7, 4, 7)))["status"].tolist() == [B.OK]
    assert prog(c, 0, 0) == (7, 8, 4, B.STATE_PROBE, False)
    assert prog(c, 0, 1)[:2] == (0, 8) and prog(c, 0, 1)[3] == B.STATE_PROBE
    assert O.arena_maybe_commit(c, 0) is False and int(c.committed[0]) == 4   # follower: no quorum commit
    # become_leader (raft.rs:1162-1203): self Replicate, noop appended at 8 = term_start
    run(c, votes, (B.CTL_BECOME_LEADER, 0))
    assert (int(c.term_start[0]), int(c.last_index[0]), int(c.committed[0])) == (8, 8, 4)
    assert prog(c, 0, 0)[3] == B.STATE_REPLICATE
    # the leader persists the noop, one follower acks it -> commit 8
    recs = np.zeros(2, dtype=O.APPEND_RESP_DTYPE)
    recs[0] = (0, 0, O.REC_LOCAL, 0, 8, 8)
    recs[1] = (0, 1, 0, 0, 8, 4)
    O.arena_apply(c, recs)
    O.arena_recompute(c)
    assert int(c.committed[0]) == 8
    # RaftLog::commit_to (raft_log.rs:286-300)
    r = run(c, votes, (B.CTL_COMMIT_TO, 0, 0, 0, (3,)), (B.CTL_COMMIT_TO, 0, 0, 0, (9,)))
    assert r["status"].tolist() == [B.OK, B.ERR_COMMIT_RANGE] and int(c.committed[0]) == 8
    # apply_conf removing a voter drops its Progress
    r = run(c, votes, (B.CTL_SET_CONF, 0, 0, 0, (0b011, 0, 0, 9)), (B.CTL_PROGRESS_OP, 0, 2, B.POP_IS_PAUSED))
    assert r["status"].tolist() == [B.OK, B.ERR_PEER_NOT_FOUND]
    assert prog(c, 0, 2) == (0, 0, 0, 0, False) and int(c.meta[0]) == O.make_meta(0b011, self_slot=0)


def _vote_impl():
    """VoteResult through a wide group's RESET_VOTES + SET_CONF + RECORD_VOTE + VOTE_RESULT commands: voter ids go to
    peer slots in sorted order (any injective assignment gives the same result)."""
    def vote(incoming, outgoing, votes):
        ids = sorted(set(incoming) | set(outgoing) | set(votes))
        assert len(ids) <= 16
        slot = {i: k for k, i in enumerate(ids)}
        mask = lambda xs: sum(1 << slot[i] for i in set(xs))
        c, vt = arena(0, wide_pairs=1)
        rows = [(B.CTL_SET_CONF, 0, 0, 0, (mask(incoming), mask(outgoing), 0, 1)), (B.CTL_RESET_VOTES, 0)]
        rows += [(B.CTL_RECORD_VOTE, 0, slot[i], int(v)) for i, v in votes.items()]
        rows += [(B.CTL_VOTE_RESULT, 0), (B.CTL_VOTE_RESULT, 1)]
        r = run(c, vt, *rows)
        assert (r["status"] == B.OK).all()
        assert r["value"][-1] == r["value"][-2]   # both halves report the group's result
        granted = sum(1 for i, v in votes.items() if v and i in set(incoming) | set(outgoing))
        assert (r["value"][-1] >> 8) & 0xFF == granted
        return int(r["value"][-1]) & 0xFF
    return dd.Impl(majority_vote=lambda v, votes: vote(v, [], votes), joint_vote=vote)


@pytest.mark.parametrize("name", ["majority_vote.txt", "joint_vote.txt"])
def test_vote_golden_files_replay_through_commands(golden_dir, name):
    cases = dd.replay_file(os.path.join(golden_dir, "quorum", name), _vote_impl())
    assert len(cases) == {"majority_vote.txt": 22, "joint_vote.txt": 39}[name]
    for d, actual in cases:
        assert actual == d.expected, f"{d.pos}\n--- actual\n{actual}--- expected\n{d.expected}"


# groups of the status table: 0 = narrow (3 voters, self 0), 1 = narrow (empty), 2/3 = a wide pair, 4.. unallocated
_STATUS_TABLE = [
    # (op, group, peer_slot, arg, a) -> status
    ((B.CTL_SET_CONF, 5), B.ERR_RANGE),
    ((B.CTL_SET_CONF, 3), B.ERR_RANGE),
    ((B.CTL_SET_CONF, 0, 0, 0, (0x100, 0, 0, 1)), B.ERR_TOO_MANY_PEERS),
    ((B.CTL_SET_CONF, 0, 0, 0, (1, 0x100, 0, 1)), B.ERR_TOO_MANY_PEERS),
    ((B.CTL_SET_CONF, 0, 0, 0, (1, 0, 1 << 40, 1)), B.ERR_TOO_MANY_PEERS),
    ((B.CTL_SET_CONF, 0, 8, 0, (1, 0, 0, 1)), B.ERR_TOO_MANY_PEERS),
    ((B.CTL_SET_CONF, 2, 0, 0, (0x10000, 0, 0, 1)), B.ERR_TOO_MANY_PEERS),
    ((B.CTL_SET_CONF, 2, 16, 0, (1, 0, 0, 1)), B.ERR_TOO_MANY_PEERS),
    ((B.CTL_SET_CONF, 2, 15, 0, (0x0F0F, 0, 0, 1)), B.OK),
    ((B.CTL_SET_CONF, 1, B.CTL_NO_SELF, 0, (0x3, 0, 0, 1)), B.OK),
] + [((op, g), B.ERR_RANGE) for op in (B.CTL_RESET, B.CTL_BECOME_LEADER, B.CTL_SET_LOG_BOUNDS, B.CTL_COMMIT_TO,
                                          B.CTL_MAYBE_COMMIT_TO, B.CTL_SET_GROUP_COMMIT, B.CTL_RESET_VOTES,
                                          B.CTL_HAS_QUORUM, B.CTL_QUORUM_RECENTLY_ACTIVE) for g in (3, 6)] + [
    ((B.CTL_SET_TERM, 3, 0, 0, (5,)), B.OK),          # set_term and vote_result take the high half
    ((B.CTL_VOTE_RESULT, 3), B.OK),
    ((B.CTL_SET_TERM, 4), B.ERR_RANGE),
    ((B.CTL_VOTE_RESULT, 4), B.ERR_RANGE),
    ((B.CTL_QUORUM_RECENTLY_ACTIVE, 0, 8), B.ERR_RANGE),
    ((B.CTL_QUORUM_RECENTLY_ACTIVE, 2, 16), B.ERR_RANGE),
    ((B.CTL_QUORUM_RECENTLY_ACTIVE, 2, 15), B.OK),
    ((B.CTL_COMMIT_TO, 0, 0, 0, (99,)), B.ERR_COMMIT_RANGE),
    ((B.CTL_COMMIT_TO, 2, 0, 0, (99,)), B.ERR_COMMIT_RANGE),
    ((B.CTL_HAS_QUORUM, 0, 0, 0, (1 << 40,)), B.OK),  # the mask is cut to the group's slots, as the single call does
] + [((op, 0, 8), B.ERR_RANGE) for op in (B.CTL_RECORD_VOTE, B.CTL_ASSIGN_COMMIT_GROUP, B.CTL_PROGRESS_OP)] + [
    ((op, 2, 16), B.ERR_RANGE) for op in (B.CTL_RECORD_VOTE, B.CTL_ASSIGN_COMMIT_GROUP, B.CTL_PROGRESS_OP)] + [
    ((op, 5, 0), B.ERR_RANGE) for op in (B.CTL_RECORD_VOTE, B.CTL_ASSIGN_COMMIT_GROUP, B.CTL_PROGRESS_OP)] + [
    ((B.CTL_RECORD_VOTE, 3, 0, 1), B.OK),             # record_vote takes the high half's own slots 0..7
    ((B.CTL_RECORD_VOTE, 0, 5, 1), B.OK),             # ... and an absent peer (votes.entry(id).or_insert)
    ((B.CTL_ASSIGN_COMMIT_GROUP, 0, 5, 0, (7,)), B.OK),   # an absent peer is skipped (raft.rs:534-540)
    ((B.CTL_PROGRESS_OP, 0, 5, B.POP_RESUME), B.ERR_PEER_NOT_FOUND),
    ((B.CTL_PROGRESS_OP, 0, 1, 19), B.ERR_INVALID),
    ((B.CTL_PROGRESS_OP, 0, 1, 0xFFFF), B.ERR_INVALID),
    ((B.CTL_PROGRESS_OP, 0, 5, 19), B.ERR_PEER_NOT_FOUND),   # the peer is checked before the method
    ((B.CTL_PROGRESS_OP, 2, 12, B.POP_INS_FULL), B.ERR_PEER_NOT_FOUND),
    ((15, 0), B.ERR_INVALID),
    ((255, 0), B.ERR_INVALID),
    ((255, 5), B.ERR_INVALID),                        # no such call, whatever the group
]


def _status_arena():
    c, votes = arena(2, wide_pairs=1)
    r = run(c, votes, (B.CTL_SET_CONF, 0, 0, 0, (0b111, 0, 0, 5)), (B.CTL_RESET, 0, 0, 0, (6, 10, 3, 10)),
            (B.CTL_SET_CONF, 2, 0, 0, (0x0F0F, 0, 0, 5)))
    assert (r["status"] == B.OK).all()
    return c, votes


@pytest.mark.parametrize("row,want", _STATUS_TABLE)
def test_refused_commands_carry_the_single_call_status(row, want):
    c, votes = _status_arena()
    before, vbefore = O.copy_columns(c), votes.copy()
    r = run(c, votes, row)
    assert r["status"][0] == want
    if want != B.OK:   # a refused command does nothing (commit_to's out-of-range refusal included)
        assert r["value"][0] == 0
        for name in O.PEER_COLUMNS + ("pflags", "meta") + O.GROUP_COLUMNS:
            assert np.array_equal(getattr(c, name), getattr(before, name)), name
        assert np.array_equal(votes, vbefore)


def test_refused_commands_do_not_stop_the_list():
    c, votes = _status_arena()
    rows = [row for row, _ in _STATUS_TABLE] + [(B.CTL_MAYBE_COMMIT_TO, 0, 0, 0, (7,))]
    r = run(c, votes, *rows)
    assert r["status"][:-1].tolist() == [w for _, w in _STATUS_TABLE]
    # the command after them all still runs: 7 lies in the leader's term [6, 10]
    assert r["status"][-1] == B.OK and r["value"][-1] == 1 and int(c.committed[0]) == 7


def test_earlier_commands_of_the_list_count():
    """A Progress method on a slot an earlier SET_CONF of the same list adds is valid; one on a slot it removes is not."""
    c, votes = arena(1)
    r = run(c, votes, (B.CTL_PROGRESS_OP, 0, 3, B.POP_IS_PAUSED), (B.CTL_SET_CONF, 0, 0, 0, (0b1001, 0, 0, 4)),
            (B.CTL_PROGRESS_OP, 0, 3, B.POP_MAYBE_UPDATE, (6,)), (B.CTL_SET_CONF, 0, 0, 0, (0b0001, 0, 0, 4)),
            (B.CTL_PROGRESS_OP, 0, 3, B.POP_IS_PAUSED))
    assert r["status"].tolist() == [B.ERR_PEER_NOT_FOUND, B.OK, B.OK, B.OK, B.ERR_PEER_NOT_FOUND]
    assert r["value"][2] == 1


def test_command_and_result_layouts_match_the_header():
    sys.path.insert(0, os.path.join(ROOT, "scripts"))
    import gen_rust_stub as G
    lay = G.struct_layouts()
    for name, dt in (("raftgpu_ctl_cmd", B.CTL_CMD_DTYPE), ("raftgpu_ctl_result", B.CTL_RESULT_DTYPE)):
        size, offs = lay[name]
        assert size == dt.itemsize, name
        assert [(f, o) for f, o, _ in offs] == [(f, dt.fields[f][1]) for f in dt.names], name
    assert lay["raftgpu_ctl_cmd"][0] == 40 and lay["raftgpu_ctl_result"][0] == 8
    assert CO.CTL_CMD_DTYPE == B.CTL_CMD_DTYPE and CO.CTL_RESULT_DTYPE == B.CTL_RESULT_DTYPE
    consts, _, _, _ = G.parse_header()
    ctl = {n[len("RAFTGPU_CTL_"):]: v for n, v, _ in consts if n.startswith("RAFTGPU_CTL_")}
    assert ctl == {n[len("CTL_"):]: getattr(B, n) for n in dir(B) if n.startswith("CTL_") and n[4:] in ctl}
    assert sorted(ctl.values()) == list(range(15))
