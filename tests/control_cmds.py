"""Control-command lists (raftgpu_control / ro_arena_control) for the control-plane tests: a builder, and random
lists over an arena of narrow and wide groups that cover every op, every Progress method and every kind of command
the single calls refuse."""
import numpy as np

from helpers import B

CTL_OPS = 15
NO_TERM_START = B.NO_TERM_START
META_WIDE_LO, META_WIDE_HI = 0x20000000, 0x40000000   # RAFTGPU_META_WIDE_*


def cmds(*rows) -> np.ndarray:
    """rows of (op, group, peer_slot=0, arg=0, a=()) -> a CTL_CMD_DTYPE array."""
    out = np.zeros(len(rows), dtype=B.CTL_CMD_DTYPE)
    for i, r in enumerate(rows):
        op, g, slot, arg, a = list(r) + [0, 0, ()][len(r) - 2:]
        out[i]["op"], out[i]["group"], out[i]["peer_slot"], out[i]["arg"] = op, g, slot, arg
        out[i]["a"][:len(a)] = a
    return out


def random_list(rng, n, groups, wide_lo, n_alloc):
    """About n commands over `groups` (group ids as the single calls take them; wide_lo: the set of wide low halves),
    in shuffled order, several per group.  n_alloc: groups >= n_alloc are unallocated (refused with ERR_RANGE)."""
    rows = []
    groups = list(groups)
    while len(rows) < n:
        g = groups[rng.integers(len(groups))]
        wide = g in wide_lo
        peers = 16 if wide else 8
        lim = 0xFFFF if wide else 0xFF
        op = int(rng.integers(CTL_OPS))
        slot = int(rng.integers(peers))
        arg = 0
        a = [0, 0, 0, 0]
        r = rng.random()
        if op == B.CTL_SET_CONF:
            inc = int(rng.integers(1, lim + 1)) & int(rng.integers(0, lim + 1)) or 1
            out = int(rng.integers(0, lim + 1)) if rng.random() < 0.3 else 0
            learn = int(rng.integers(0, lim + 1)) & ~(inc | out) & lim if rng.random() < 0.4 else 0
            present = [p for p in range(peers) if (inc | out | learn) >> p & 1]
            slot = int(rng.choice(present)) if rng.random() < 0.85 else B.CTL_NO_SELF
            a = [inc, out, learn, int(rng.integers(1, 40))]
            if r < 0.05:
                a[0] |= lim + 1            # a mask too wide
            elif r < 0.08:
                slot = peers + int(rng.integers(0, 4))   # a self slot the group does not have
        elif op == B.CTL_RESET:
            li = int(rng.integers(0, 40))
            a = [NO_TERM_START if rng.random() < 0.3 else int(rng.integers(1, li + 2)), li,
                 int(rng.integers(0, li + 1)), int(rng.integers(0, li + 1))]
        elif op == B.CTL_SET_LOG_BOUNDS:
            li = int(rng.integers(0, 50))
            a = [int(rng.integers(1, li + 2)), li]
        elif op in (B.CTL_SET_TERM, B.CTL_COMMIT_TO, B.CTL_MAYBE_COMMIT_TO):
            a = [int(rng.integers(0, 50))]
        elif op in (B.CTL_SET_GROUP_COMMIT, B.CTL_RECORD_VOTE):
            arg = int(rng.integers(0, 2))
        elif op == B.CTL_ASSIGN_COMMIT_GROUP:
            a = [int(rng.integers(0, 4))]
        elif op == B.CTL_HAS_QUORUM:
            a = [int(rng.integers(0, 1 << 20))]   # the call masks to the group's slots
        elif op == B.CTL_PROGRESS_OP:
            arg = int(rng.integers(0, 19))
            a = [int(rng.integers(0, 45)), int(rng.integers(0, 45)), 0 if rng.random() < 0.7 else int(rng.integers(1, 45))]
            if r < 0.03:
                arg = 19 + int(rng.integers(0, 100))   # an unknown method
        if op in (B.CTL_RECORD_VOTE, B.CTL_ASSIGN_COMMIT_GROUP, B.CTL_PROGRESS_OP, B.CTL_QUORUM_RECENTLY_ACTIVE) \
                and r > 0.97:
            slot = peers + int(rng.integers(0, 8))    # a peer slot the group does not have
        gg = g
        if wide and rng.random() < 0.08:
            gg = g + 1                                # the high half named on its own
        if rng.random() < 0.01:
            gg = n_alloc + int(rng.integers(0, 16))   # an unallocated group
        if rng.random() < 0.005:
            op = CTL_OPS + int(rng.integers(0, 200))  # an unknown op
        rows.append((op, gg, slot, arg, a))
    return cmds(*rows)
