"""The 16-bit offset window of next_idx and peer_committed at the passes that rewrite a whole group in one call (the
bump of raftgpu_vote_request_wire, raftgpu_follower_term_wire and raftgpu_leader_term_wire: become_follower_arena,
reset_group) and at the wire step's later waves (several MsgAppendResponse frames of a cell applied in one call), for
the tests.  offset16.py holds the bounds and the generators of the fused step; these are the same edges for these
passes, with the Inflights windows filled:

- bump_edges16 sets every group of a voter scenario so that its reset lands its cells on the bounds: the new next_idx
  of every peer 2^15 - 1, 2^15 or 2^15 + 1 above matched 0, the self slot's next_idx at each distance of EDGE16_D from
  the table's persisted, its peer_committed (= committed) on either side of both bounds, and every kept peer_committed
  crossing the window one way or the other, or landing on its upper bound.
- wave_world builds leaders with full windows and scripted frames: in one call a wave moves a cell's next_idx or
  peer_committed out of the window and a later wave brings it back (or the reverse), and frames of wave 2 and later
  free full windows.
- bump_counts and wave_counts count the transitions from the oracle's columns, for the tests to assert that each
  one occurred."""
import numpy as np

from helpers import B, O, offset_of
from oracle import control_oracle as CO
from oracle import follow_term_oracle as FT
from oracle import leader_runs_oracle as LR
from oracle import leader_term_oracle as LT
from oracle import read_oracle as RO
from oracle import vote_request_oracle as VR
from offset16 import EDGE16_D, EDGE16_FITS, I16_MAX, I16_MIN, RESET16_LAST, edge_state16, fits16
import append_reject as R
import app_follow as A
import follow_term as T
import leader_term as L
import vote_request_frames as Q

INS_CAP = 4
COMMIT16_D = (I16_MAX, I16_MAX + 1, I16_MIN + 1, I16_MIN, 0)   # committed - persisted: the self slot's new peer_committed
# how a kept peer_committed sits against the bump's new matched 0
(PC_ESCAPES, PC_RETURNS, PC_AT_MAX, PC_PAST_MAX, PC_ANY) = range(5)


def slot_masks(meta):
    """[SLOTS][n] bool each: the slots with a Progress, and the self slot."""
    m = meta.astype(np.int64)
    slot = np.arange(O.SLOTS)[:, None]
    present = (((m | m >> 8 | m >> 16) & 0xFF)[None, :] >> slot) & 1 == 1
    is_self = ((m & O.META_HAS_SELF) != 0)[None, :] & (((m >> 24) & 7)[None, :] == slot)
    return present, is_self


def ins_fill(groups, slots, first, k=INS_CAP):
    """RAFTGPU_POP_INS_ADD commands: k inflights first, first + 1, ... into each cell (group, slot)."""
    out = np.zeros(len(groups) * k, B.CTL_CMD_DTYPE)
    out["op"], out["arg"] = B.CTL_PROGRESS_OP, B.POP_INS_ADD
    out["group"], out["peer_slot"] = np.repeat(groups, k), np.repeat(slots, k)
    out["a"][:, 0] = np.repeat(np.asarray(first, np.uint64), k) + np.tile(np.arange(k, dtype=np.uint64), len(groups))
    return out


# --------------------------------------------------------------------------- the bump passes


def bump_edges16(s, c, rng, fill=0.5):
    """Every group of scenario s (Q.Scenario / follow_term.scenario, its oracle columns c of s.n groups) set for a
    bump at the 16-bit edges, in place on c, s.table["persisted"], s.last and s.committed:
    - last_index (a pair's larger half, either one) from RESET16_LAST, so that the reset's next_idx = last_index + 1
      sits 2^15 - 1, 2^15 or 2^15 + 1 (or far) above matched 0;
    - the table's persisted at each distance of EDGE16_D below last_index + 1 (the self slot's new next_idx - matched),
      and committed at a distance of COMMIT16_D above it (the self slot's new peer_committed - matched);
    - a leader's term_start at most committed, so that a share of them take MsgReadIndex requests into their queues;
    - each present cell's matched, next_idx and peer_committed such that the kept peer_committed fits before the bump
      and escapes after it (PC_ESCAPES: an old matched near it, above 2^20), escapes before and fits after (PC_RETURNS: an
      old matched near 2^20 and a small peer_committed), or lands at 2^15 - 1 or 2^15 (PC_AT_MAX, PC_PAST_MAX).
    A fraction `fill` of the other present cells become Replicate peers; the returned control list fills their windows
    (RAFTGPU_POP_INS_ADD up to INS_CAP, for an arena with enable_inflights(INS_CAP)).  Returns (commands, kind of every
    cell [SLOTS][n]).

    Not every state built here is one a Raft node reaches: committed may lie above last_index (d small, COMMIT16_D
    2^15 - 1 or 2^15), and an old matched, near 2^20 to 2^30, above a last_index near 2^15.  A live group keeps
    matched <= last_index and committed <= last_index, and its small last indexes leave no room for a kept
    peer_committed to cross the window.  The passes under test read none of these relations: a bump keeps committed
    and peer_committed as they are and re-encodes against the new matched, so these states reach the codec's bounds
    that the reachable ones at these last indexes cannot."""
    n = s.n
    lows = np.array(s.lows)
    k = len(lows)
    wide = s.wide[lows]
    last = np.array(RESET16_LAST, np.int64)[rng.integers(0, len(RESET16_LAST), k)]
    d = EDGE16_D[rng.integers(0, len(EDGE16_D), k)]
    last[last + 1 - d < 0] = RESET16_LAST[-1]
    persisted = last + 1 - d
    committed = persisted + np.array(COMMIT16_D)[rng.integers(0, len(COMMIT16_D), k)]
    committed = np.where(committed < 0, persisted + I16_MAX, committed)
    other_last = last - rng.integers(0, 4, k)
    other_com = np.maximum(committed - rng.integers(0, 4, k), 0)
    swap = rng.random(k) < 0.5                                            # the larger half is the high one
    c.last_index[lows] = np.where(swap & wide, other_last, last).astype(np.uint64)
    c.committed[lows] = np.where(swap & wide, other_com, committed).astype(np.uint64)
    hi = lows[wide] + 1
    c.last_index[hi] = np.where(swap, last, other_last)[wide].astype(np.uint64)
    c.committed[hi] = np.where(swap, committed, other_com)[wide].astype(np.uint64)
    s.table["persisted"][lows] = persisted.astype(np.uint64)
    lead = lows[c.term_start[lows] != B.NO_TERM_START]                  # a leader committed in its term: reads queue
    c.term_start[lead] = np.minimum(c.committed[lead], c.last_index[lead])
    c.term_start[lead[s.wide[lead]] + 1] = c.term_start[lead[s.wide[lead]]]
    for arr, v in ((s.last, last), (s.committed, committed)):
        arr[lows] = v.astype(np.uint64)
        arr[hi] = v[wide].astype(np.uint64)

    shape = (O.SLOTS, n)
    present, is_self = slot_masks(c.meta[:n])
    kind = rng.integers(0, 5, shape)
    far = rng.integers(1 << 20, 1 << 30, shape)
    pc = np.select([kind == PC_ESCAPES, kind == PC_RETURNS, kind == PC_AT_MAX, kind == PC_PAST_MAX],
                   [far + np.array(EDGE16_FITS)[rng.integers(0, len(EDGE16_FITS), shape)],
                    rng.integers(0, I16_MAX, shape), I16_MAX, I16_MAX + 1], rng.integers(0, 1 << 30, shape))
    m = pc - EDGE16_D[rng.integers(0, len(EDGE16_D), shape)]
    m = np.where((kind == PC_ESCAPES) | (kind == PC_RETURNS), far, np.where(m < 0, pc, m))
    nx = m + EDGE16_D[rng.integers(0, len(EDGE16_D), shape)]
    nx = np.where(nx < 0, m, nx)
    for col, v in (("matched", m), ("next_idx", nx), ("peer_committed", pc)):
        getattr(c, col)[:, :n] = np.where(present, v, getattr(c, col)[:, :n]).astype(np.uint64)
    rep = present & ~is_self & (rng.random(shape) < fill)
    c.pflags[:, :n][rep] = O.STATE_REPLICATE | O.PF_RECENT_ACTIVE
    ss, gs = np.nonzero(rep)
    return ins_fill(gs.astype(np.uint32), ss.astype(np.uint8), m[ss, gs] + 1), np.where(present, kind, -1)


def bump_counts(before, after, persisted, n, q_before=None, q_after=None):
    """Counts of the transitions the bumps made, from the oracle's columns before and after the pass (`persisted`: the
    table's per group slot, both halves of a pair) -> {name: count}.  A group is bumped where its term changed."""
    bumped = (after.term[:n] != before.term[:n])[None, :]
    present, is_self = slot_masks(after.meta[:n])
    peer, own = present & ~is_self & bumped, is_self & bumped
    mb, ma = before.matched[:, :n], after.matched[:, :n]
    pcb, pca, nxa = before.peer_committed[:, :n], after.peer_committed[:, :n], after.next_idx[:, :n]
    d_nx, d_pc = offset_of(nxa, ma), offset_of(pca, ma)
    out = {"peer next_idx - 0 at 2^15 - 1": peer & (d_nx == I16_MAX), "at 2^15": peer & (d_nx == I16_MAX + 1),
           "at 2^15 + 1": peer & (d_nx == I16_MAX + 2),
           "peer peer_committed fits, then escapes": peer & fits16(pcb, mb) & ~fits16(pca, ma),
           "peer peer_committed escaped, then fits": peer & ~fits16(pcb, mb) & fits16(pca, ma),
           "peer peer_committed at 2^15 - 1": peer & (d_pc == I16_MAX),
           "peer peer_committed at 2^15": peer & (d_pc == I16_MAX + 1)}
    assert np.array_equal(ma[peer], np.zeros(np.count_nonzero(peer), np.uint64))
    pers = np.broadcast_to(np.asarray(persisted, np.uint64)[:n], ma.shape)
    assert np.array_equal(ma[own], pers[own])
    for dd in EDGE16_D.tolist():
        out[f"self next_idx - persisted = {dd}"] = own & (d_nx == dd)
    for dd in COMMIT16_D:
        out[f"self peer_committed - persisted = {dd}"] = own & (d_pc == dd)
    out = {k: int(np.count_nonzero(v)) for k, v in out.items()}
    if getattr(before, "ins_cap", 0):
        full = ((before.ins_meta[:, :n] >> 16) == before.ins_cap) & bumped
        emptied = full & ((after.ins_meta[:, :n] >> 16) == 0) & ((after.pflags[:, :n] & O.PF_INS_FULL) == 0)
        out["full window emptied"] = int(np.count_nonzero(emptied))
        out["full window kept"] = int(np.count_nonzero(full & ~emptied))
    if q_before is not None:
        had = (q_before.count[:n] > 0) & bumped[0]
        out["read queue emptied"] = int(np.count_nonzero(had & (q_after.count[:n] == 0)))
        out["read queue kept"] = int(np.count_nonzero(had & (q_after.count[:n] != 0)))
    return out


def read_requests(rng, groups, per_group=3, ctx0=1):
    """1..per_group MsgReadIndex requests (B.READ_REQ_DTYPE) to each listed group, in group order, distinct contexts."""
    k = rng.integers(1, per_group + 1, len(groups))
    reqs = np.zeros(int(k.sum()), B.READ_REQ_DTYPE)
    reqs["group"] = np.repeat(np.asarray(groups, np.uint32), k)
    reqs["ctx"] = ctx0 + np.arange(len(reqs), dtype=np.uint64)
    return reqs


FLOOR = 30                          # the fewest cells (groups for the read queues) of each transition a test asserts
ROLES = {"vote_request": (0.5, 0.15, 0.25, 0.1), "follower_term": (0.5, 0.15, 0.25, 0.1),
         "leader_term": (0.0, 0.0, 0.0, 1.0)}
BATCH = {"vote_request": VR.batch, "follower_term": FT.batch, "leader_term": LT.batch}


def bump_world(rng, name, n_narrow, n_wide):
    """A scenario for pass `name` (ROLES: its groups' roles) set by bump_edges16, its oracle columns with the windows
    filled and read requests queued -> (scenario, columns, votes, queues, fill commands, read requests).  The arena
    takes s.setup, then the columns (load_columns), then the fill commands and the requests."""
    s = T.scenario(rng, n_narrow, n_wide, p_role=ROLES[name])
    c, vt = Q.state_of(s)
    fill, _ = bump_edges16(s, c, rng)
    O.enable_inflights(c, INS_CAP)
    assert np.all(CO.arena_control(c, vt, fill)["status"] == 0)
    q = RO.ReadQueues(c.cap, 8)
    q.allocated[: s.n] = 1
    reqs = read_requests(rng, s.lows)
    q.request(c, reqs)
    return s, c, vt, q, fill, reqs


def bump_frames(rng, s, name):
    """The pass's own frames (the scenario's vote requests, T.frames or L.frames) to every group, shuffled."""
    if name == "vote_request":
        frames_ = s.frames(rng)
    elif name == "follower_term":
        frames_ = T.frames(rng, s, per_group=(1, 3))
    else:
        frames_ = L.frames(rng, s, per_group=(1, 3))[0]
    return [frames_[i] for i in rng.permutation(len(frames_))]


def persisted_of(s):
    """The table's persisted per group slot, a pair's on both halves (become_follower_arena reads the low half's)."""
    p = s.table["persisted"].copy()
    hi = np.arange(s.n_narrow + 1, s.n, 2)
    p[hi] = p[hi - 1]
    return p


def check_bump_counts(counts, name):
    """Every transition of bump_counts at least FLOOR times, none kept; read queues emptied only by leader_term (the
    other two passes bump no leader, and only a leader holds reads)."""
    for what, k in counts.items():
        if what.endswith("kept"):
            assert k == 0, (name, what, counts)
        elif what == "read queue emptied":
            assert (k >= FLOOR) == (name == "leader_term"), (name, what, counts)
        else:
            assert k >= FLOOR, (name, what, counts)


# --------------------------------------------------------------------------- the wire step's waves

# scripts of a cell's frames (wave_world)
(S_FREE_LATE, S_PC_OUT_BACK, S_PC_BACK_OUT, S_NEXT_OUT_BACK, S_NEXT_BACK_OUT, S_RANDOM) = range(6)
PEERS = range(1, 5)
MAX_FRAMES = 6


def wave_world(rng, n, edge_frac=0.15):
    """n narrow leaders x 5 voters (self slot 0), their leader-run rows, the control list that fills their windows
    (INS_CAP each) and one batch of 2-6 MsgAppendResponse frames per peer cell, the cells interleaved in arrival order
    -> (columns, rows, fill commands, blob, offsets, script of every cell [SLOTS][n]).

    Each leader's log ends at last_index, far above 2^20; its own term runs from term_start, an older term below.  A
    peer cell follows one script (the frames after it are random accepts, stale accepts and rejections with and
    without log_term):
    - S_FREE_LATE: a full window; the first frame is stale or matches below the window, a later one frees it;
    - S_PC_OUT_BACK: a full window; (a stale accept, then) an accept whose commit lands peer_committed 2^15 and more
      above matched, then one that raises matched to bring it back, onto 2^15 - 1 at the closest;
    - S_PC_BACK_OUT: peer_committed escaped above matched; an accept brings it back, a later commit escapes again;
    - S_NEXT_OUT_BACK: a Probe peer; (a stale accept, then) a rejection whose hint lands next_idx 2^15 - 1, 2^15 or
      2^15 + 1 below matched, then an accept (becomes Replicate, next_idx = matched + 1);
    - S_NEXT_BACK_OUT: a peer in the Raft::reset shape (matched 0, next_idx escaped); an accept near last_index, a
      rejection (becomes Probe), then a hinted rejection that lands next_idx 2^15 and more below matched;
    - S_RANDOM: a window partly filled, random frames.
    Then offset16.edge_state16 on a fraction edge_frac of the peer cells."""
    c = O.new_columns(n, n)
    term = rng.integers(3, 1 << 20, n)
    last = rng.integers(1 << 20, 1 << 32, n) + (1 << 18)
    ts = last - rng.integers(0, 1 << 12, n)
    c.term[:n], c.last_index[:n], c.term_start[:n] = term, last, ts
    c.committed[:n] = ts - 1 - rng.integers(0, 100, n)
    c.meta[:n] = O.make_meta(0x1F, self_slot=0)
    c.matched[0, :n], c.next_idx[0, :n], c.peer_committed[0, :n] = last, last + 1, c.committed[:n]
    c.pflags[0, :n] = O.STATE_REPLICATE
    rows = np.zeros(n, LR.ROW_DTYPE)
    rows["group"], rows["term"], rows["term_start"] = np.arange(n), term, ts
    rows["run_start"][:, 0], rows["run_term"][:, 0] = 1, rng.integers(1, term)

    shape = (O.SLOTS, n)
    script = np.full(shape, -1)
    script[1:5] = rng.choice(6, size=(4, n), p=(0.25, 0.2, 0.15, 0.15, 0.1, 0.15))
    m = (last - rng.integers(1 << 16, 1 << 17, n))[None, :] + rng.integers(0, 64, shape)
    span = np.select([rng.random(shape) < 0.6, rng.random(shape) < 0.5],
                     [rng.integers(5, 300, shape), I16_MAX + rng.integers(0, 3, shape)], I16_MAX - 1)
    nx = m + span                                                     # the window's last inflight is next_idx - 1
    pc = m - rng.integers(0, 200, shape)
    pc = np.where(script == S_PC_BACK_OUT, m + I16_MAX + 1 + rng.integers(0, 3, shape), pc)
    flags = np.full(shape, O.STATE_REPLICATE | O.PF_RECENT_ACTIVE)
    probe = script == S_NEXT_OUT_BACK
    nx = np.where(probe, m + 1, nx)
    flags = np.where(probe, O.STATE_PROBE | np.where(rng.random(shape) < 0.5, O.PF_PAUSED, 0), flags)
    reset = script == S_NEXT_BACK_OUT
    m, nx = np.where(reset, 0, m), np.where(reset, last[None, :] + 1, nx)
    flags = np.where(reset, O.STATE_PROBE, flags)
    peer = script >= 0
    c.matched[:, :n] = np.where(peer, m, c.matched[:, :n])
    c.next_idx[:, :n] = np.where(peer, nx, c.next_idx[:, :n])
    c.peer_committed[:, :n] = np.where(peer, pc, c.peer_committed[:, :n])
    c.pflags[:, :n] = np.where(peer, flags, c.pflags[:, :n])
    # the windows: INS_CAP inflights up to next_idx - 1 (full), or 1-3 of them for S_RANDOM
    win = peer & ~probe & ~reset
    cnt = np.where(script == S_RANDOM, rng.integers(1, INS_CAP, shape), INS_CAP)
    ss, gs = np.nonzero(win)
    k = cnt[ss, gs]
    j = np.concatenate([np.arange(x) for x in k]) if len(k) else np.zeros(0, np.int64)
    top = np.repeat(nx[ss, gs] - 1, k)
    sp = np.repeat(span[ss, gs] - 1, k)
    kk = np.repeat(k, k)
    fill = np.zeros(int(k.sum()), B.CTL_CMD_DTYPE)
    fill["op"], fill["arg"] = B.CTL_PROGRESS_OP, B.POP_INS_ADD
    fill["group"], fill["peer_slot"] = np.repeat(gs, k), np.repeat(ss, k)
    fill["a"][:, 0] = top - sp * (kk - 1 - j) // kk                    # rising, the last at next_idx - 1

    # the frames
    first_inflight = nx - 1 - (span - 1) * (INS_CAP - 1) // INS_CAP      # of a full window
    cells = []
    u = rng.random((O.SLOTS, n, 8))
    r = rng.integers(0, 1 << 62, (O.SLOTS, n, 8))
    for g in range(n):
        t, li = int(term[g]), int(last[g])
        for s in PEERS:
            sc = int(script[s, g])
            mm, nn, pp = int(m[s, g]), int(nx[s, g]), int(pc[s, g])
            uu, rr = u[s, g], r[s, g]
            fr = []
            if sc == S_FREE_LATE:
                fi = int(first_inflight[s, g])
                if uu[0] < 0.4:
                    fr.append(R.response(t, index=mm - int(rr[0] % 4), commit=int(rr[1] % (pp + 1))))   # stale
                elif uu[0] < 0.7:
                    fr.append(R.response(t, index=mm + int(rr[0] % max(1, fi - mm)) if fi > mm else mm))   # below
                else:
                    fr.append(R.response(t, index=max(mm - 1, 0), reject=True, hint=int(rr[0] % (mm + 1))))  # stale
                top_ = nn - 1 if uu[1] < 0.5 else nn - 1 - int(rr[2] % 3)
                fr.append(R.response(t, index=top_, commit=int(rr[3] % (top_ + 1))))
            elif sc == S_PC_OUT_BACK:
                if uu[2] < 0.4:                                           # (the crossings one wave later)
                    fr.append(R.response(t, index=mm - int(rr[5] % 3)))
                i1 = mm + 1 + int(rr[0] % 4)
                up = int(rr[1] % 3)
                fr.append(R.response(t, index=i1, commit=i1 + I16_MAX + 1 + up))
                fr.append(R.response(t, index=i1 + 1 + up + int(rr[2] % 3), commit=int(rr[3] % (i1 + 1))))
            elif sc == S_PC_BACK_OUT:
                i1 = pp - I16_MAX + int(rr[0] % 3)
                fr.append(R.response(t, index=i1, commit=int(rr[1] % (i1 + 1))))
                i2 = i1 + int(rr[2] % 3)
                fr.append(R.response(t, index=i2, commit=i2 + I16_MAX + 1 + int(rr[3] % 3)))
            elif sc == S_NEXT_OUT_BACK:
                if uu[2] < 0.5:
                    fr.append(R.response(t, index=mm - int(rr[5] % 3)))
                fr.append(R.response(t, index=nn - 1, reject=True, hint=mm - I16_MAX - 3 + int(rr[0] % 3)))
                fr.append(R.response(t, index=mm + 1 + int(rr[1] % 50), commit=int(rr[2] % (mm + 1))))
            elif sc == S_NEXT_BACK_OUT:
                i1 = li - int(rr[0] % 100)
                fr.append(R.response(t, index=i1, commit=int(rr[1] % (i1 + 1))))
                fr.append(R.response(t, index=i1 + 1 + int(rr[2] % 3), reject=True, hint=i1))
                fr.append(R.response(t, index=i1, reject=True, hint=i1 - I16_MAX - 1 - int(rr[3] % 3)))
            want = 2 + int(rr[4] % 5)
            hi_ = max(mm, 1)
            while len(fr) < want:
                x = rng.random()
                if x < 0.55:
                    hi_ = min(li, hi_ + int(rng.integers(0, 2000)))
                    fr.append(R.response(t, index=hi_, commit=int(rng.integers(0, hi_ + 1))))
                elif x < 0.7:
                    fr.append(R.response(t, index=int(rng.integers(0, hi_ + 1))))
                else:
                    lt = int(rng.integers(1, t + 1)) if rng.random() < 0.4 else 0
                    fr.append(R.response(t, index=int(rng.integers(0, li + 1)), reject=True,
                                         hint=int(rng.integers(0, li + 1)), log_term=lt))
            cells.append([A.frame(g, s, f) for f in fr])
    order = rng.permutation(sum(len(f) for f in cells))
    owner = np.repeat(np.arange(len(cells)), [len(f) for f in cells])[order]
    pos = [0] * len(cells)
    frames = []
    for cell in owner.tolist():
        frames.append(cells[cell][pos[cell]])
        pos[cell] += 1
    # a share of the cells onto the bounds (every slot but the peers' is kept as it was)
    keep = O.copy_columns(c)
    edge_state16(c, rng, frac=edge_frac)
    for col in ("matched", "next_idx", "peer_committed", "pflags", "pending_snapshot", "pending_request_snapshot"):
        arr, old = getattr(c, col), getattr(keep, col)
        arr[0], arr[5:] = old[0], old[5:]
    blob, off = A.batch(frames)
    return c, rows, fill, blob, off, script


WAVE_COUNTS = ("INS_FULL cleared", "full window emptied", "next_idx escapes", "next_idx returns",
               "peer_committed escapes", "peer_committed returns")


def wave_counts(c, rows, blob, off, waves, ww_leader):
    """What the frames of wave 2 and later of one call at `waves` did, from the wave oracle (ww_leader = WW.leader) run at
    j - 1 and j waves on copies of c: {name: cells}, summed over j = 2 .. waves."""
    n = c.n_groups
    out = dict.fromkeys(WAVE_COUNTS, 0)
    prev = O.copy_columns(c)
    ww_leader(prev, rows, blob, off, 1)
    for j in range(2, min(waves, MAX_FRAMES) + 1):             # (no cell has a frame for a later wave)
        cur = O.copy_columns(c)
        ww_leader(cur, rows, blob, off, j)
        fb, fa = (prev.pflags[:, :n] & O.PF_INS_FULL) != 0, (cur.pflags[:, :n] & O.PF_INS_FULL) != 0
        kb, ka = prev.ins_meta[:, :n] >> 16, cur.ins_meta[:, :n] >> 16
        out["INS_FULL cleared"] += int(np.count_nonzero(fb & ~fa))
        out["full window emptied"] += int(np.count_nonzero((kb == INS_CAP) & (ka == 0)))
        for name, col in (("next_idx", "next_idx"), ("peer_committed", "peer_committed")):
            xb = fits16(getattr(prev, col)[:, :n], prev.matched[:, :n])
            xa = fits16(getattr(cur, col)[:, :n], cur.matched[:, :n])
            out[f"{name} escapes"] += int(np.count_nonzero(xb & ~xa))
            out[f"{name} returns"] += int(np.count_nonzero(~xb & xa))
        prev = cur
    return out
