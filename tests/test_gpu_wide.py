"""GPU parity of WIDE groups (include/raftgpu.h raftgpu_group_alloc_wide): up to 16 peers as two consecutive
8-slot group slots.  The reference has no peer limit (majority.rs:86-93 sorts any number of voters on the heap);
this is how the engine covers configurations the 8-slot group cannot hold (ADVICE r1: "a joint change of two
disjoint 5-voter sets needs 10 slots").

  * the reference's own quorum vectors (src/quorum/testdata) replayed through a wide group whose peers straddle both
    halves;
  * random configurations of up to 16 voters against the oracle's quorum functions (majority.rs / joint.rs restated
    on id lists of any length);
  * whole steps -- every ingest path that accepts an arena with wide groups -- over arenas that mix ordinary and
    wide groups, column by column against the oracle; send list, heartbeat commits, vote tally likewise."""
import os
import random

import numpy as np
import pytest

from oracle import datadriven as dd
from helpers import B, O, assert_columns_equal, GpuQuorum, random_cell_batch, random_config_state

pytestmark = pytest.mark.gpu

WIDE_LO, WIDE_HI = 0x20000000, 0x40000000
# voter k of a test case -> peer slot of the wide group: alternate the halves so that every configuration of two or
# more voters is evaluated across both
SPREAD = [0, 8, 1, 9, 2, 10, 3, 11, 12, 4, 13, 5, 14, 6, 15, 7]


@pytest.fixture(scope="module")
def small():
    a = B.Arena(4096)
    yield a
    a.close()


class WideQuorum(GpuQuorum):
    def __init__(self, arena):
        self.a = arena
        arena.group_alloc()                 # an odd number of ordinary groups in front: the pair must still start even
        self.g = arena.group_alloc_wide()
        assert self.g % 2 == 0

    def _setup(self, incoming, outgoing, lookup, gc):
        ids = []
        for i in list(incoming) + list(outgoing):
            if i not in ids:
                ids.append(i)
        assert len(ids) <= 16
        slot = {i: SPREAD[k] for k, i in enumerate(ids)}
        m_in = sum(1 << slot[i] for i in set(incoming))
        m_out = sum(1 << slot[i] for i in set(outgoing))
        self.a.group_set_conf(self.g, 0, 0, 0, None, 1)
        self.a.group_set_conf(self.g, m_in, m_out, 0, None, 1)
        self.a.set_group_commit(self.g, gc)
        for i, s in slot.items():
            p = self.a.progress_get(self.g, s)
            p.matched, p.commit_group_id = lookup.get(i, (0, 0))
            self.a.progress_set(self.g, s, p)
        return slot


@pytest.mark.parametrize("name,count", [("majority_commit.txt", 16), ("joint_commit.txt", 50),
                                        ("joint_group_commit.txt", 14), ("majority_vote.txt", 22),
                                        ("joint_vote.txt", 39)])
def test_golden_vectors_through_a_wide_group(small, golden_dir, name, count):
    q = WideQuorum(small)
    cases = dd.replay_file(os.path.join(golden_dir, "quorum", name), q.impl())
    assert len(cases) == count
    for d, actual in cases:
        assert actual == d.expected, f"{d.pos}\n--- gpu (wide)\n{actual}--- expected\n{d.expected}"
    small.group_free(q.g)


def test_up_to_sixteen_voters_vs_oracle(small):
    """Random majority / joint configurations of 1..16 distinct voters (what an 8-slot group cannot hold), with and
    without group commit: committed index, use_group_commit and the vote result against majority.rs / joint.rs."""
    rng = random.Random(16)
    q = WideQuorum(small)
    big = 0
    for it in range(300):
        n_ids = rng.randrange(1, 17)
        ids = rng.sample(range(1, 40), n_ids)
        k = rng.randrange(0, n_ids + 1)
        inc = ids[:k] if rng.random() < 0.6 else ids
        out = rng.sample(ids, rng.randrange(0, n_ids + 1)) if rng.random() < 0.6 else []
        if not set(inc) | set(out):
            inc = ids
        used = list(dict.fromkeys(list(inc) + list(out)))
        big += len(used) > 8
        lookup = {i: (rng.randrange(0, 50), rng.randrange(0, 3)) for i in used if rng.random() < 0.9}
        gc = rng.random() < 0.4
        full = {i: lookup.get(i, (0, 0)) for i in used}
        want = O.joint_committed_index(inc, out, full, gc)
        got = q.joint(inc, out, lookup, gc)
        assert tuple(got) == tuple(want), (it, inc, out, lookup, gc)
        votes = {i: rng.random() < 0.6 for i in used if rng.random() < 0.8}
        assert q.joint_vote(inc, out, votes) == O.joint_vote_result(inc, out, votes), (it, inc, out, votes)
    assert big > 100
    small.group_free(q.g)


def test_wide_control_plane(small):
    """set_conf limits, has_quorum over 16-bit masks, quorum_recently_active across the halves, progress access by
    wide slot, commit_to / maybe_commit_to / group_get on the pair, free + reuse."""
    a = small
    g = a.group_alloc_wide()
    narrow = a.group_alloc()
    with pytest.raises(B.RaftGpuError) as e:      # nine peers do not fit an ordinary group
        a.group_set_conf(narrow, 0x1ff, 0, 0, 0, 1)
    assert e.value.status == B.ERR_TOO_MANY_PEERS
    with pytest.raises(B.RaftGpuError) as e:      # seventeen do not fit a wide one
        a.group_set_conf(g, 0x1ffff, 0, 0, 0, 1)
    assert e.value.status == B.ERR_TOO_MANY_PEERS
    # a joint change between two disjoint 5-voter sets + a learner: 11 peers, leader = peer 2
    inc, out, learn = 0b0000000000011111, 0b0000001111100000, 0b0000010000000000
    a.group_set_conf(g, inc, out, learn, 2, 5)
    a.group_reset(g, B.NO_TERM_START, 9, 4, 9)
    a.group_become_leader(g)                  # the noop at 10 = term_start = last_index, on both halves
    st = a.group_get(g)
    assert (st.term_start, st.last_index, st.committed) == (10, 10, 4)
    a.group_set_log_bounds(g, 5, 10)          # (for the test: entries 5.. are of the leader's term)
    for s in range(16):
        p = a.progress_get(g, s) if (inc | out | learn) >> s & 1 else None
        if p is not None:
            assert p.next_idx == 10 or s == 2
    assert a.has_quorum(g, 0b0000000011100111)          # 3 of each half
    assert not a.has_quorum(g, 0b0000000001100111)      # 2 of the outgoing half
    assert not a.has_quorum(g, 0b0000001111100011)      # 2 of the incoming half
    rng = random.Random(5)
    for _ in range(30):
        flags = {}
        for s in range(11):
            p = a.progress_get(g, s)
            p.recent_active = rng.randrange(0, 2)
            flags[s] = p.recent_active
            a.progress_set(g, s, p)
        me = rng.randrange(0, 11)
        act = {s + 1: True for s, f in flags.items() if f or s == me}
        want = O.joint_vote_result([1, 2, 3, 4, 5], [6, 7, 8, 9, 10], act) == O.VOTE_WON
        assert a.quorum_recently_active(g, me) == want
        for s in flags:
            assert a.progress_get(g, s).recent_active == (1 if s == me else 0)
    # acks through records: peers 8.. are (g + 1, slot - 8)
    recs = np.zeros(7, dtype=B.APPEND_RESP_DTYPE)
    recs[0] = (g, 2, B.REC_LOCAL, 0, 10, 10)
    recs[1] = (g, 0, 0, 0, 9, 0)
    recs[2] = (g, 1, 0, 0, 8, 0)
    recs[3] = (g, 5, 0, 0, 7, 0)
    recs[4] = (g, 6, 0, 0, 9, 0)
    recs[5] = (g + 1, 0, 0, 0, 6, 0)      # peer 8
    recs[6] = (g + 1, 2, 0, 0, 9, 0)      # peer 10, the learner: does not count
    a.enqueue(recs)
    r = a.step(B.STEP_READ_COMMITTED)
    # incoming {9, 8, 10, 0, 0} -> 8; outgoing {7, 9, 0, 6, 0} -> 6; joint = 6
    assert r.n_advanced == 1
    st = a.group_get(g)
    assert st.committed == 6 and a.maximal_committed_index(g)[0] == 6
    assert a.progress_get(g, 8).matched == 6 and a.progress_get(g, 2).committed_index == 6
    assert a.group_maybe_commit_to(g, 8) and a.group_get(g).committed == 8
    assert a.group_commit_to(g, 9) == 0 and a.group_get(g).committed == 9
    with pytest.raises(B.RaftGpuError):
        a.group_free(g + 1)                  # the pair is freed through its low half
    a.group_free(g)
    a.group_free(narrow)
    g2 = a.group_alloc()                      # the halves went back to the free list as ordinary slots
    a.group_set_conf(g2, 0b111, 0, 0, 0, 1)
    assert a.has_quorum(g2, 0b011)
    a.group_free(g2)


def _widen(c, n, rng, frac=0.3):
    """Turn a random subset of the even/odd pairs of `c` into wide groups: the halves share the group's log bounds,
    commit index, term and group-commit bit; the leader's own Progress lives in at most one half."""
    wide = np.zeros(n, dtype=bool)
    for g in range(0, n - 1, 2):
        if rng.random() >= frac:
            continue
        lo, hi = int(c.meta[g]), int(c.meta[g + 1])
        hi = (hi & ~O.META_GROUP_COMMIT) | (lo & O.META_GROUP_COMMIT)
        if (lo & O.META_HAS_SELF) and (hi & O.META_HAS_SELF):
            if rng.random() < 0.5:
                lo &= ~(O.META_HAS_SELF | (7 << 24))
            else:
                hi &= ~(O.META_HAS_SELF | (7 << 24))
        c.meta[g], c.meta[g + 1] = lo | WIDE_LO, hi | WIDE_HI
        for name in ("last_index", "term_start", "committed", "term"):
            getattr(c, name)[g + 1] = getattr(c, name)[g]
        wide[g] = True
    return wide


@pytest.mark.parametrize("seed", [11, 12])
def test_steps_over_mixed_ordinary_and_wide_groups(seed):
    """Arenas that mix ordinary and wide groups, random batches (accepts, leader-local records, rejections, several
    records per cell in the later rounds), through the ring path, bulk staging, the records API (compact stream and
    raw), the packed and compact zero-copy paths: columns, advanced bitmap, advanced count, commit indexes, then the
    send list, the heartbeat commits and the vote tally of the result -- all against the oracle."""
    rng = np.random.default_rng(seed)
    n = 3000
    init = random_config_state(n, rng)
    wide = _widen(init, n, rng)
    assert 300 < wide.sum() < 700
    ref = O.copy_columns(init)
    names = ["enqueue", "bulk", "records", "raw", "packed", "compact"]
    arenas = {}
    for name in names:
        a = B.Arena(32 * n if name in ("enqueue", "bulk", "records") else n)   # (room for the later waves)
        a.group_alloc_range(n)
        a.load_columns(init)
        arenas[name] = a
    pk_host = arenas["packed"].host_alloc_packed(40 * n)
    blob_host = arenas["compact"].host_alloc_bytes(B.compact_bound(40 * n))
    words = (n + 31) // 32
    adv_wide = 0
    for rnd in range(5):
        per_cell = 3 if rnd >= 3 else 1
        recs = random_cell_batch(ref, n, rng, per_cell)
        O.arena_apply(ref, recs, mode=0)
        want_adv, want_bm, _, _ = O.arena_recompute(ref)
        lo_bits, hi_bits = np.nonzero(wide)[0], np.nonzero(wide)[0] + 1
        assert not np.any(want_bm[hi_bits >> 5] >> (hi_bits & 31).astype(np.uint32) & 1)
        adv_wide += int(np.count_nonzero(want_bm[lo_bits >> 5] >> (lo_bits & 31).astype(np.uint32) & 1))
        for name in names:
            a = arenas[name]
            if per_cell > 1 and name in ("packed", "raw", "compact"):
                continue                      # zero-copy forms: one record per cell unless the fused kernel walks them
            if name == "enqueue":
                a.enqueue(recs)
                r = a.step(B.STEP_READ_COMMITTED)
            elif name == "bulk":
                a.enqueue_bulk(recs, sorted_by_group=True)
                r = a.step(B.STEP_READ_COMMITTED)
            elif name == "records":
                a.step_begin_records(recs, B.STEP_READ_COMMITTED)
                r = a.step_wait()
            elif name == "raw":
                a.step_begin_records(recs, B.STEP_READ_COMMITTED | B.STEP_RAW)
                r = a.step_wait()
            elif name == "packed":
                k = a.pack_records(recs, pk_host)
                a.step_begin_packed(pk_host, k, B.STEP_READ_COMMITTED)
                r = a.step_wait()
            else:
                nb, _ = B.pack_compact(recs, blob_host)
                a.step_begin_compact(blob_host, nb, B.STEP_READ_COMMITTED)
                r = a.step_wait()
            assert r.n_advanced == want_adv and r.n_duplicates == 0, (name, rnd)
            bm, com = a.step_results(n)
            assert np.array_equal(bm[:words], want_bm[:words]), (name, rnd)
            adv = np.unpackbits(bm[:words].view(np.uint8), bitorder="little")[:n].astype(bool)
            assert np.array_equal(com[adv], ref.committed[:n][adv]), (name, rnd)
            assert_columns_equal(a.read_columns(n), ref, n, f"{name}, round {rnd}, seed {seed}")
        if per_cell > 1:
            for name in ("packed", "raw", "compact"):
                arenas[name].load_columns(ref)

    assert adv_wide > 20          # wide groups did commit in these rounds
    a = arenas["records"]
    # send list of the last step (the high half follows the group's advanced bit)
    def as_set(e):
        return sorted(zip(e["group"].tolist(), e["peer_slot"].tolist(), e["flags"].tolist(), e["next_idx"].tolist()))
    want = O.arena_send_list(ref, want_bm)
    got = a.step_send_list(8 * n)
    assert as_set(got) == as_set(want)
    assert any((g - 1 >= 0) and wide[g - 1] for g in got["group"].tolist())
    # heartbeat commits (per half: both carry the group's commit index)
    d_out = a.device_alloc(8 * 8 * n)
    a.heartbeat_commits_device(0, n, d_out)
    hb = np.zeros((8, n), dtype=np.uint64)
    a.d2h(hb, d_out)
    assert np.array_equal(hb, O.arena_heartbeat_commits(ref, 0, n))
    # vote tally: both halves of a wide group report the result over its 16 peers
    votes = rng.integers(0, 3, (B.SLOTS, n), dtype=np.uint8)
    for s in range(B.SLOTS):
        a.column_write(B.COL_VOTES, s, 0, votes[s])
    d_t = a.device_alloc(4 * a.cap)
    a.tally_votes(0, n, d_t)
    got_t = np.zeros(a.cap, dtype=np.uint32)
    a.d2h(got_t, d_t)
    for g in range(n):
        gr, rj, res = O.arena_vote_result(ref, votes, g)
        assert int(got_t[g]) == res | (gr << 8) | (rj << 16), (g, bool(wide[g]), bool(g and wide[g - 1]))
    # maximal_committed_index of every wide group, one by one (mci_kernel)
    for g in np.nonzero(wide)[0][:200]:
        assert tuple(a.maximal_committed_index(int(g))) == tuple(O.arena_mci(ref, int(g)))
    for a in arenas.values():
        a.close()


def test_device_fused_entry_points_refuse_wide_arenas():
    a = B.Arena(1024)
    a.group_alloc_range(512)
    a.group_set_conf(0, 0b111, 0, 0, 0, 1)
    g = a.group_alloc_wide()
    assert g == 512
    pk = np.zeros((16, 2), dtype=np.uint64)
    d = a.device_alloc(pk.nbytes)
    d_off = a.device_alloc(4 * (1024 // B.tile_groups() + 2))
    with pytest.raises(B.RaftGpuError):
        a.step_sorted_device(d, 0, d_off)
    a.group_free(g)
    a.step_sorted_device(d, 0, d_off)         # no wide group left: allowed again
    a.close()
