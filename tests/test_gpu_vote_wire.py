"""Vote responses at a candidate on the GPU (raftgpu_vote_wire[_device]) against the batch oracle
(oracle/vote_wire_oracle.c): the reference's election table, every status, random 100K-group elections with joint
configurations, learners, wide pairs and hostile frames, a 1M-group storm against INTEGRATION.md section 6's control
list on a twin arena, and the refusals (one buffer through every wire pass: test_gpu_wire_batches.py).  Run with
-m gpu."""
import ctypes as C

import numpy as np
import pytest

from oracle import vote_wire_oracle as VW
from helpers import B, arena_of, votes
from control_cmds import cmds
import hb_frames as F
import pass_forms as PF
import vote_frames as V

pytestmark = pytest.mark.gpu


# --------------------------------------------------------------------------- 1. the table and the statuses


@pytest.mark.parametrize("case", range(len(V.ONE_ROUND)))
def test_leader_election_in_one_round_rpc(case):
    size, votes, state = V.ONE_ROUND[case]
    a = B.Arena(64)
    assert a.group_alloc_range(1) == 0
    a.control(cmds((B.CTL_SET_CONF, 0, 0, 0, ((1 << size) - 1, 0, 0, 11)), (B.CTL_RESET, 0, 0, 0, (B.NO_TERM_START, 10, 5, 10))))
    camp = cmds((B.CTL_RESET, 0, 0, 0, (B.NO_TERM_START, 10, 5, 10)), (B.CTL_SET_TERM, 0, 0, 0, (1,)),
                (B.CTL_RESET_VOTES, 0), (B.CTL_RECORD_VOTE, 0, 0, 1), (B.CTL_VOTE_RESULT, 0))
    first = int(a.control(camp)["value"][-1])
    frames = [F.frame(0, k - 1, V.message(6, 1, not v, to=1, frm=k)) for k, v in votes.items()]
    st, outs = a.vote_wire(F.Frames(frames), V.bitmap([True]))
    assert np.all(st == (B.WIRE_OK << 4 | B.RES_OK))
    assert V.expected_state(first, outs) == state and len(outs) == (state != "Candidate" and bool(frames))
    a.close()


def test_statuses_match_the_oracle():
    """test_statuses_in_order's frames and arena through the C ABI (host form) and the device form."""
    meta = B.make_meta(0x1F, 0, 0, 0)
    for device in (False, True):
        a = B.Arena(64)
        assert a.group_alloc_range(4) == 0
        a.control(cmds(*[(B.CTL_SET_CONF, g, 0, 0, (0x1F, 0, 0, 11)) for g in range(4)],
                       *[(B.CTL_RESET, g, 0, 0, (11 if g == 2 else B.NO_TERM_START, 10, 5, 10)) for g in range(4)],
                       *[(B.CTL_SET_TERM, g, 0, 0, (7,)) for g in range(4)]))
        c, vt = V.candidates([meta] * 4, [7] * 4)
        c.term_start[2] = 11
        frames = [F.frame(9, 1, V.message(6, 7)), F.frame(0, 1, b"\x08"), F.frame(0, 1, V.message(4, 7)),
                  F.frame(3, 1, V.message(6, 7)), F.frame(2, 1, V.message(6, 7)), F.frame(0, 1, V.message(18, 7)),
                  F.frame(1, 1, V.message(6, 7)), F.frame(0, 1, V.message(6, 0)), F.frame(0, 1, V.message(6, 8)),
                  F.frame(1, 1, V.message(18, 6)), F.frame(1, 1, V.message(18, 8, True)),
                  F.frame(0, 2, V.message(6, 7, commit=6, commit_term=7)), F.frame(0, 2, V.message(6, 7, commit=6)),
                  F.frame(0, 3, V.message(6, 7, True)), F.frame(0, 2, V.message(6, 7, True)), F.frame(1, 1, V.message(18, 8)),
                  F.frame(1, 9, V.message(18, 7)), F.frame(0, 4, V.message(6, 7))]
        sel, pre = V.bitmap([True, True, True, False]), V.bitmap([False, True, False, False])
        want_st, want_out, _ = V.run_batch(c, vt, frames, [True, True, True, False], [False, True, False, False])
        blob, off = F.batch(frames)
        got = PF.device(a, "vote_wire", np.concatenate([blob, np.zeros(16, np.uint8)]), off, sel, pre,
                                           n_bytes=len(blob) + 16) if device else \
            a.vote_wire(F.Frames(frames), sel, pre)
        assert np.array_equal(got[0], want_st) and np.array_equal(got[1], want_out), (device, got, want_st, want_out)
        assert np.array_equal(votes(a, 4), vt[:, :4]) and np.count_nonzero(vt[:, :4]) == 4
        a.close()


# --------------------------------------------------------------------------- 2. random 100K-group elections


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_random_elections_vs_oracle(device):
    rng = np.random.default_rng(0x7077 + device)
    e = V.Election(rng, 96_000, 2_000)
    a = arena_of(e)
    c, vt = V.state_of(e)
    assert np.array_equal(votes(a, e.n), vt[:, :e.n])
    kinds = np.zeros(16, np.int64)
    for rnd in range(2):
        frames = e.frames(rng, commit_vote=True)
        frames = [frames[i] for i in rng.permutation(len(frames))]
        blob, off = F.batch(frames)
        sel = V.bitmap(np.isin(e.role, (V.PRE_CANDIDATE, V.CANDIDATE)) & (rng.random(e.n) < 0.95))  # some unselected
        sel = np.concatenate([sel, np.zeros(4, np.uint32)])
        pre = np.concatenate([e.pre(), np.zeros(4, np.uint32)])
        before = a.counters()["votes_tallied"]
        want_st, want_out, tallied = VW.batch(c, vt, blob, off, sel, pre)
        got_st, got_out = PF.device(a, "vote_wire", np.concatenate([blob, np.zeros(16, np.uint8)]), off, sel, pre,
                                           n_bytes=len(blob) + 16) if device else \
            a.vote_wire(F.Frames(frames), sel, pre)
        assert np.array_equal(got_st, want_st), (rnd, np.flatnonzero(got_st != want_st)[:5])
        assert np.array_equal(got_out, want_out), rnd
        assert np.array_equal(votes(a, e.n), vt[:, :e.n]), rnd
        assert a.counters()["votes_tallied"] - before == tallied
        kinds += np.bincount(got_st >> 4, minlength=16)
        assert len(want_out) > 10_000
    for k in (B.WIRE_OK, B.WIRE_DUP, B.WIRE_ROLE, B.WIRE_TERM, B.WIRE_SKIP_TYPE, B.WIRE_MALFORMED, B.WIRE_COMMIT_VOTE):
        assert kinds[k] > 100, (k, kinds)
    a.close()


# --------------------------------------------------------------------------- 3. the 1M-group storm


def _storm_list(groups, slots, granted):
    """Section 6 step 2: RECORD_VOTE + VOTE_RESULT per response."""
    out = np.zeros(2 * len(groups), B.CTL_CMD_DTYPE)
    out["group"] = np.repeat(groups, 2)
    out["op"][0::2], out["op"][1::2] = B.CTL_RECORD_VOTE, B.CTL_VOTE_RESULT
    out["peer_slot"][0::2], out["arg"][0::2] = slots, granted
    return out


def test_1m_storm_against_the_control_list():
    rng = np.random.default_rng(0x7078)
    n = 1_000_000
    arenas = []
    for _ in range(2):
        a = B.Arena(n)
        assert a.group_alloc_range(n) == 0
        arenas.append(a)
    g = np.arange(n, dtype=np.uint32)
    last = rng.integers(10, 1 << 30, n).astype(np.uint64)
    com = last - rng.integers(0, 10, n).astype(np.uint64)
    term = rng.integers(1, 1 << 30, n).astype(np.uint64)
    setup = np.zeros(5 * n, B.CTL_CMD_DTYPE)
    setup["group"] = np.tile(g, 5)
    setup["op"][:n], setup["peer_slot"][:n] = B.CTL_SET_CONF, 0
    setup["a"][:n, 0], setup["a"][:n, 3] = 0x1F, last + 1
    setup["op"][n:2 * n] = B.CTL_RESET                                        # section 6 step 1: the campaign
    setup["a"][n:2 * n] = np.stack([np.full(n, B.NO_TERM_START, np.uint64), last, com, last], 1)
    setup["op"][2 * n:3 * n], setup["a"][2 * n:3 * n, 0] = B.CTL_SET_TERM, term
    setup["op"][3 * n:4 * n] = B.CTL_RESET_VOTES
    setup["op"][4 * n:], setup["arg"][4 * n:] = B.CTL_RECORD_VOTE, 1
    for a in arenas:
        assert np.all(a.control(setup)["status"] == 0)
    # 4M responses, shuffled: each peer of every group answers once
    gs = np.repeat(g, 4)
    slots = np.tile(np.arange(1, 5, dtype=np.uint32), n)
    granted = (rng.random(4 * n) < 0.55).astype(np.uint32)
    perm = rng.permutation(4 * n)
    gs, slots, granted = gs[perm], slots[perm], granted[perm]
    e = np.zeros(4 * n, B.SYNTH_VOTE_DTYPE)
    e["hdr"], e["msg_type"], e["to"], e["from"] = gs << 4 | slots, 6, 1, slots + 1
    e["term"], e["reject"] = term[gs], 1 - granted
    blob, off = B.synth_encode_votes(e)
    st, out = PF.device(arenas[0], "vote_wire", blob, off, V.bitmap(np.ones(n, bool)), V.bitmap(np.zeros(n, bool)))
    assert np.all(st == (B.WIRE_OK << 4 | B.RES_OK))
    res = arenas[1].control(_storm_list(gs, slots, granted))
    assert np.all(res["status"] == 0)
    last_word = np.zeros(n, np.uint32)
    last_word[gs] = res["value"][1::2].astype(np.uint32)                     # (the last write of a group wins)
    decided = np.flatnonzero(last_word & 0xFF != B.VOTE_PENDING)
    assert np.array_equal(out["group"], decided) and np.array_equal(out["result"], last_word[decided])
    assert len(out) == n                                                     # 5 voters, every vote in: all decided
    assert np.array_equal(votes(arenas[0], n), votes(arenas[1], n))
    won = out["group"][(out["result"] & 0xFF) == B.VOTE_WON]
    win = np.zeros(2 * len(won), B.CTL_CMD_DTYPE)                            # section 6 step 3 on both arenas
    win["group"] = np.repeat(won, 2)
    win["op"][0::2], win["op"][1::2] = B.CTL_RESET, B.CTL_BECOME_LEADER
    win["a"][0::2] = np.stack([last[won] + 1, last[won], com[won], last[won]], 1)
    for a in arenas:
        assert np.all(a.control(win)["status"] == 0)
    c0, c1 = arenas[0].read_columns(n), arenas[1].read_columns(n)
    for name in B.COLUMNS:
        assert np.array_equal(getattr(c0, name), getattr(c1, name)), name
    assert np.array_equal(votes(arenas[0], n), votes(arenas[1], n))
    for a in arenas:
        a.close()


# --------------------------------------------------------------------------- 5. freed slots and the outcome bound


def test_freed_selected_groups_stay_within_capacity():
    """100 group slots of which 99 are freed (raftgpu_group_free leaves their term behind) but still selected, each hit
    by a response at that term: only the allocated group is recorded and listed, and with capacity = min(n, allocated)
    = 1 nothing is written past the first outcome, in either form."""
    a = B.Arena(128)
    assert a.group_alloc_range(100) == 0
    a.control(cmds(*[(B.CTL_SET_CONF, g, 0, 0, (0b11, 0, 0, 11)) for g in range(100)],
                   *[(B.CTL_SET_TERM, g, 0, 0, (4,)) for g in range(100)], (B.CTL_RECORD_VOTE, 0, 0, 1)))
    for g in range(1, 100):
        a.group_free(g)
    info = a.get_info()
    assert (info.hi, info.n_alloc) == (100, 1)
    assert np.all(a.column_read(B.COL_TERM, 0, 0, 100, np.uint64) == 4)
    frames = [F.frame(g, 1, V.message(6, 4)) for g in range(99, -1, -1)]
    blob, off = F.batch(frames)
    blob = np.concatenate([blob, np.zeros(16, np.uint8)])
    n, sel = len(frames), V.bitmap(np.ones(128, bool))
    want = [B.WIRE_ROLE << 4] * 99 + [B.WIRE_OK << 4 | B.RES_OK]
    # the device form, with a guard entry after the one outcome the capacity allows
    bufs = [a.device_alloc(x) for x in (len(blob), 4 * (n + 1), sel.nbytes, n, 16, 8)]
    d_b, d_o, d_s, d_st, d_out, d_c = bufs
    for p, x in ((d_b, blob), (d_o, off), (d_s, sel), (d_out, np.full(16, 0xEE, np.uint8))):
        a.h2d(p, x)
    a.vote_wire_device(d_b, len(blob) - 16, d_o, n, d_s, None, d_st, d_out, 1, d_c)
    a.synchronize()
    st, out, cnt = np.zeros(n, np.uint8), np.zeros(16, np.uint8), np.zeros(1, np.uint64)
    a.d2h(st, d_st), a.d2h(out, d_out), a.d2h(cnt, d_c)
    assert st.tolist() == want and cnt.tolist() == [1]
    assert out[:8].view(B.VOTE_OUTCOME_DTYPE).tolist() == [(0, B.VOTE_WON | 2 << 8)] and np.all(out[8:] == 0xEE)
    v = votes(a, 100)
    assert v[1, 0] == 2 and np.count_nonzero(v[:, 1:]) == 0
    for p in bufs:
        a.device_free(p)
    # the host form, on the same votes (or_insert: the second frame of group 0 finds its vote, result 0)
    st, outs = a.vote_wire(F.Frames(frames), sel)
    assert st.tolist() == want[:-1] + [B.WIRE_OK << 4] and outs.tolist() == [(0, B.VOTE_WON | 2 << 8)]
    a.close()


# --------------------------------------------------------------------------- 6. refusals


def test_refusals_before_any_launch():
    a = B.Arena(64)
    assert a.group_alloc_range(16) == 0
    a.control(cmds(*[(B.CTL_SET_CONF, g, 0, 0, (0x1F, 0, 0, 11)) for g in range(16)], *[(B.CTL_SET_TERM, g, 0, 0, (3,)) for g in range(16)]))
    L, h = a._L, a._h
    n = 16
    blob, off = F.batch([F.frame(g, 1, V.message(6, 3)) for g in range(n)])
    sel = V.bitmap(np.ones(64, bool))
    nb = len(blob)
    with PF.refusals(a, "vote_wire", blob, off, sel, None, capacity=n) as r:
        dev, d = r.call, r.args
        refused = [dev(cap=n - 1), dev(cap=0, out=None), dev(b=d["b"] + 4), dev(nb=1 << 32), dev(n=1 << 32, cap=1 << 32),
                   dev(s=None), dev(c=None), dev(st=None), dev(o=None), dev(b=None), dev(out=None)]
        assert refused == [B.ERR_INVALID] * len(refused), refused
        assert r.untouched()                                                     # nothing was launched
        assert np.all(votes(a, 16) == 0)
        cnt, outs = C.c_uint64(), np.zeros(n, B.VOTE_OUTCOME_DTYPE)
        assert L.raftgpu_vote_wire(h, blob.ctypes.data, nb, off.ctypes.data, n, sel.ctypes.data, None, None, outs.ctypes.data,
                                   n - 1, C.byref(cnt)) == B.ERR_INVALID
        # the capacity rule counts allocated groups: 16 of them, so 16 frames need 16
        assert dev(cap=16) == B.OK
        gc = r.read("c", np.zeros(1, np.uint64))
        assert gc.tolist() == [0] and np.all(votes(a, 16)[1] == 2)
    a.close()
