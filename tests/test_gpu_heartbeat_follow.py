"""MsgHeartbeat frames at the follower on the GPU (raftgpu_follower_heartbeat[_device]) against the oracle
(oracle/hb_follow_oracle.c): random 100K-group follower arenas fed with raftgpu_heartbeat_frames output and hostile
frames, 1M followers with one heartbeat each, the refusals, and the whole heartbeat loop on one device -- leader frames
-> the transport's header rewrite -> the followers' responses -> back -> raftgpu_heartbeat_wire.  Run with -m gpu."""
import numpy as np
import pytest

from oracle import oracle as O
from oracle import hb_follow_oracle as HL
from oracle import hb_frames_oracle as HF
from oracle import hb_wire_oracle as H
from helpers import B
from control_cmds import cmds
import hb_follow as FL
import hb_frames as F
import pass_forms as PF
import read_cases as R

pytestmark = pytest.mark.gpu

P = 8
U64 = (1 << 64) - 1
OK_RESP = B.WIRE_OK << 4 | B.RES_OK


def _compare(a, c, q, blob, off, sel, ids, device, what):
    """One pass through the arena (host or device form) and through the oracle: every output and the group columns."""
    want = HL.follower_heartbeats(c, q, blob, off, sel, ids)
    if device:
        got = PF.device(a, "follower_heartbeat", blob, off, sel, ids)
    else:
        fb = F.Frames([])
        fb.bytes, fb.offsets, fb.n, fb.n_bytes = np.concatenate([blob, np.zeros(16, np.uint8)]), off, len(off) - 1, len(blob)
        full_ids, full_sel = np.zeros(a.cap, np.uint64), np.zeros((a.cap + 31) // 32, np.uint32)
        full_ids[:len(ids)], full_sel[:len(sel)] = ids[:a.cap], sel[:len(full_sel)]
        got = a.follower_heartbeat(fb, full_ids, full_sel)
    for k, name in enumerate(("status", "from", "response bytes", "response offsets", "totals")):
        assert np.array_equal(got[k], want[k]), (what, name, np.flatnonzero(got[k] != want[k])[:5]
                                                 if len(got[k]) == len(want[k]) else (len(got[k]), len(want[k])))
    s = FL.group_state(a, c.n_groups)
    for name, col in s.items():
        assert np.array_equal(col, getattr(c, name)[:c.n_groups]), (what, name)
    return want


# --------------------------------------------------------------------------- 1. random 100K-group follower arenas

N_NARROW, N_WIDE = 99_000, 500


def _leader_frames(seed, n_l):
    """raftgpu_heartbeat_frames of an arena of n_l leaders x 5 peers after two steps of synthetic traffic, with a read
    pending in three quarters of the groups -> [(term, commit, frame body)]."""
    rng = np.random.default_rng(seed)
    s = B.Synth(n_l, seed, k_peers=5)
    la = B.Arena(n_l)
    la.enable_read_index(P)
    assert la.group_alloc_range(n_l) == 0
    la.load_columns(s.initial)
    la.column_write(B.COL_TERM, 0, 0, rng.integers(1, 1000, n_l).astype(np.uint64))
    reqs = np.zeros(n_l, B.READ_REQ_DTYPE)
    reqs["group"], reqs["ctx"] = np.arange(n_l), rng.integers(0, 1 << 63, n_l, dtype=np.uint64)
    la.read_index_request(reqs[rng.random(n_l) < 0.75])
    for _ in range(2):
        la.step_begin_records(s.next_round().copy(), B.STEP_READ_COMMITTED)
        la.step_wait()
    rc, blob, off, tot = la.heartbeat_frames(0, n_l, rng.integers(1, 1 << 63, (9, n_l), dtype=np.uint64))
    assert rc == B.OK and int(tot[0]) > 3 * n_l
    la.close()
    out = []
    for _, body in FL.frames_of(blob, off):
        m = H.decode_message(body)
        out.append((m["term"], m["commit"], body))
    return out


def _hostile(rng, terms, k):
    """k frames that must not pass: garbage, unknown groups, truncated or foreign messages, bad contexts (at the group's
    term, so that they reach that check), term 0."""
    out, n_f = [], len(terms)
    for j in range(k):
        g, x = int(rng.integers(0, n_f)), int(rng.integers(16))
        kind = j % 7
        if kind == 0:
            out.append(F.frame(g, x, rng.integers(0, 256, int(rng.integers(0, 24)), dtype=np.uint8).tobytes()))
        elif kind == 1:
            out.append(F.frame(n_f + int(rng.integers(0, 100)), x, F.message(8, term=5, commit=1)))
        elif kind == 2:
            out.append(F.frame(g, x, F.message(8, term=5, commit=1 << 40, frm=3)[:-1]))
        elif kind == 3:
            out.append(F.frame(g, x, F.message(int(rng.choice([3, 4, 9, 17])), term=5, commit=1)))
        elif kind == 4:
            out.append(F.frame(g, x, F.message(8, term=int(terms[g]), commit=0, context=bytes(int(rng.choice([1, 4, 9, 16]))))))
        elif kind == 5:
            out.append(F.frame(g, x, F.message(8, term=0, commit=1)))
        else:
            out.append(np.array([g << 4 | x], "<u4").tobytes()[: int(rng.integers(0, 4))])
    return out


@pytest.mark.parametrize("reads", [True, False], ids=["read_queues", "no_read_queues"])
def test_random_arenas_vs_oracle(reads):
    rng = np.random.default_rng(0x4EF2 + reads)
    n = N_NARROW + 2 * N_WIDE
    a = B.Arena(n + 64)
    if reads:
        a.enable_read_index(P)
    assert a.group_alloc_range(N_NARROW) == 0
    for k in range(N_WIDE):
        assert a.group_alloc_wide() == N_NARROW + 2 * k
    leader = _leader_frames(0x4EF3 + reads, 25_000)
    nl = len(leader)
    # follower state shaped by the frames it will get: most terms and logs match, some do not
    fg = rng.integers(0, n, nl)
    terms = rng.integers(1, 1000, n).astype(np.uint64)
    last = rng.integers(0, 1 << 20, n).astype(np.uint64)
    lt = np.array([t for t, _, _ in leader], np.uint64)
    lc = np.array([c for _, c, _ in leader], np.uint64)
    hit = rng.random(nl) < 0.92
    terms[fg[hit]] = lt[hit]
    over = rng.random(nl) < 0.9
    last[fg[over]] = lc[over] + rng.integers(0, 40, int(over.sum())).astype(np.uint64)
    last[fg[~over]] = lc[~over] - np.minimum(lc[~over], rng.integers(1, 5, int((~over).sum())).astype(np.uint64))
    committed = last - np.minimum(last, rng.integers(0, 60, n).astype(np.uint64))
    term_start = np.where(rng.random(n) < 0.1, np.uint64(1), np.uint64(B.NO_TERM_START))
    for col, arr in ((B.COL_TERM, terms), (B.COL_LAST_INDEX, last), (B.COL_COMMITTED, committed), (B.COL_TERM_START, term_start)):
        a.column_write(col, 0, 0, arr)
    c = a.read_columns(n)
    c.term = a.column_read(B.COL_TERM, 0, 0, n, np.uint64)
    q = None
    if reads:
        q = R.RO.ReadQueues(c.cap, P)
        q.allocated[:n] = 1
    ids = FL.self_ids(rng, n)
    kinds = np.zeros(16, np.int64)
    for rnd, device in enumerate((False, True)):
        order = rng.permutation(nl)
        order = np.concatenate([order, order[rng.random(nl) < 0.15]])   # repeated heartbeats: DUP
        frames = [F.frame(int(fg[i]), int(rng.integers(16)), leader[i][2]) for i in order]
        frames += _hostile(rng, terms, nl // 20)
        frames = [frames[i] for i in rng.permutation(len(frames))]
        blob, off = F.batch(frames)
        sel = FL.bitmap(rng.random(n) < 0.85)
        st = _compare(a, c, q, blob, off, sel, ids, device, ("round", rnd))[0]
        kinds += np.bincount(st >> 4, minlength=16)
    assert kinds[B.WIRE_OK] > 20_000 and kinds[B.WIRE_DUP] > 5_000, kinds
    for k in (B.WIRE_MALFORMED, B.WIRE_SKIP_TYPE, B.WIRE_ROLE, B.WIRE_TERM, B.WIRE_CONTEXT, B.WIRE_COMMIT_RANGE):
        assert kinds[k] > 100, (k, kinds)
    a.close()


# --------------------------------------------------------------------------- 2. 1M followers, one heartbeat each

def test_1m_followers():
    rng = np.random.default_rng(0x4EF4)
    n = 1_000_000
    lc = O.new_columns(n, n)                                  # n leaders with one peer each (slot 1), as frame source
    lc.meta[:] = B.make_meta(0b11, 0, 0, 0)
    lc.term_start[:] = 1
    lc.term[:] = rng.integers(1, 1 << 33, n)
    lc.committed[:] = rng.integers(0, 1 << 40, n)
    lc.matched[1] = rng.integers(0, 1 << 40, n)
    q = R.RO.ReadQueues(n, 1)
    q.allocated[:] = 1
    q.count[:] = rng.random(n) < 0.75                         # 3/4 of the heartbeats carry an 8-byte context
    q.ctx[:, 0] = rng.integers(1, 1 << 63, n, dtype=np.uint64)
    lids = rng.integers(1, 1 << 63, (9, n), dtype=np.uint64)
    hb, hoff, htot = HF.bcast_heartbeats(lc, q, 0, n, lids)
    assert int(htot[0]) == n
    perm = rng.permutation(n).astype(np.uint32)               # leader g's follower: group perm[g]
    blob = FL.with_headers(hb, hoff, perm << 4 | rng.integers(0, 16, n).astype(np.uint32))
    commit = np.minimum(lc.matched[1], lc.committed)
    a = B.Arena(n)
    assert a.group_alloc_range(n) == 0
    terms, last = np.zeros(n, np.uint64), np.zeros(n, np.uint64)
    terms[perm] = lc.term
    last[perm] = commit + rng.integers(0, 1000, n).astype(np.uint64)
    short = rng.random(n) < 0.02
    last[perm[short]] = commit[short] - np.minimum(commit[short], np.uint64(1))
    committed = last - np.minimum(last, rng.integers(0, 2000, n).astype(np.uint64))
    for col, arr in ((B.COL_TERM, terms), (B.COL_LAST_INDEX, last), (B.COL_COMMITTED, committed),
                     (B.COL_TERM_START, np.full(n, B.NO_TERM_START, np.uint64))):
        a.column_write(col, 0, 0, arr)
    c = a.read_columns(n)
    c.term = terms.copy()
    sel = FL.bitmap(np.ones(n, bool))
    st = _compare(a, c, None, blob, hoff, sel, FL.self_ids(rng, n), True, "1M")[0]
    assert (st == OK_RESP).sum() > 0.95 * n and (st == B.WIRE_COMMIT_RANGE << 4).sum() > 0.01 * n
    a.close()


# --------------------------------------------------------------------------- 3. refusals

def test_refusals_before_any_launch():
    d = R.ArenaDriver(64)
    a = d.a
    for g in range(16):
        a.group_set_term(g, 3)
    before = FL.group_state(a, 64)
    L, h = a._L, a._h
    blob, off = F.batch([F.frame(g, 0, F.message(8, term=3, commit=0)) for g in range(16)])
    n = 16
    bound = B.follower_heartbeat_bound(n)
    assert bound == 60 * n
    sel, ids = FL.bitmap(np.ones(a.cap, bool)), np.arange(a.cap, dtype=np.uint64)
    nb = len(blob)
    with PF.refusals(a, "follower_heartbeat", blob, off, sel, ids) as r:
        dev, d = r.call, r.args
        big = (1 << 32) // 60 + 1                                 # the first n whose bound exceeds u32 offsets
        assert B.follower_heartbeat_bound(big - 1) < (1 << 32) <= B.follower_heartbeat_bound(big)
        refused = [dev(cap=bound - 1), dev(cap=0), dev(b=d["b"] + 4), dev(rb=d["rb"] + 8), dev(n=big, cap=60 * big),
                   dev(n=1 << 32, cap=U64), dev(nb=1 << 32), dev(s=None), dev(ro=None), dev(t=None)]
        assert refused == [B.ERR_INVALID] * len(refused), refused
        st, tot, rb = np.zeros(n, np.uint8), np.zeros(2, np.uint64), np.zeros(bound, np.uint8)
        ro = np.zeros(n + 1, np.uint32)
        host = lambda cap: L.raftgpu_follower_heartbeat(h, blob.ctypes.data, nb, off.ctypes.data, n, sel.ctypes.data, ids.ctypes.data,
                                                        st.ctypes.data, None, rb.ctypes.data, cap, ro.ctypes.data, tot.ctypes.data)
        assert host(bound - 1) == B.ERR_INVALID
        assert r.untouched()   # nothing was launched
        after = FL.group_state(a, 64)
        assert all(np.array_equal(before[k], after[k]) for k in before)
        # the exact bound is accepted
        assert host(bound) == B.OK and tot.tolist()[0] == 16 and np.all(st == OK_RESP)
    a.close()


# --------------------------------------------------------------------------- 4. the whole loop on one device

def test_full_loop_on_one_device():
    """Leader arena (read queues, 20K narrow + 200 wide groups) -> raftgpu_heartbeat_frames_device -> the transport
    rewrites every header on the device (leader cell (g, s) <-> follower group map[g, s], x = s) ->
    raftgpu_follower_heartbeat_device on a follower arena, a random subset unselected -> headers back ->
    raftgpu_heartbeat_wire_device.  Released reads, the leader's tracker and the followers' committed equal the same
    chain on the oracles."""
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(0x4EF5)
    n_narrow, n_wide = 20_000, 200
    n = n_narrow + 2 * n_wide
    la = B.Arena(n + 64)
    la.enable_read_index(P)
    assert la.group_alloc_range(n_narrow) == 0
    for k in range(n_wide):
        assert la.group_alloc_wide() == n_narrow + 2 * k
    d = R.OracleDriver(n, max_pending=P)
    for k in range(n_wide):
        lo = n_narrow + 2 * k
        d.c.meta[lo], d.c.meta[lo + 1] = R.META_WIDE_LO, R.META_WIDE_HI
    setup = R.random_setup(rng, n_narrow, n_wide)
    assert np.array_equal(la.control(setup), d.q.control(d.c, d.votes, setup))
    cells = [(g, int(s)) for g in range(n) for s in rng.choice(8, 3, replace=False)]
    ups = cmds(*[(B.CTL_PROGRESS_OP, g, s, B.POP_MAYBE_UPDATE, (int(rng.integers(0, 90)),)) for g, s in cells])
    assert np.array_equal(la.control(ups), d.q.control(d.c, d.votes, ups))  # matched > 0: heartbeats carry commits
    terms = np.zeros(la.cap, np.uint64)
    terms[:n] = rng.integers(1, 50, n)
    terms[n_narrow + 1:n:2] = terms[n_narrow:n:2]
    la.column_write(B.COL_TERM, 0, 0, terms[:n].copy())
    d.c.term[:] = 0
    d.c.term[:n] = terms[:n]
    reqs = R.random_requests(rng, n, 0.8, 1 << 40)
    res, _ = la.read_index_request(reqs)
    want_res, _ = d.q.request(d.c, reqs)
    assert np.array_equal(res, want_res)
    ids = rng.integers(1, 1 << 63, (9, n), dtype=np.uint64)
    # the followers: one group per leader cell, in a random order
    nf = 8 * n
    fmap = rng.permutation(nf).astype(np.int64)               # cell g * 8 + s -> follower group
    inv = np.argsort(fmap)
    fa = B.Arena(nf)
    assert fa.group_alloc_range(nf) == 0
    fterm = np.zeros(nf, np.uint64)
    fterm[fmap] = np.repeat(terms[:n], 8)                     # (a wide pair's high half has its low half's term)
    fterm[rng.random(nf) < 0.03] += np.uint64(1)              # some followers are at another term
    flast = rng.integers(0, 100, nf).astype(np.uint64)
    fcomm = flast - np.minimum(flast, rng.integers(0, 40, nf).astype(np.uint64))
    for col, arr in ((B.COL_TERM, fterm), (B.COL_LAST_INDEX, flast), (B.COL_COMMITTED, fcomm),
                     (B.COL_TERM_START, np.full(nf, B.NO_TERM_START, np.uint64))):
        fa.column_write(col, 0, 0, arr)
    fc = fa.read_columns(nf)
    fc.term = fterm.copy()
    fsel = FL.bitmap(rng.random(nf) < 0.8)
    fids = np.zeros(nf, np.uint64)
    fids[fmap] = ids[np.arange(nf) % 8, np.arange(nf) // 8]  # the follower of cell (g, s) is peer s's id

    # the oracle chain
    hb, hoff, htot = HF.bcast_heartbeats(d.c, d.q, 0, n, ids)
    lh = FL.headers(hb, hoff)
    to_f = FL.with_headers(hb, hoff, (fmap[(lh >> 4) * 8 + (lh & 15)] << 4 | (lh & 15)).astype(np.uint32))
    fst, _, rb, ro, rt = HL.follower_heartbeats(fc, None, to_f, hoff, fsel, fids)
    rh = FL.headers(rb, ro)
    back = FL.with_headers(rb, ro, ((inv[rh >> 4] // 8) << 4 | (rh & 15)).astype(np.uint32))
    wst, want_rel = H.apply(d.c, d.q, back, ro, terms)
    assert (fst == OK_RESP).sum() > 0.5 * len(fst) and (fst == B.WIRE_ROLE << 4).sum() > 0.1 * len(fst)
    assert (fst == B.WIRE_COMMIT_RANGE << 4).sum() > 100 and len(want_rel) > 500

    # the device chain: every buffer a torch tensor, every step on torch's current stream
    dev = torch.device("cuda", la.info.device)
    stream = torch.cuda.current_stream(dev).cuda_stream
    u8 = lambda k: torch.zeros(max(16, k), dtype=torch.uint8, device=dev)
    i32 = lambda k: torch.zeros(max(1, k), dtype=torch.int32, device=dev)
    i64 = lambda k: torch.zeros(max(1, k), dtype=torch.int64, device=dev)
    bound = B.heartbeat_frames_bound(n)
    t_ids = torch.from_numpy(ids.view(np.int64)).to(dev)
    t_blob, t_off, t_tot = u8(bound), i32(8 * n + 1), i64(3)
    la.heartbeat_frames_device(0, n, None, t_ids.data_ptr(), t_blob.data_ptr(), bound, t_off.data_ptr(), 8 * n, t_tot.data_ptr(),
                               stream=stream)
    frames, nbytes = (int(x) for x in t_tot[:2].cpu())
    t_fmap, t_inv = torch.from_numpy(fmap).to(dev), torch.from_numpy(inv).to(dev)

    def rewrite(blob_t, off_t, count, fn):                   # the transport: headers read, mapped and written in place
        o = off_t[:count].to(torch.int64)
        b = blob_t.to(torch.int64)
        hdr = b[o] | (b[o + 1] << 8) | (b[o + 2] << 16) | (b[o + 3] << 24)
        new = fn(hdr)
        for k in range(4):
            blob_t[o + k] = ((new >> (8 * k)) & 0xFF).to(torch.uint8)

    rewrite(t_blob, t_off, frames, lambda h: t_fmap[(h >> 4) * 8 + (h & 15)] << 4 | (h & 15))
    t_sel = torch.from_numpy(fsel.view(np.int32)).to(dev)
    t_fids = torch.from_numpy(fids.view(np.int64)).to(dev)
    rbound = B.follower_heartbeat_bound(frames)
    t_st, t_from, t_rb, t_ro, t_rt = u8(frames), i64(frames), u8(rbound), i32(frames + 1), i64(2)
    fa.follower_heartbeat_device(t_blob.data_ptr(), nbytes, t_off.data_ptr(), frames, t_sel.data_ptr(), t_fids.data_ptr(),
                                 t_st.data_ptr(), t_from.data_ptr(), t_rb.data_ptr(), rbound, t_ro.data_ptr(), t_rt.data_ptr(),
                                 stream=stream)
    resp, rbytes = (int(x) for x in t_rt.cpu())
    rewrite(t_rb, t_ro, resp, lambda h: (t_inv[h >> 4] // 8) << 4 | (h & 15))
    cap = min(resp, la.get_info().n_alloc) * P
    t_wst, t_rel, t_cnt = u8(resp), u8(24 * max(1, cap)), i64(1)
    la.heartbeat_wire_device(t_rb.data_ptr(), rbytes, t_ro.data_ptr(), resp, t_wst.data_ptr(), t_rel.data_ptr(), cap,
                             t_cnt.data_ptr(), stream=stream)
    torch.cuda.synchronize(dev)

    assert [frames, nbytes] == htot[:2].tolist()
    assert np.array_equal(t_st.cpu().numpy()[:frames], fst)
    assert [resp, rbytes] == rt.tolist()
    assert np.array_equal(t_rb.cpu().numpy()[:rbytes], back) and np.array_equal(t_ro.cpu().numpy()[:resp + 1].view(np.uint32), ro)
    assert np.array_equal(t_wst.cpu().numpy()[:resp], wst)
    got_rel = t_rel.cpu().numpy()[: 24 * int(t_cnt.cpu()[0])].view(B.READ_STATE_DTYPE)
    g, w = R.by_group(got_rel), R.by_group(want_rel)
    assert len(g) == len(w) and np.array_equal(g, w)
    lc = la.read_columns(n)
    for name in ("matched", "next_idx", "peer_committed", "pflags", "committed"):
        assert np.array_equal(getattr(lc, name), getattr(d.c, name)[..., :n]), name
    cnt, _, _, _ = la.read_index_read(0, n)
    assert np.array_equal(cnt, d.q.count[:n])
    assert np.array_equal(fa.read_columns(nf).committed, fc.committed[:nf])
    la.close()
    fa.close()
