"""Every wire-frame pass past the prologue it shares with the others (k_wire.cuh: wire_stage_block, wire_open), in its
host and device form, against its oracle: batches whose blocks lie on both sides of the 16 KiB stage (ballast frames
that every pass skips), hostile offset layouts, the golden decoder vectors through every decoder instantiation, and
one store's receive buffer through all five passes.  The batches and their scenarios are built on the CPU
(wire_batches.py; test_wire_batches.py checks the geometries they reach).  Run with -m gpu."""
import numpy as np
import pytest

from oracle import hb_follow_oracle as HL
from oracle import hb_wire_oracle as H
from oracle import vote_request_oracle as VR
from oracle import vote_wire_oracle as VW
from helpers import B, arena_of, assert_columns_equal, oracle_wire_step, votes
import hb_follow as FL
import hb_frames as F
import pass_forms as PF
import vote_frames as V
import vote_request_frames as Q
import wire_batches as WB

pytestmark = pytest.mark.gpu


# --------------------------------------------------------------------------- 1. across the stage


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("name", WB.PASSES)
def test_every_pass_across_the_stage(name, device):
    """A batch whose blocks are staged, unstaged by their span at 16384 / 16385 bytes from both ends of a 16-byte line,
    or hold frames past 16 KiB and 64 KiB, against the oracle; and the same frames without the ballast through a
    second arena: the same statuses and outputs for every frame, the same arena."""
    sc = WB.scenario(name)
    frames, ballast = WB.stage_batch(sc, 0x5B00 + WB.PASSES.index(name))
    blob, off = F.batch(frames)
    assert WB.geometry(off, len(blob)) >= {WB.STAGED, WB.SPAN, "frame>16K", "frame>64K"}
    a, st = sc.fresh()
    got = sc.run(a, st, blob, len(blob), off, device, (name, "ballast"))
    sc.check(a, st, (name, "ballast"))
    assert np.all(got[0][ballast] >> 4 == B.WIRE_SKIP_TYPE)
    assert np.count_nonzero(got[0][~ballast] >> 4 == B.WIRE_OK) > 1000
    # the oracle-free property: without the ballast, every other frame is decided the same way
    a2, st2 = sc.fresh()
    blob2, off2 = F.batch([f for f, b in zip(frames, ballast) if not b])
    got2 = sc.run(a2, st2, blob2, len(blob2), off2, device, (name, "plain"))
    for k, (x, y) in enumerate(zip(got, got2)):
        assert np.array_equal(x[~ballast] if k in sc.PER_FRAME else x, y), (name, "output", k)
    sc.check(a2, st, (name, "plain against the ballast run"))
    a.close()
    a2.close()


# --------------------------------------------------------------------------- 2. hostile offsets


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("name", WB.PASSES)
def test_hostile_offsets(name, device):
    """Descending offsets, frames past n_bytes, frames of 0 to 3 bytes, a valid frame before offsets[0], n_bytes at every
    residue mod 16 and n in {1, 255, 256, 257}: statuses equal the oracle's, and the arena stays the oracle's (a
    MALFORMED frame changes nothing).  The device form is the one that catches a missing `b > n_bytes` guard: its buffer
    holds valid frames past n_bytes, and its frames past n_bytes end on their boundaries.  The host form copies only the
    batch, and its offsets past n_bytes reach only the offsets the same call copies in (after at most 15 bytes left by
    the batch of valid frames it runs first); that keeps every read inside the staging buffer."""
    sc = WB.scenario(name, 2_000)
    a, st = sc.fresh()
    seen = np.zeros(16, np.int64)
    if not device:
        blob, off = F.batch(sc.frames(np.random.default_rng(1)))
        sc.run(a, st, blob, len(blob), off, False, (name, "valid"))
    for k, (buf, n_bytes, off) in enumerate(WB.hostile_batches(sc, 0x5B10 + WB.PASSES.index(name), device)):
        got = sc.run(a, st, buf, n_bytes, off, device, (name, k))[0]
        sc.check(a, st, (name, k))
        seen += np.bincount(got >> 4, minlength=16)
    assert seen[B.WIRE_MALFORMED] > 100 and seen[B.WIRE_SKIP_TYPE] + seen[B.WIRE_OK] > 100, seen
    a.close()


# --------------------------------------------------------------------------- 3. the golden encodings, every decoder


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("name", WB.PASSES)
def test_golden_encodings_through_every_decoder(name, device):
    """python-protobuf's verdicts on canonical, non-canonical and edge encodings (padded varints, repeated fields,
    unknown fields, known fields of the wrong wire type, 10-byte varints) through every wire_decode instantiation:
    every output against the oracle, so the fields each pass echoes or decides on -- from (3: d_from, d_out, the
    response's to), term, context (12), priority (14), commit_term (15) and commit -- are the golden ones.  A rejected
    vector is MALFORMED everywhere; both the non_canonical and the edge vectors reach OK."""
    seen = {}
    for variant in (0, 1) if name in ("vote", "voter") else (0,):
        sc, frames, kinds, ok = WB.golden_scenario(name, variant)
        blob, off = F.batch(frames)
        a, st = sc.fresh()
        got = sc.run(a, st, blob, len(blob), off, device, (name, variant))
        sc.check(a, st, (name, variant))
        a.close()
        status = got[0] >> 4
        assert np.all(status[~ok] == B.WIRE_MALFORMED), (name, variant)
        assert np.all(status[ok] != B.WIRE_MALFORMED), (name, variant, np.flatnonzero(ok & (status == B.WIRE_MALFORMED)))
        for k in ("non_canonical", "edge"):
            seen[k] = seen.get(k, 0) + int(np.count_nonzero((kinds == k) & (status == B.WIRE_OK)))
        seen["ok"] = seen.get("ok", 0) + int(np.count_nonzero(status == B.WIRE_OK))
    assert seen["non_canonical"] > 0 and seen["edge"] > 0 and seen["ok"] > len(frames) // 3, (name, seen)


# --------------------------------------------------------------------------- 4. one receive buffer, five passes


def test_store_buffer_through_every_pass():
    """One store's receive buffer -- MsgAppendResponse (4) and MsgHeartbeatResponse (9) to leaders, vote responses (6)
    to candidates, MsgHeartbeat (8) to followers, MsgRequestVote (5) and MsgRequestPreVote (17) to followers and
    candidates, and ballast -- through the five passes in a fixed order on one arena, each against its oracle on the
    shared oracle state: a frame is OK in at most one pass, and in the pass of its type whenever it is well-formed for
    it."""
    rng = np.random.default_rng(0x5B20)
    e = V.Election(rng, 6000, 0, p_role=(0.3, 0.2, 0.25, 0.25))
    n = e.n
    a = arena_of(e)
    c, vt = V.state_of(e)
    table = Q.voters(n)
    table["id"] = e.self_slot + 1
    table["last_term"] = e.term
    table["flags"] = np.where(e.role == V.LEADER, 0, B.VOTER_SELECT)
    follower = e.role == V.FOLLOWER
    ids = (e.self_slot + 1).astype(np.uint64)
    frames, kind = [], []
    for g in range(n):
        t, com, li = int(e.term[g]), int(e.committed[g]), int(e.last[g])
        peers = [s for s in range(1, 5) if int(e.present[g]) >> s & 1 and s != e.self_slot[g]]
        if e.role[g] == V.LEADER:
            for s in peers:
                frames += [F.frame(g, s, F.message(4, term=t, index=li)), F.frame(g, s, F.message(9, term=t, commit=com))]
                kind += [4, 9]
        if follower[g]:
            frames.append(F.frame(g, 1, F.message(8, term=t, commit=min(com, li), frm=2)))
            kind.append(8)
        if e.role[g] != V.LEADER and rng.random() < 0.5:
            typ = Q.PRE_VOTE if rng.random() < 0.5 else Q.VOTE
            frames.append(F.frame(g, 0, Q.request(typ, t + 1, t, li, frm=int(rng.integers(1, 6)))))
            kind.append(typ)
    for f in e.frames(rng, noise=False):
        frames.append(f)
        kind.append(6)
    order = rng.permutation(len(frames))
    frames, kind = [frames[i] for i in order], np.array(kind)[order]
    frames, ballast = WB.across_the_stage(frames, rng)
    kinds = np.zeros(len(frames), np.int64)
    kinds[~ballast] = kind
    blob, off = F.batch(frames)
    assert WB.geometry(off, len(blob)) >= {WB.STAGED, WB.SPAN, "frame>16K", "frame>64K"}
    nb = len(blob)
    terms = np.zeros(a.cap, np.uint64)
    terms[:n] = c.term[:n]
    sel_f, pad = FL.bitmap(follower), np.zeros(4, np.uint32)
    sel_v, pre_v = np.concatenate([e.select(), pad]), np.concatenate([e.pre(), pad])
    ok = []
    # 1. the AppendResponse step
    fb = PF.host_batch(blob, off, nb)
    fb.records = None
    a.step_begin_wire(fb)
    a.step_wait()
    got = a.wire_status().copy()
    want, _, _, _ = oracle_wire_step(c, fb, n, terms)
    PF.equal([want], [got], ["status"], "append")
    ok.append((got >> 4 == B.WIRE_OK, 4))
    # 2. heartbeat responses
    got, _ = a.heartbeat_wire(fb)
    want, _ = H.apply(c, None, blob, off, terms)
    PF.equal([want], [got], ["status"], "heartbeat")
    ok.append((got >> 4 == B.WIRE_OK, 9))
    # 3. vote responses
    got = a.vote_wire(fb, sel_v, pre_v)
    want = VW.batch(c, vt, blob, off, sel_v, pre_v)[:2]
    PF.equal(want, got, ("status", "outcomes"), "vote")
    ok.append((got[0] >> 4 == B.WIRE_OK, 6))
    # 4. heartbeats at the followers
    full_ids, full_sel = np.zeros(a.cap, np.uint64), np.zeros((a.cap + 31) // 32, np.uint32)
    full_ids[:n], full_sel[: len(sel_f)] = ids, sel_f
    got = a.follower_heartbeat(fb, full_ids, full_sel)
    want = HL.follower_heartbeats(c, None, blob, off, sel_f, ids)
    PF.equal(want, got, ("status", "from", "response bytes", "response offsets", "totals"), "follower")
    ok.append((got[0] >> 4 == B.WIRE_OK, 8))
    # 5. vote requests
    got = a.vote_request_wire(fb, table)
    want = VR.batch(c, None, vt, blob, off, table)
    PF.equal(want, got, ("status", "out", "response bytes", "response offsets", "totals"), "voter")
    ok.append((got[0] >> 4 == B.WIRE_OK, (5, 17)))
    assert_columns_equal(a.read_columns(n), c, n, "store buffer")
    assert np.array_equal(votes(a, n), vt[:, :n])
    assert np.array_equal(a.column_read(B.COL_TERM, 0, 0, n, np.uint64), c.term[:n])
    hits = np.stack([x for x, _ in ok])
    assert np.all(hits.sum(0) <= 1)
    for row, (x, k) in enumerate(ok):
        mine = np.isin(kinds, k)
        assert np.all(x <= mine) and x[mine].mean() > 0.5, (k, x[mine].mean())
    assert not hits[:, ballast].any()
    a.close()
