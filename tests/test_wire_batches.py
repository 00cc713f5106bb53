"""The wire-batch geometry on the CPU: every wire oracle bounds a frame by the batch's length as wire_open does, the
stage rule of wire_stage_block restated, the batches test_gpu_wire_batches.py runs reaching every stage geometry in
every pass, so that the GPU tests cannot stop reaching the unstaged path unnoticed, and the golden decoder vectors
keeping their verdicts when retargeted to another message type."""
import numpy as np
import pytest

from oracle import oracle as O
from oracle import hb_follow_oracle as HL
from oracle import hb_wire_oracle as H
from oracle import vote_request_oracle as VR
from oracle import vote_wire_oracle as VW
from helpers import B
import hb_frames as F
import vote_frames as V
import vote_request_frames as Q
import wire_batches as WB

NO_TERM_START = (1 << 64) - 1


# --------------------------------------------------------------------------- 1. the oracles bound frames by n_bytes


def _columns(n=4):
    c = O.new_columns(16, n)
    c.term_start[:] = NO_TERM_START
    c.meta[:n] = O.make_meta(0b11)
    c.term[:n] = 7
    c.last_index[:n] = 10
    return c


def _statuses(blob, off, n_bytes):
    """Status (WIRE_*) of every frame in each batch oracle."""
    c = _columns()
    sel, ids = V.bitmap(np.ones(4, bool)), np.arange(1, 5, dtype=np.uint64)
    votes = np.zeros((O.SLOTS, c.cap), np.uint8)
    t = Q.voters(4)
    t["flags"] = VR.SELECT
    return {
        "append": O.wire_decode_batch(blob, off, 4, None, n_bytes)[0],
        "heartbeat": H.apply(c, None, blob, off, n_bytes=n_bytes)[0] >> 4,
        "follower": HL.follower_heartbeats(c, None, blob, off, sel, ids, n_bytes=n_bytes)[0] >> 4,
        "vote": VW.batch(c, votes, blob, off, sel, n_bytes=n_bytes)[0] >> 4,
        "voter": VR.batch(c, None, votes, blob, off, t, n_bytes=n_bytes)[0] >> 4,
    }


def test_oracles_bound_frames_by_n_bytes():
    """A blob of seven copies of one valid frame (a MsgAppend, SKIP_TYPE everywhere) with n_bytes = six of them:
    wire_open's verdicts for one-frame batches -- after a prefix, descending, ending past n_bytes while the bytes are
    there, ending exactly at n_bytes, 0 and 3 bytes long."""
    x = F.frame(1, 1, F.message(3, term=7, index=5))
    L = len(x)
    blob = np.frombuffer(x * 7, np.uint8).copy()
    cases = [((L, 2 * L), False), ((2 * L, L), True), ((6 * L, 7 * L), True), ((5 * L, 6 * L), False),
             ((5 * L, 6 * L + 1), True), ((L, L), True), ((L, L + 3), True), ((0, L), False)]
    for (a, b), malformed in cases:
        off = np.array([a, b], np.uint32)
        for name, st in _statuses(blob, off, 6 * L).items():
            assert st.tolist() == [B.WIRE_MALFORMED if malformed else B.WIRE_SKIP_TYPE], (name, a, b)
    # every frame of a batch, and n_bytes defaults to the whole blob
    off = np.array([5 * L, 6 * L, 5 * L, 6 * L, 7 * L], np.uint32)
    S, M = B.WIRE_SKIP_TYPE, B.WIRE_MALFORMED
    for n_bytes, want in ((None, [S, M, S, S]), (6 * L, [S, M, S, M])):
        for name, st in _statuses(blob, off, n_bytes).items():
            assert st.tolist() == want, (name, n_bytes)


def test_literal_forms_bound_frames_by_n_bytes():
    """The literal forms step no frame that ends past n_bytes: a granted vote response records no vote, a vote request
    gets no response."""
    resp = F.frame(0, 1, V.message(6, 7, to=1, frm=2))
    req = F.frame(0, 0, Q.request(Q.VOTE, 8, 7, 10, frm=2))
    for n_bytes, inside in ((len(resp), True), (len(resp) - 1, False)):
        c, votes = _columns(1), np.zeros((O.SLOTS, 16), np.uint8)
        blob, off = F.batch([resp])
        VW.literal(c, votes, np.full(1, VW.CANDIDATE, np.uint8), blob, off, n_bytes=n_bytes)
        assert votes[1, 0] == (2 if inside else 0)
    for n_bytes, inside in ((len(req), True), (len(req) - 1, False)):
        c, votes = _columns(1), np.zeros((O.SLOTS, 16), np.uint8)
        t = Q.voters(1)
        t["flags"] = VR.SELECT
        blob, off = F.batch([req])
        _, _, totals = VR.literal(c, None, votes, np.zeros(1, np.uint8), t, blob, off, n_bytes=n_bytes)
        assert totals[0] == inside


# --------------------------------------------------------------------------- 2. the stage rule


def test_stage_rule_restated():
    """wire_stage_block's three conditions, at their edges."""
    S = WB.STAGE
    cases = [([0, S], S, WB.STAGED), ([0, S + 1], S + 1, WB.SPAN), ([15, S], S, WB.STAGED),
             ([15, S + 1], S + 1, WB.SPAN), ([16, S + 16], S + 16, WB.STAGED), ([17, S + 17], S + 17, WB.SPAN),
             ([5, 4], 100, WB.ORDER), ([0, 101], 100, WB.PAST), ([5, 5], 100, WB.STAGED)]
    for off, n_bytes, want in cases:
        assert WB.stage_blocks(off, n_bytes) == [want], (off, n_bytes)
    # blocks of 256 frames: a block is judged on offsets[first] and offsets[min(first + 256, n)] only
    off = np.arange(0, 600 * 10, 10)
    off[255] = 10 ** 6
    assert WB.stage_blocks(off, off[-1]) == [WB.STAGED, WB.STAGED, WB.STAGED]
    off[256] = 10 ** 6
    assert WB.stage_blocks(off, off[-1]) == [WB.PAST, WB.ORDER, WB.STAGED]


def test_ballast_frames_are_exact_and_skipped():
    for size in list(range(8, 300)) + [16383, 16384, 16385, 16386, 16387, 16388, 65536, 70001]:
        for kind in (WB.MSG_APPEND, WB.MSG_SNAPSHOT):
            f = WB.ballast(size, kind)
            assert len(f) == size
            m = O.wire_decode_message(f[4:])
            assert m is not None and m["msg_type"] == kind and f[:4] == b"\0\0\0\0"


@pytest.mark.parametrize("name", ["append", "heartbeat", "follower", "vote", "voter"])
def test_gpu_batches_reach_every_stage_geometry(name):
    """The batches of test_gpu_wire_batches.py -- the stage batch and the hostile batches of both forms -- reach every
    geometry of WB.WANT_GEOMETRY in this pass (staging cannot be seen in any output: this is what shows the unstaged path
    ran)."""
    i = WB.PASSES.index(name)
    sc = WB.scenario(name)
    frames, ballast = WB.stage_batch(sc, 0x5B00 + i)
    blob, off = F.batch(frames)
    got = WB.geometry(off, len(blob))
    hostile = WB.scenario(name, 2_000)
    for device in (False, True):
        for buf, n_bytes, off in WB.hostile_batches(hostile, 0x5B10 + i, device):
            assert n_bytes % 16 in range(16) and (len(buf) - n_bytes >= 4096 if device else len(buf) == n_bytes)
            assert int(off.max()) <= (len(buf) if device else n_bytes + 4 * len(off))
            got |= WB.geometry(off, n_bytes)
    assert got >= WB.WANT_GEOMETRY, WB.WANT_GEOMETRY - got
    residues = {n_bytes % 16 for _, n_bytes, _ in WB.hostile_batches(hostile, 0x5B10 + i, True)}
    sizes = {len(off) - 1 for _, _, off in WB.hostile_batches(hostile, 0x5B10 + i, True)}
    assert residues == set(range(16)) and sizes == {1, 255, 256, 257}


# --------------------------------------------------------------------------- 3. the golden vectors, retargeted


@pytest.mark.parametrize("msg_type", sorted(set(WB.GOLDEN_TYPE.values())))
def test_retargeted_golden_vectors_keep_their_fields(msg_type):
    """Appending 0x08 <type> to an accepted messages.json vector changes its msg_type and nothing else (field 1 is a
    scalar: the last value wins), so python-protobuf's recorded fields stay the expected ones; a rejected vector stays
    rejected.  Both kinds the GPU test counts on are there."""
    vs = WB.golden()
    for v in vs:
        raw, fields = WB.retarget(v, msg_type)
        got = O.wire_decode_message(raw)
        if fields is None:
            assert got is None and raw == bytes.fromhex(v["hex"]), v["hex"]
            continue
        assert got is not None and fields["msg_type"] == msg_type, v["hex"]
        assert {k: got[k] for k in fields} == {k: int(x) for k, x in fields.items()}, v["hex"]
    kinds = {v["kind"] for v in vs if v["ok"]}
    assert {"non_canonical", "edge"} <= kinds and any(not v["ok"] for v in vs)
