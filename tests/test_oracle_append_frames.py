"""The MsgAppend-frame oracle (oracle/app_frames_oracle.c): its encoder against python-protobuf's bytes
(tests/golden/wire/appends.json, scripts/gen_wire_append_golden.py), its frames decoded back to the fields they were
built from, the reference's send_append tests restated, and frames + rest list against the send list on random
arenas."""
import json
import os

import numpy as np

from oracle import app_frames_oracle as AF
from helpers import B, O
import app_frames as A
import read_cases as R

HERE = os.path.dirname(os.path.abspath(__file__))
U64 = A.U64
EDGES = {0, 1, 127, 128, 1 << 32, 1 << 63, U64}


def test_golden_vectors_encode_byte_for_byte():
    with open(os.path.join(HERE, "golden", "wire", "appends.json")) as f:
        vs = json.load(f)["vectors"]
    for v in vs:
        got = AF.encode_append(v["to"], v["from"], v["term"], v["log_term"], v["index"], v["commit"])
        assert got.hex() == v["hex"], v
        assert len(got) <= 68
    for name in ("to", "from", "term", "log_term", "index", "commit"):
        assert EDGES <= {v[name] for v in vs}, name
    # log_term 0 and index 0 with every other field set
    assert any(v["log_term"] == 0 and all(v[k] for k in ("to", "from", "term", "index", "commit")) for v in vs)
    assert any(v["index"] == 0 and all(v[k] for k in ("to", "from", "term", "log_term", "commit")) for v in vs)


def _want(c, first, n, ids, select):
    """The sends, restated from the columns: (frames [(g, s, fields)], rest [(g, s, flags, next_idx)], no_term)."""
    frames, rest, no_term = [], [], 0
    for g in range(first, first + n):
        lo = g - 1 if c.meta[g] & R.META_WIDE_HI else g
        if select is not None and not (int(select[lo // 32]) >> (lo % 32)) & 1:
            continue
        if c.term_start[lo] == R.NO_TERM_START:
            continue
        term = int(c.term[lo])
        if term == 0:
            no_term += lo == g
            continue
        wide = c.meta[lo] & R.META_WIDE_LO
        committed = int(max(c.committed[lo], c.committed[lo + 1])) if wide else int(c.committed[g])
        last = int(max(c.last_index[lo], c.last_index[lo + 1])) if wide else int(c.last_index[g])
        ts = int(c.term_start[lo])
        meta = int(c.meta[g])
        peers = (meta | meta >> 8 | meta >> 16) & 0xFF
        if meta & B.META_HAS_SELF:
            peers &= ~(1 << (meta >> 24 & 7))
        for s in range(8):
            if not peers >> s & 1:
                continue
            f = int(c.pflags[s, g])
            st = f & 3
            if (st == 0 and f & B.PF_PAUSED) or (st == 1 and f & B.PF_INS_FULL) or st == 2:
                continue
            nx = int(c.next_idx[s, g])
            snap = int(c.pending_request_snapshot[s, g]) != 0
            if snap or nx <= last or nx - 1 < ts:
                rest.append((g, s, int(snap), nx))
                continue
            frames.append((g, s, {"term": term, "log_term": term if nx - 1 <= last else 0, "index": nx - 1,
                                  "commit": committed, "lo": lo}))
    return frames, rest, no_term


def test_frames_decode_to_their_fields():
    """Random leaders of every configuration: each frame decodes through hwo_decode_message to exactly the fields
    prepare_send_entries + send give it, the rest list is the sends the log has to add to, both in (group, slot)
    order."""
    rng = np.random.default_rng(0xA99)
    n = 3000
    c = A.random_columns(rng, n, 200)
    ids = A.ids_for(rng, n)
    blob, offsets, rest, totals = AF.bcast_append(c, None, 0, n, ids)
    got = A.frames_of(blob, offsets)
    want_f, want_r, no_term = _want(c, 0, n, ids, None)
    assert totals.tolist() == [len(want_f), len(blob), len(want_r), no_term]
    assert len(want_f) > 1000 and len(want_r) > 2000 and no_term > 50
    assert offsets[0] == 0 and offsets[-1] == len(blob)
    for (g, s, m), (wg, ws, w) in zip(got, want_f):
        assert (g, s) == (wg, ws)
        assert m == {"msg_type": 3, "reject": 0, "to": int(ids[s, g]), "from": int(ids[8, w["lo"]]), "term": w["term"],
                     "log_term": w["log_term"], "index": w["index"], "commit": w["commit"], "commit_term": 0,
                     "request_snapshot": 0, "reject_hint": 0, "priority": 0, "context": b""}, (g, s)
    assert [tuple(map(int, r)) for r in rest[["group", "peer_slot", "flags", "next_idx"]].tolist()] == want_r
    assert any(m["log_term"] == 0 for _, _, m in got) and any(m["log_term"] != 0 for _, _, m in got)


def _one_leader(voters, term, term_start, last_index, committed):
    c = O.new_columns(8, 1)
    c.meta[0] = B.make_meta(voters, self_slot=0)
    c.term[0], c.term_start[0], c.last_index[0], c.committed[0] = term, term_start, last_index, committed
    c.matched[0, 0] = last_index
    return c


IDS3 = np.array([[1], [2], [3], [0], [0], [0], [0], [0], [1]], np.uint64)


def test_msg_append_response_wait_reset():
    """test_raft.rs:1484-1502 up to the commit broadcast: leader 1 of {1, 2, 3} at term 1 has its empty entry at index 1
    and sent it to both followers (3 is now a paused probe); node 2 acks index 1 (Replicate, next_idx 2) and the
    commit reaches 1.  bcast_append: one MsgAppend to node 2 with index 1, the leader's term and commit 1; node 3 gets
    nothing."""
    c = _one_leader(0b111, 1, 1, 1, 1)
    c.matched[1, 0], c.next_idx[1, 0], c.pflags[1, 0] = 1, 2, B.STATE_REPLICATE
    c.matched[2, 0], c.next_idx[2, 0], c.pflags[2, 0] = 0, 1, B.STATE_PROBE | B.PF_PAUSED
    blob, offsets, rest, totals = AF.bcast_append(c, None, 0, 1, IDS3)
    assert totals.tolist() == [1, len(blob), 0, 0] and len(rest) == 0
    [(g, s, m)] = A.frames_of(blob, offsets)
    assert (g, s) == (0, 1)
    assert (m["msg_type"], m["to"], m["from"], m["term"], m["log_term"], m["index"], m["commit"]) == (3, 2, 1, 1, 1, 1, 1)
    # node 3's probe resumed (a heartbeat response) would need entry 1: the rest list
    c.pflags[2, 0] = B.STATE_PROBE
    _, _, rest, totals = AF.bcast_append(c, None, 0, 1, IDS3)
    assert totals[:3].tolist()[0] == 1 and rest[["group", "peer_slot", "flags", "next_idx"]].tolist() == [(0, 2, 0, 1)]


def test_send_append_for_progress_replicate():
    """test_raft.rs:2830-2846: peer 2 in Replicate; each appended entry makes send_append send it: a rest entry with
    next_idx = the new entry, never a frame."""
    c = _one_leader(0b11, 1, 1, 1, 1)
    c.matched[1, 0], c.next_idx[1, 0], c.pflags[1, 0] = 0, 1, B.STATE_REPLICATE
    for k in range(10):
        c.last_index[0] = c.matched[0, 0] = 2 + k
        blob, _, rest, totals = AF.bcast_append(c, None, 0, 1, IDS3)
        assert totals.tolist() == [0, 0, 1, 0] and len(blob) == 0
        assert rest[["group", "peer_slot", "flags", "next_idx"]].tolist() == [(0, 1, 0, int(c.next_idx[1, 0]))]
        c.next_idx[1, 0] = c.last_index[0] + 1          # update_state (optimistic) after the host sent the entries
    # the window full: paused, nothing
    c.last_index[0] += 1
    c.pflags[1, 0] = B.STATE_REPLICATE | B.PF_INS_FULL
    assert AF.bcast_append(c, None, 0, 1, IDS3)[3].tolist() == [0, 0, 0, 0]


def test_send_append_for_progress_probe():
    """test_raft.rs:2848-2894: peer 2 in Probe; the first send_append sends entries from index 0 + 1 (a rest entry),
    then the probe is paused and nothing goes out until a heartbeat response resumes it."""
    c = _one_leader(0b11, 1, 1, 2, 1)
    c.matched[1, 0], c.next_idx[1, 0], c.pflags[1, 0] = 0, 1, B.STATE_PROBE
    _, _, rest, totals = AF.bcast_append(c, None, 0, 1, IDS3)
    assert totals.tolist() == [0, 0, 1, 0] and rest[["peer_slot", "next_idx"]].tolist() == [(1, 1)]
    c.pflags[1, 0] |= B.PF_PAUSED
    for k in range(10):
        c.last_index[0] += 1
        assert AF.bcast_append(c, None, 0, 1, IDS3)[3].tolist() == [0, 0, 0, 0]
    c.pflags[1, 0] = B.STATE_PROBE                       # the heartbeat response resumed it
    _, _, rest, totals = AF.bcast_append(c, None, 0, 1, IDS3)
    assert totals.tolist() == [0, 0, 1, 0] and rest[["peer_slot", "next_idx"]].tolist() == [(1, 1)]


def test_send_append_for_progress_snapshot():
    """test_raft.rs:2896-2913: a peer in Snapshot state gets nothing however many entries are appended; a
    pending_request_snapshot goes to the rest list with SNAPSHOT, caught up or not."""
    c = _one_leader(0b111, 1, 1, 1, 1)
    c.matched[1, 0], c.next_idx[1, 0], c.pflags[1, 0] = 0, 1, B.STATE_SNAPSHOT
    c.matched[2, 0], c.next_idx[2, 0], c.pflags[2, 0] = 1, 2, B.STATE_REPLICATE
    for k in range(10):
        c.last_index[0] = c.matched[0, 0] = 1 + k
        blob, offsets, rest, totals = AF.bcast_append(c, None, 0, 1, IDS3)
        assert all(s != 1 for _, s in A.frame_cells(blob, offsets)) and all(rest["peer_slot"] != 1)
    c.last_index[0], c.next_idx[2, 0] = 1, 2
    c.pending_request_snapshot[2, 0] = 7
    _, _, rest, totals = AF.bcast_append(c, None, 0, 1, IDS3)
    assert totals.tolist() == [0, 0, 1, 0]
    assert rest[["group", "peer_slot", "flags", "next_idx"]].tolist() == [(0, 2, B.SEND_SNAPSHOT, 2)]


def test_random_frames_and_rest_partition_the_send_list():
    """On random arenas the framed cells and the rest list are disjoint and together are the send list of the same
    selection, over the groups that send (allocated leaders with a term)."""
    rng = np.random.default_rng(0x5E9D)
    for n, n_wide, first, m, density in ((4000, 300, 0, 4000, None), (4000, 300, 96, 3000, 0.4), (2000, 0, 33, 1500, 0.7)):
        c = A.random_columns(rng, n, n_wide)
        sel = None if density is None else A.select_bits(rng, c.cap + 32, density)
        ids = A.ids_for(rng, m)
        blob, offsets, rest, totals = AF.bcast_append(c, None, first, m, ids, sel)
        framed = A.frame_cells(blob, offsets)
        listed = [(int(g), int(s)) for g, s in rest[["group", "peer_slot"]].tolist()]
        assert len(framed) > 200 and len(listed) > 200
        assert not set(framed) & set(listed)
        want = A.send_list_of_senders(c, first, m, sel)
        assert sorted(framed + listed) == sorted((int(g), int(s)) for g, s in want[["group", "peer_slot"]].tolist())
        # the rest list is the send list's entries, flags and next_idx included
        w = {(int(e["group"]), int(e["peer_slot"])): e for e in want}
        for e in rest:
            assert tuple(w[(int(e["group"]), int(e["peer_slot"]))].tolist()) == tuple(e.tolist())
