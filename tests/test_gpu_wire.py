"""GPU parity of the wire path (SURVEY 8(f4)): serialized eraftpb.Message frames -> raftgpu_step_begin_wire
(varint decode + apply on the device) against the oracle (oracle/wire_oracle.c decode, then the same
ro_arena_apply / ro_arena_recompute every other path is checked with).  The decoder's own pinning is
tests/test_wire_oracle.py (python-protobuf vectors; "parity unpinned by the reference")."""
import importlib
import json
import os

import numpy as np
import pytest

from helpers import B, O, assert_columns_equal, bitmap_to_bool, checksum, oracle_wire_step

pytestmark = pytest.mark.gpu

W = importlib.import_module("raft-rs_b200.wire")
HERE = os.path.dirname(os.path.abspath(__file__))
FLAGS = B.STEP_READ_COMMITTED


def test_golden_messages_through_the_gpu():
    """Every golden vector as a frame (all message types, malformed bytes, term mismatches, rejections that need the
    log, second frames of a cell): status bytes and every column against the oracle."""
    with open(os.path.join(HERE, "golden", "wire", "messages.json")) as f:
        vs = json.load(f)["vectors"]
    n = 512
    s = B.Synth(n, 0x31AE, k_peers=5)
    a = B.Arena(n)
    assert a.group_alloc_range(n) == 0
    a.load_columns(s.initial)
    ref = O.copy_columns(s.initial)
    terms = np.zeros(a.cap, dtype=np.uint64)
    terms[:n:2] = 7
    a.column_write(B.COL_TERM, 0, 0, terms[:n].copy())
    frames = []
    for i, v in enumerate(vs):
        g, slot = (i * 7) % n, 1 + i % 7            # slots 5..7 have no Progress: RES_NO_PROGRESS
        if i % 11 == 0 and frames:
            g, slot = prev
        prev = (g, slot)
        frames.append(np.array([g << 4 | slot], dtype="<u4").tobytes() + bytes.fromhex(v["hex"]))
    frames.append(b"\x01\x02")
    frames.append(np.array([n << 4], dtype="<u4").tobytes() + bytes.fromhex("0804"))
    frames.append(np.array([3 << 4 | 9], dtype="<u4").tobytes() + bytes.fromhex("0804200730644063"))   # slot 9: no such slot
    wb = W.WireBuffers(a, len(frames) + 8, bytes_per_record=1024)
    wb.set_frames(frames)
    a.step_begin_wire(wb, FLAGS | B.STEP_READ_RESULTS)
    sr = a.step_wait()
    want, bm, adv, _ = oracle_wire_step(ref, wb, n, terms)
    got = a.wire_status().copy()
    bad = np.nonzero(got != want)[0]
    assert len(bad) == 0, [(int(i), hex(got[i]), hex(want[i]), vs[i]["hex"] if i < len(vs) else None) for i in bad[:5]]
    assert set(int(x) >> 4 for x in got) == {0, 1, 2, 3, 4, 5}
    assert_columns_equal(a.read_columns(n), ref, n, "golden frames")
    gbm, _ = a.step_results(n)
    assert np.array_equal(gbm, bm[: len(gbm)]) and sr.n_advanced == adv
    wb.free()
    a.close()


@pytest.mark.parametrize("joint", [False, True])
def test_synthetic_rounds_through_the_wire(joint):
    """cfg2-sized stream (100K groups): every round serialized the way a transport holds it, term check on;
    every column, the advanced bitmap, the commit indexes and the status bytes after every round."""
    n = 100_000
    s = B.Synth(n, 0x5EED0002, k_peers=5, joint=joint)
    a = B.Arena(n)
    assert a.group_alloc_range(n) == 0
    a.load_columns(s.initial)
    ref = O.copy_columns(s.initial)
    terms = np.zeros(a.cap, dtype=np.uint64)
    terms[:n] = s.initial.term[:n]
    a.column_write(B.COL_TERM, 0, 0, terms[:n].copy())
    wb = W.WireBuffers(a, 7 * n + 64)
    for rnd in range(4):
        recs = s.next_round().copy()
        wb.encode(recs, terms)
        assert wb.n + wb.n_records == int(np.count_nonzero((recs["flags"] & B.REC_EXT) == 0))
        if rnd == 2:       # a stale term on some frames of round 2: they must come back as WIRE_TERM, unapplied
            terms_sent = terms.copy()
            terms_sent[: n // 3] += 1
            wb.encode(recs, terms_sent)
        a.step_begin_wire(wb, FLAGS)
        sr = a.step_wait()
        want, bm, adv, _ = oracle_wire_step(ref, wb, n, terms)
        got = a.wire_status()
        assert np.array_equal(got, want), rnd
        if rnd == 2:
            assert np.count_nonzero((got >> 4) == B.WIRE_TERM) > n // 4
        assert sr.n_advanced == adv and sr.n_duplicates == 0
        gbm, com = a.step_results(n)
        assert np.array_equal(gbm, bm[: len(gbm)])
        advb = bitmap_to_bool(gbm, n)
        assert np.array_equal(com[advb], ref.committed[:n][advb])
        assert_columns_equal(a.read_columns(n), ref, n, f"wire round {rnd}")
    wb.free()
    a.close()


def test_wire_step_equals_record_step_at_1m():
    """Size-independent property at the headline size: the same rounds through raftgpu_step_begin_records (24-byte
    records) and through raftgpu_step_begin_wire (the frames a transport holds) leave identical arenas."""
    n = 1_000_000
    s = B.Synth(n, 0x5EED0003, k_peers=5)
    a1, a2 = B.Arena(n), B.Arena(n)
    for a in (a1, a2):
        assert a.group_alloc_range(n) == 0
        a.load_columns(s.initial)
    wb = W.WireBuffers(a2, 5 * n + 64)
    for rnd in range(3):
        recs = s.next_round().copy()
        a1.step_begin_records(recs, FLAGS)
        r1 = a1.step_wait()
        wb.encode(recs)
        a2.step_begin_wire(wb, FLAGS)
        r2 = a2.step_wait()
        assert r1.n_advanced == r2.n_advanced and r2.n_duplicates == 0
        st = a2.wire_status()
        assert np.all((st >> 4) == B.WIRE_OK)
        b1, c1 = a1.step_results(n)
        b2, c2 = a2.step_results(n)
        assert np.array_equal(b1, b2)
        adv = bitmap_to_bool(b1, n)
        assert checksum(c1[adv]) == checksum(c2[adv])
    g1, g2 = a1.read_columns(n), a2.read_columns(n)
    for name in ("matched", "next_idx", "peer_committed", "pflags", "committed", "last_index"):
        assert checksum(getattr(g1, name)) == checksum(getattr(g2, name)), name
    wb.free()
    a1.close()
    a2.close()
