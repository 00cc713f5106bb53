"""The frame every step form shares, on a small arena: raftgpu_step_begin (enqueued records), _packed, _compact,
_records, _records(RAFTGPU_STEP_RAW) and _wire.

* a third step of any form with two in flight is refused with ERR_BUSY, and the two steps still complete;
* every form but raftgpu_step_begin is refused with ERR_INVALID after raftgpu_enqueue_*, and the enqueued step
  still runs;
* every raftgpu_step_result field equals what the batch implies, with and without READ_COMMITTED /
  READ_RESULTS: records, waves, groups, bytes each way, advanced groups (the oracle) and duplicates.

What the forms compute is checked against the oracle elsewhere; here the oracle only keeps the arena's expected
state and advanced count in step."""
import ctypes as C
import importlib

import numpy as np
import pytest

from helpers import B, O, assert_columns_equal

pytestmark = pytest.mark.gpu

W = importlib.import_module("raft-rs_b200.wire")

N = 30_000           # groups: a full round (~105K records) is large enough for the hybrid split (>= 65536 records)
PART = 3_000         # groups of a partial batch: < 16384 records, which the records API packs as ONE slice
CHUNK = 2048         # records per staging chunk (arena.cu kChunk)
BLOCK = 2048         # RAFTGPU_COMPACT_BLOCK
N_RINGS = 16         # the arena's default ring count
PK_EXT = 1 << 37     # packed record: EXT payload or padding
RC, RR = B.STEP_READ_COMMITTED, B.STEP_READ_RESULTS
FLAG_SETS = [0, RC, RR, RC | RR]
FORMS = ["ring", "packed", "compact", "records", "raw", "wire"]


def align16(x):
    return (x + 15) & ~15


class Rig:
    """One arena with the pinned buffers of every form and the oracle's copy of its state."""

    def __init__(self, seed):
        self.synth = B.Synth(N, seed, k_peers=5)
        self.a = B.Arena(N)
        assert self.a.group_alloc_range(N) == 0
        self.a.load_columns(self.synth.initial)
        self.ref = O.copy_columns(self.synth.initial)
        cap_recs = 5 * N + 64
        self.pk = self.a.host_alloc_packed(4 * cap_recs)
        self.blob = self.a.host_alloc_bytes(B.compact_bound(cap_recs))
        self.scratch = self.a.host_alloc_bytes(B.compact_bound(cap_recs))   # expected values only, never submitted
        self.pinned = self.a.host_alloc_bytes(24 * cap_recs).view(B.APPEND_RESP_DTYPE)
        self.wb = W.WireBuffers(self.a, cap_recs)
        # the set's pinned staging buffer, whose size fixes where the records API puts the units (meta_bytes)
        n_chunks = -(-max(4096, 5 * self.a.cap) // CHUNK) + N_RINGS
        self.meta_bytes = (64 + n_chunks * CHUNK * 16 // BLOCK + 4096) & ~4095

    def close(self):
        self.wb.free()
        self.a.close()

    def round(self, part=True):
        recs = self.synth.next_round().copy()
        if not part:
            return recs
        keep = recs["group"] < PART
        ext = (recs["flags"] & B.REC_EXT) != 0
        keep[1:][ext[1:]] = keep[:-1][ext[1:]]          # an EXT stays with its REJECT
        return np.ascontiguousarray(recs[keep])

    def applied(self, recs):
        O.arena_apply(self.ref, recs, mode=0)
        adv, _, _, _ = O.arena_recompute(self.ref)
        return adv

    def compact_hdr(self, recs):
        B.pack_compact(recs, self.scratch)
        return self.scratch[: B.COMPACT_HDR_DTYPE.itemsize].view(B.COMPACT_HDR_DTYPE)[0]

    def staged(self, recs):
        """raftgpu_enqueue_append_resp on one ring: (wave-0 chunks, later-wave packed records, later waves)."""
        k = self.a.pack_records(recs, self.scratch[: 16 * 4 * len(recs)].view(np.uint64).reshape(-1, 2))
        w0 = self.scratch[: 16 * k].view(np.uint64)[0::2]
        main = np.nonzero((w0 & np.uint64(PK_EXT)) == 0)[0]
        n_pk = np.diff(np.append(main, k)).tolist()
        m = (recs["flags"] & B.REC_EXT) == 0
        cells = ((recs["group"][m].astype(np.int64) << 3) | recs["peer_slot"][m]).tolist()
        assert len(cells) == len(n_pk)
        seen, fill, chunks, ov, depth = {}, CHUNK, 0, 0, 0
        for c, p in zip(cells, n_pk):
            d = seen.get(c, 0)
            seen[c] = d + 1
            if d:
                ov += p
                depth = max(depth, d)
                continue
            if fill + p > CHUNK:
                chunks, fill = chunks + 1, 0
            fill += p
        return chunks, ov, depth

    def begin(self, form, recs, flags):
        """Submit `recs` as `form`; returns the expected (n_records, n_waves, h2d_bytes, result bytes copied back)."""
        a, rr = self.a, bool(flags & RR)
        if form == "ring":
            a.enqueue(recs)
            a.step_begin(flags)
            chunks, ov, depth = self.staged(recs)
            slots = chunks * CHUNK + ov
            return len(recs), (1 + depth) if len(recs) else 0, 16 * slots, slots if rr else 0
        if form == "packed":
            k = a.pack_records(recs, self.pk)
            a.step_begin_packed(self.pk, k, flags)
            return k, 1 if k else 0, 16 * k, k if rr else 0
        if form == "compact":
            nb, _ = B.pack_compact(recs, self.blob)
            h = self.blob[: B.COMPACT_HDR_DTYPE.itemsize].view(B.COMPACT_HDR_DTYPE)[0]
            a.step_begin_compact(self.blob, nb, flags)
            n = int(h["n_records"])
            return n, 1 if n else 0, int(h["total_bytes"]), int(h["n_units"]) if rr else 0
        if form == "records":
            assert len(recs) < 16384          # one slice: the stream is exactly raftgpu_pack_compact's, in blocks
            a.step_begin_records(recs, flags)
            h = self.compact_hdr(recs)
            n, units = int(h["n_records"]), -(-int(h["n_units"]) // BLOCK) * BLOCK
            h2d = align16(self.meta_bytes + 4 * units) + align16(24 * int(h["n_side"]))
            return n, 1 if n else 0, h2d, units if rr else 0
        if form == "raw":
            a.step_begin_records(recs, flags | B.STEP_RAW)
            n = len(recs)
            return n, 1 if n else 0, 24 * n, n if rr else 0
        if form == "wire":
            wb = self.wb.encode(recs)
            a.step_begin_wire(wb, flags)
            n = wb.n + wb.n_records
            # the status bytes of every frame come back, with or without READ_RESULTS
            return n, 1 if n else 0, wb.n_bytes + 4 * (wb.n + 1) + 24 * wb.n_records, wb.n
        raise AssertionError(form)

    def check(self, r, want, flags, adv, what):
        n_records, n_waves, h2d, res_bytes = want
        d2h = 8 + 4 * ((N + 31) // 32) + (8 * N if flags & RC else 0) + res_bytes
        got = (r.n_records, r.n_waves, r.n_groups, r.h2d_bytes, r.d2h_bytes, r.n_advanced, r.n_duplicates)
        assert got == (n_records, n_waves, N, h2d, d2h, adv, 0), (what, got)


@pytest.fixture
def rig():
    r = Rig(0x5F4A3E)
    yield r
    r.close()


def test_every_form_reports_its_batch(rig):
    for flags in FLAG_SETS:
        for form in FORMS:
            recs = rig.round()
            want = rig.begin(form, recs, flags)
            r = rig.a.step_wait()
            rig.check(r, want, flags, rig.applied(recs), (form, flags))
    # later waves: the second and third record of a cell go to waves 1 and 2
    for flags in (RR, RC):
        recs = rig.round()
        plain = recs[(recs["flags"] & (B.REC_EXT | B.REC_REJECT)) == 0]
        recs = np.ascontiguousarray(np.concatenate([recs, plain[:300], plain[:100]]))
        want = rig.begin("ring", recs, flags)
        assert want[1] == 3
        r = rig.a.step_wait()
        rig.check(r, want, flags, rig.applied(recs), ("ring waves", flags))
    assert_columns_equal(rig.a.read_columns(N), rig.ref, N, "every form")


def test_full_rounds_async_and_hybrid(rig, monkeypatch):
    """Full rounds through the records API: several slices, asynchronous, and split with the raw form (the hybrid
    split at 50 %: the raw part is exactly the tail behind the first group boundary past half the batch)."""
    monkeypatch.setenv("RAFTGPU_HYBRID_PACK_PCT", "50")
    for extra in (B.STEP_ASYNC, B.STEP_HYBRID, B.STEP_HYBRID | B.STEP_ASYNC):
        for flags in (0, RC):
            recs = rig.round(part=False)
            k = len(recs)
            rig.pinned[:k] = recs
            rig.a.step_begin_records(rig.pinned[:k], flags | extra)
            c = k
            if extra & B.STEP_HYBRID:
                assert k >= 65536
                c = int(0.5 * k)
                while 0 < c < k and (recs["flags"][c] & B.REC_EXT or recs["group"][c] == recs["group"][c - 1]):
                    c += 1
            head = rig.compact_hdr(recs[:c])
            r = rig.a.step_wait()
            adv = rig.applied(recs)
            want_n = int(head["n_records"]) + (k - c)
            d2h = 8 + 4 * ((N + 31) // 32) + (8 * N if flags & RC else 0)
            got = (r.n_records, r.n_waves, r.n_groups, r.d2h_bytes, r.n_advanced, r.n_duplicates)
            assert got == (want_n, 1, N, d2h, adv, 0), (extra, flags, got)
            # several slices, each padded to a unit block (the stream's layout is the packer's): at least one unit
            # per packed record, at most the single-slice stream plus a block per slice (<= 64 slices)
            floor = rig.meta_bytes + 4 * int(head["n_records"]) + 24 * (k - c)
            top = rig.meta_bytes + 4 * (int(head["n_units"]) + 65 * BLOCK) + 24 * int(head["n_side"]) + 32 + 24 * (k - c)
            assert floor <= r.h2d_bytes <= top, (extra, flags, r.h2d_bytes, floor, top)
    assert_columns_equal(rig.a.read_columns(N), rig.ref, N, "full rounds")


def test_a_third_step_is_busy(rig):
    """With two steps in flight every form is refused with ERR_BUSY; both steps then complete as submitted."""
    third = rig.round()
    for form in FORMS + ["records async"]:
        e1, e2 = rig.round(), rig.round()
        want1 = rig.begin("records", e1, RC)
        want2 = rig.begin("ring", e2, RC | RR)
        with pytest.raises(B.RaftGpuError) as ei:
            if form == "records async":
                rig.a.step_begin_records(third, B.STEP_ASYNC)
            elif form == "ring":
                rig.a.step_begin(RC)
            else:
                rig.begin(form, third, RC)
        assert ei.value.status == B.ERR_BUSY, form
        r1 = rig.a.step_wait()
        rig.check(r1, want1, RC, rig.applied(e1), (form, "first"))
        r2 = rig.a.step_wait()
        rig.check(r2, want2, RC | RR, rig.applied(e2), (form, "second"))
    assert_columns_equal(rig.a.read_columns(N), rig.ref, N, "after ERR_BUSY")


def test_enqueued_records_do_not_mix(rig):
    """After raftgpu_enqueue_append_resp only raftgpu_step_begin may submit: every other form is refused with
    ERR_INVALID and the enqueued step still runs whole."""
    other = rig.round()
    recs = rig.round()
    rig.a.enqueue(recs)
    for form in FORMS[1:] + ["hybrid"]:
        with pytest.raises(B.RaftGpuError) as ei:
            if form == "hybrid":
                rig.pinned[: len(other)] = other
                rig.a.step_begin_records(rig.pinned[: len(other)], B.STEP_HYBRID | B.STEP_ASYNC)
            else:
                rig.begin(form, other, RC)
        assert ei.value.status == B.ERR_INVALID, form
        assert "cannot mix" in str(ei.value), form
    rig.a.step_begin(RC | RR)
    chunks, ov, depth = rig.staged(recs)
    r = rig.a.step_wait()
    rig.check(r, (len(recs), 1 + depth, 16 * (chunks * CHUNK + ov), chunks * CHUNK + ov), RC | RR,
              rig.applied(recs), "enqueued")
    assert_columns_equal(rig.a.read_columns(N), rig.ref, N, "after ERR_INVALID")


def test_record_results_of_other_forms_are_empty(rig):
    """raftgpu_step_record_results after a step of another form reports and writes nothing, even on the staging set
    whose last step was an enqueued one with later waves (the sets rotate: every third step reuses one).  The call
    gets a non-null buffer of capacity 0, as a caller with an empty buffer may pass."""
    recs = rig.round()
    plain = recs[(recs["flags"] & (B.REC_EXT | B.REC_REJECT)) == 0]
    recs = np.ascontiguousarray(np.concatenate([recs, plain[:300]]))
    want = rig.begin("ring", recs, RR)
    assert want[1] == 2
    rig.check(rig.a.step_wait(), want, RR, rig.applied(recs), "ring with a later wave")
    assert len(rig.a.record_results(0)) == len(recs)
    L, h = rig.a._L, rig.a._h
    out = np.full(len(recs) + 4096, 0xAB, dtype=np.uint8)    # covers every seq of the step above
    n = C.c_uint64(12345)
    for form in FORMS[1:]:
        for _ in range(3):
            recs = rig.round()
            want = rig.begin(form, recs, RR)
            rig.check(rig.a.step_wait(), want, RR, rig.applied(recs), form)
            assert L.raftgpu_step_record_results(h, 0, out.ctypes.data, 0, C.byref(n)) == B.OK, form
            assert n.value == 0, (form, n.value)
            assert np.all(out == 0xAB), (form, np.nonzero(out != 0xAB)[0][:5])
    assert_columns_equal(rig.a.read_columns(N), rig.ref, N, "after the other forms")
