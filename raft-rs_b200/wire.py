"""Wire batches for the tests and bench.py (SURVEY 8(f4)): host buffers holding serialized
eraftpb.Message frames, filled from synthetic records by libraftgpu_synth.so.  Input generation only --
the decode itself is the CUDA path (raftgpu_step_begin_wire)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import binding as B


class WireBuffers:
    """Frames + offsets + leader-local records for one step, in the arena's pinned memory when an arena is
    given (so that the H2D copies are asynchronous), else in ordinary numpy arrays."""

    def __init__(self, arena, max_records: int, bytes_per_record: int = 48):
        self.arena = arena
        cap_b = max_records * bytes_per_record + 128
        if arena is not None:
            self.bytes = arena.host_alloc_bytes(cap_b)
            self._off_raw = arena.host_alloc_bytes(4 * (max_records + 2))
            self._rec_raw = arena.host_alloc_bytes(24 * max_records)
        else:
            self.bytes = np.zeros(cap_b, dtype=np.uint8)
            self._off_raw = np.zeros(4 * (max_records + 2), dtype=np.uint8)
            self._rec_raw = np.zeros(24 * max_records, dtype=np.uint8)
        self.offsets = self._off_raw.view(np.uint32)
        self.records = self._rec_raw.view(B.APPEND_RESP_DTYPE)
        self.n = self.n_bytes = self.n_records = 0

    def encode(self, recs: np.ndarray, term: np.ndarray | None = None):
        """records of one round -> frames (followers) + local records (leader); returns self."""
        nf, nb, nl = C.c_uint64(), C.c_uint64(), C.c_uint64()
        rc = B.synth_lib().raftgpu_synth_wire_encode(
            recs.ctypes.data, len(recs), None if term is None else term.ctypes.data, self.bytes.ctypes.data,
            len(self.bytes), self.offsets.ctypes.data, C.byref(nf), C.byref(nb), self.records.ctypes.data, C.byref(nl))
        if rc != B.OK:
            raise B.RaftGpuError(rc, "raftgpu_synth_wire_encode")
        self.n, self.n_bytes, self.n_records = nf.value, nb.value, nl.value
        return self

    def encode_heartbeats(self, recs: np.ndarray, term: np.ndarray | None = None):
        """REC_HEARTBEAT records -> MsgHeartbeatResponse frames, one per record in order (term, commit, and the ctx id of a
        REC_READ_CTX record as an 8-byte little-endian context when it is non-zero); returns self."""
        nf, nb = C.c_uint64(), C.c_uint64()
        rc = B.synth_lib().raftgpu_synth_wire_encode_heartbeats(
            recs.ctypes.data, len(recs), None if term is None else term.ctypes.data, self.bytes.ctypes.data,
            len(self.bytes), self.offsets.ctypes.data, C.byref(nf), C.byref(nb))
        if rc != B.OK:
            raise B.RaftGpuError(rc, "raftgpu_synth_wire_encode_heartbeats")
        self.n, self.n_bytes, self.n_records = nf.value, nb.value, 0
        return self

    def set_frames(self, frames: list[bytes], records: np.ndarray | None = None):
        """Arbitrary frames (tests): each already starts with its 4-byte header."""
        blob = b"".join(frames)
        self.bytes[: len(blob)] = np.frombuffer(blob, dtype=np.uint8)
        self.offsets[: len(frames) + 1] = np.concatenate([[0], np.cumsum([len(f) for f in frames])]).astype(np.uint32)
        self.n, self.n_bytes = len(frames), len(blob)
        self.n_records = 0 if records is None else len(records)
        if self.n_records:
            self.records[: self.n_records] = records
        return self

    def free(self):
        if self.arena is not None:
            for b in (self.bytes, self._off_raw, self._rec_raw):
                self.arena.host_free(b)
            self.arena = None
