"""ctypes binding of libraftgpu.so (include/raftgpu.h) for the tests and bench.py.

This is plumbing around the C-ABI: it never computes a quorum, a Progress
transition or a commit index itself -- every such call goes to the CUDA library
and raises when that fails (RAFTGPU_ERR_NO_DEVICE on a box without a GPU: there
is no CPU fallback).
"""
from __future__ import annotations

import ctypes as C
import os
import re
import types

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("RAFTGPU_LIB") or os.path.join(_HERE, "libraftgpu.so")   # (RAFTGPU_LIB: experimental builds)
SYNTH_LIB_PATH = os.path.join(_HERE, "libraftgpu_synth.so")
HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "raftgpu.h")
SYNTH_HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "raftgpu_synth.h")

SLOTS = 8
U64_MAX = (1 << 64) - 1
NO_TERM_START = U64_MAX

OK, ERR_INVALID, ERR_CUDA, ERR_NOMEM, ERR_NO_DEVICE, ERR_RANGE, ERR_FULL, ERR_PEER_NOT_FOUND, \
    ERR_COMMIT_RANGE, ERR_BUSY, ERR_TOO_MANY_PEERS = 0, -1, -2, -3, -4, -5, -6, -7, -8, -9, -10

STATE_PROBE, STATE_REPLICATE, STATE_SNAPSHOT = 0, 1, 2
VOTE_PENDING, VOTE_LOST, VOTE_WON = 0, 1, 2
PF_STATE_MASK, PF_PAUSED, PF_RECENT_ACTIVE, PF_INS_FULL = 0x03, 0x04, 0x08, 0x10
META_HAS_SELF, META_GROUP_COMMIT = 0x08000000, 0x10000000
REC_REJECT, REC_LOCAL, REC_HEARTBEAT, REC_EXT = 0x01, 0x02, 0x04, 0x80
RES_OK, RES_OLD_PAUSED, RES_NO_PROGRESS, RES_SEND = 0x01, 0x02, 0x04, 0x08
STEP_READ_COMMITTED, STEP_READ_RESULTS, STEP_ASYNC, STEP_RAW, STEP_HYBRID = 0x1, 0x2, 0x4, 0x8, 0x10
BULK_SORTED = 0x1
(POP_MAYBE_UPDATE, POP_MAYBE_DECR_TO, POP_UPDATE_COMMITTED, POP_OPTIMISTIC_UPDATE, POP_BECOME_PROBE,
 POP_BECOME_REPLICATE, POP_BECOME_SNAPSHOT, POP_SNAPSHOT_FAILURE, POP_MAYBE_SNAPSHOT_ABORT, POP_IS_PAUSED,
 POP_RESUME, POP_PAUSE, POP_UPDATE_STATE, POP_RESET, POP_INS_ADD, POP_INS_FREE_TO, POP_INS_FREE_FIRST_ONE,
 POP_INS_RESET, POP_INS_FULL) = range(19)

(COL_MATCHED, COL_NEXT_IDX, COL_PEER_COMMITTED, COL_PENDING_SNAPSHOT, COL_PENDING_REQ_SNAPSHOT,
 COL_COMMIT_GROUP_ID, COL_PFLAGS, COL_VOTES, COL_META, COL_COMMITTED, COL_TERM_START,
 COL_LAST_INDEX, COL_TERM, COL_INS_META) = range(14)
WIRE_OK, WIRE_SKIP_TYPE, WIRE_TERM, WIRE_NEEDS_LOG, WIRE_MALFORMED, WIRE_DUP, WIRE_CONTEXT = range(7)
WIRE_ROLE, WIRE_COMMIT_RANGE = 7, 8  # raftgpu_follower_heartbeat (ROLE also raftgpu_vote_wire)
WIRE_COMMIT_VOTE = 9  # raftgpu_vote_wire, raftgpu_vote_request_wire, raftgpu_leader_vote_request_wire
WIRE_IGNORED = 10  # raftgpu_vote_request_wire, raftgpu_leader_vote_request_wire, raftgpu_leader_term_wire,
#                    raftgpu_follower_response_wire
WIRE_STALE = 11  # raftgpu_follower_term_wire, raftgpu_leader_term_wire, raftgpu_follower_response_wire
WIRE_WAVES_MAX = 64  # raftgpu_arena_set_wire_waves
# raftgpu_vote_request_wire: the caller's table (raftgpu_voter), its flags, and the low nibble of an applied frame
VOTER_SELECT, VOTER_LEADER, VOTER_LEASE = 0x1, 0x2, 0x4
VREQ_GRANTED, VREQ_VOTED, VREQ_BUMPED = 0x1, 0x2, 0x4
# raftgpu_follower_term_wire: the voter table's extra flag and the claimant's low nibble
VOTER_STALE_REPLY = 0x8
FTERM_BUMPED = 0x4
# raftgpu_follower_response_wire (and raftgpu_follower_term_wire's step-down): the candidate flags, the step-down's nibble
VOTER_CANDIDATE, VOTER_PRE_CANDIDATE = 0x10, 0x20
FTERM_STEPPED = 0x8
VOTER_DTYPE = np.dtype([("id", "<u8"), ("vote", "<u8"), ("last_term", "<u8"), ("commit_term", "<u8"),
                        ("persisted", "<u8"), ("priority", "<u8"), ("flags", "<u4"), ("reserved", "<u4"),
                        ("reserved2", "<u8")])
assert VOTER_DTYPE.itemsize == 64
# raftgpu_follower_append: the caller's log table (raftgpu_follower_log), its flag, and the low nibble's extra bits
FOLLOWER_SELECT = 0x1
FAPP_REJECT, FAPP_STALE = 0x2, 0x4
FOLLOWER_LOG_DTYPE = np.dtype([("id", "<u8"), ("run_start", "<u8"), ("run_term", "<u8"), ("flags", "<u4"),
                               ("reserved", "<u4")])
assert FOLLOWER_LOG_DTYPE.itemsize == 32
# raftgpu_leader_runs_set: one group's leader runs (raftgpu_leader_runs)
LEADER_RUNS_DTYPE = np.dtype([("group", "<u4"), ("reserved", "<u4"), ("term", "<u8"), ("term_start", "<u8"),
                              ("run_start", "<u8", (2,)), ("run_term", "<u8", (2,))])
assert LEADER_RUNS_DTYPE.itemsize == 56
# raftgpu_follower_runs_set / _get: one group's follower runs (raftgpu_follower_runs)
FOLLOWER_RUNS_DTYPE = np.dtype([("group", "<u4"), ("reserved", "<u4"), ("anchor_start", "<u8"), ("anchor_term", "<u8"),
                                ("run_start", "<u8", (2,)), ("run_term", "<u8", (2,))])
assert FOLLOWER_RUNS_DTYPE.itemsize == 56
# raftgpu_follower_append_entries: an applied frame's extra bit and its record (raftgpu_follower_appended)
FAPP_APPENDED = 0x8
FOLLOWER_APPENDED_DTYPE = np.dtype([("first_index", "<u8"), ("last_index", "<u8"), ("run_start", "<u8"),
                                    ("run_term", "<u8"), ("span_off", "<u4"), ("span_len", "<u4")])
assert FOLLOWER_APPENDED_DTYPE.itemsize == 40
# raftgpu_vote_wire's outcome: the group (a pair's low half) and its tally word (VoteResult | granted << 8 | rejected << 16)
VOTE_OUTCOME_DTYPE = np.dtype([("group", "<u4"), ("result", "<u4")])
assert VOTE_OUTCOME_DTYPE.itemsize == 8

APPEND_RESP_DTYPE = np.dtype(
    [("group", "<u4"), ("peer_slot", "u1"), ("flags", "u1"), ("reserved", "<u2"),
     ("index", "<u8"), ("commit", "<u8")]
)
assert APPEND_RESP_DTYPE.itemsize == 24
SEND_ENTRY_DTYPE = np.dtype([("group", "<u4"), ("peer_slot", "u1"), ("flags", "u1"), ("reserved", "<u2"),
                             ("next_idx", "<u8")])
assert SEND_ENTRY_DTYPE.itemsize == 16
SEND_SNAPSHOT = 0x1
# raftgpu_control (the batched control plane): one command per single-group control call, and its result
(CTL_SET_CONF, CTL_RESET, CTL_BECOME_LEADER, CTL_SET_LOG_BOUNDS, CTL_SET_TERM, CTL_COMMIT_TO, CTL_MAYBE_COMMIT_TO,
 CTL_SET_GROUP_COMMIT, CTL_ASSIGN_COMMIT_GROUP, CTL_RESET_VOTES, CTL_RECORD_VOTE, CTL_VOTE_RESULT, CTL_HAS_QUORUM,
 CTL_QUORUM_RECENTLY_ACTIVE, CTL_PROGRESS_OP) = range(15)
CTL_NO_SELF = 0xFF
CTL_CMD_DTYPE = np.dtype([("group", "<u4"), ("op", "u1"), ("peer_slot", "u1"), ("arg", "<u2"), ("a", "<u8", (4,))])
assert CTL_CMD_DTYPE.itemsize == 40
CTL_RESULT_DTYPE = np.dtype([("status", "<i4"), ("value", "<i4")])
assert CTL_RESULT_DTYPE.itemsize == 8
# ReadIndex (ReadOnlyOption::Safe): requests, released reads, result bytes, the heartbeat record flag
READ_REQ_DTYPE = np.dtype([("group", "<u4"), ("reserved", "<u4"), ("ctx", "<u8")])
assert READ_REQ_DTYPE.itemsize == 16
READ_STATE_DTYPE = np.dtype([("group", "<u4"), ("reserved", "<u4"), ("ctx", "<u8"), ("index", "<u8")])
assert READ_STATE_DTYPE.itemsize == 24
REC_READ_CTX = 0x08
READ_QUEUED, READ_READY, READ_DUP, READ_DROPPED, READ_FULL, READ_NO_GROUP, READ_NO_CTX = range(1, 8)
READ_MAX_PENDING = 64

# host column name -> (column id, numpy dtype, per-peer?)
COLUMNS = {
    "matched": (COL_MATCHED, np.uint64, True),
    "next_idx": (COL_NEXT_IDX, np.uint64, True),
    "peer_committed": (COL_PEER_COMMITTED, np.uint64, True),
    "pending_snapshot": (COL_PENDING_SNAPSHOT, np.uint64, True),
    "pending_request_snapshot": (COL_PENDING_REQ_SNAPSHOT, np.uint64, True),
    "commit_group_id": (COL_COMMIT_GROUP_ID, np.uint64, True),
    "pflags": (COL_PFLAGS, np.uint8, True),
    "meta": (COL_META, np.uint32, False),
    "committed": (COL_COMMITTED, np.uint64, False),
    "term_start": (COL_TERM_START, np.uint64, False),
    "last_index": (COL_LAST_INDEX, np.uint64, False),
}
# (the term column, COL_TERM, is written separately: only the wire path reads it)


class RaftGpuError(RuntimeError):
    def __init__(self, status, what, detail=""):
        self.status = status
        super().__init__(f"{what}: {strerror(status)} ({status}){': ' + detail if detail else ''}")


class Progress(C.Structure):
    _fields_ = [("matched", C.c_uint64), ("next_idx", C.c_uint64),
                ("pending_snapshot", C.c_uint64), ("pending_request_snapshot", C.c_uint64),
                ("commit_group_id", C.c_uint64), ("committed_index", C.c_uint64),
                ("state", C.c_uint8), ("paused", C.c_uint8), ("recent_active", C.c_uint8),
                ("ins_full", C.c_uint8), ("present", C.c_uint8), ("reserved", C.c_uint8 * 3)]


class GroupState(C.Structure):
    _fields_ = [("meta", C.c_uint32), ("reserved", C.c_uint32), ("committed", C.c_uint64),
                ("term_start", C.c_uint64), ("last_index", C.c_uint64)]


class Info(C.Structure):
    _fields_ = [("abi_version", C.c_uint32), ("device", C.c_int32), ("cap", C.c_uint32),
                ("slots", C.c_uint32), ("n_alloc", C.c_uint32), ("hi", C.c_uint32),
                ("sm_count", C.c_uint32), ("reserved", C.c_uint32), ("l2_bytes", C.c_uint64),
                ("device_bytes", C.c_uint64), ("pinned_bytes", C.c_uint64)]


class Counters(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("recomputes", "advanced", "records", "updates", "rejects",
                                          "decrements", "no_progress", "votes_tallied")]

    def as_dict(self):
        return {n: int(getattr(self, n)) for n, _ in self._fields_}


class StepResult(C.Structure):
    _fields_ = [("n_records", C.c_uint64), ("n_waves", C.c_uint32), ("n_groups", C.c_uint32),
                ("n_advanced", C.c_uint64), ("h2d_bytes", C.c_uint64), ("d2h_bytes", C.c_uint64),
                ("n_duplicates", C.c_uint64)]


class WireBatch(C.Structure):
    _fields_ = [("bytes", C.c_void_p), ("n_bytes", C.c_uint64), ("offsets", C.c_void_p), ("n", C.c_uint64),
                ("records", C.c_void_p), ("n_records", C.c_uint64)]


class SynthColumns(C.Structure):
    _fields_ = [("cap", C.c_uint32), ("n_groups", C.c_uint32)] + \
        [(n, C.c_void_p) for n in ("matched", "next_idx", "peer_committed", "pflags", "meta",
                                   "committed", "term_start", "last_index", "term", "sim_acked",
                                   "sim_last", "sim_flags")]


def compact_bound(n_records: int) -> int:
    return int(lib().raftgpu_compact_bound(n_records))


def pack_compact(recs: np.ndarray, out: np.ndarray, want_units: bool = False):
    """records -> compact stream blob in `out` (u8, 16-byte aligned).  Returns (bytes, unit_of_record|None)."""
    assert recs.dtype == APPEND_RESP_DTYPE and recs.flags.c_contiguous and out.dtype == np.uint8
    nb = C.c_uint64()
    units = np.empty(len(recs), dtype=np.uint32) if want_units else None
    rc = lib().raftgpu_pack_compact(recs.ctypes.data, len(recs), out.ctypes.data, out.nbytes, C.byref(nb),
                                    units.ctypes.data if want_units else None)
    if rc != 0:
        raise RuntimeError(f"raftgpu_pack_compact failed: {rc}")
    return nb.value, units


COMPACT_HDR_DTYPE = np.dtype([("magic", "<u4"), ("n_units", "<u4"), ("n_blocks", "<u4"), ("n_side", "<u4"),
                              ("n_records", "<u8"), ("off_blocks", "<u8"), ("off_units", "<u8"),
                              ("off_side", "<u8"), ("total_bytes", "<u8"), ("flags", "<u4"), ("reserved", "<u4")])
COMPACT_TILEABLE, COMPACT_ONE_WAVE = 0x1, 0x2


def unpack_compact(blob: np.ndarray) -> np.ndarray:
    """Decode a compact stream back to public records (tests; mirrors load_compact in kernels.cuh)."""
    h = blob[:COMPACT_HDR_DTYPE.itemsize].view(COMPACT_HDR_DTYPE)[0]
    assert h["magic"] == 0x31434752
    nu, ns = int(h["n_units"]), int(h["n_side"])
    units = blob[int(h["off_units"]):int(h["off_units"]) + 4 * nu].view(np.uint32)
    g_base = blob[int(h["off_blocks"]):int(h["off_blocks"]) + 4 * int(h["n_blocks"])].view(np.uint32)
    side = blob[int(h["off_side"]):int(h["off_side"]) + 24 * ns].view(APPEND_RESP_DTYPE)
    out = []
    for i in range(nu):
        u = int(units[i])
        kind = u & 3
        if kind == 3:
            k = u >> 2
            if k < 0x1fffffff and k < ns:     # (payload units and padding carry no record of their own)
                out.append(tuple(side[k]))
                if (side[k]["flags"] & REC_REJECT) and k + 1 < ns and (side[k + 1]["flags"] & REC_EXT):
                    out.append(tuple(side[k + 1]))
            continue
        if kind != 0:
            continue
        back = (u >> 3) & 7
        hpos = i - back - 2
        ha, hb = int(units[hpos]), int(units[hpos + 1])
        assert ha & 3 == 1 and hb & 3 == 2
        g = int(g_base[hpos // 2048]) + ((hb >> 2) & 0xfff)
        base = (ha >> 2) | ((hb >> 14) << 30)
        index = base + ((u >> 10) & 0x3fff)
        cd = u >> 24
        local, reject = bool(u & 4), bool(u & (1 << 9))
        commit = (0 if cd == 255 else index + cd) if local else index - cd
        out.append((g, (u >> 6) & 7, REC_LOCAL if local else (REC_REJECT if reject else 0), 0, index, commit))
        if reject:
            pl = int(units[i + 1])
            assert pl & 3 == 3 and (pl >> 2) & (1 << 29)
            d = (pl >> 2) & ((1 << 29) - 1)
            if d >= 1 << 28:
                d -= 1 << 29
            out.append((g, (u >> 6) & 7, REC_EXT, 0, (index + d) & ((1 << 64) - 1), 0))
    return np.array(out, dtype=APPEND_RESP_DTYPE)


def declared_symbols() -> list[str]:
    """Every function include/raftgpu.h declares (parsed from the header text)."""
    with open(HEADER_PATH, encoding="utf-8") as f:
        text = f.read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(raftgpu_[a-z0-9_]+)\s*\(", text)))


_lib = None


def lib() -> C.CDLL:
    """Load libraftgpu.so; raises if it has not been built (no fallback)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} is missing: run __graft_entry__.build() / make -C raft-rs_b200")
        L = C.CDLL(LIB_PATH)
        vp, u32, i32, u64 = C.c_void_p, C.c_uint32, C.c_int32, C.c_uint64
        sig = {
            "raftgpu_strerror": ([i32], C.c_char_p),
            "raftgpu_abi_version": ([], u32),
            "raftgpu_arena_create": ([i32, u32, u32, u32, u32, C.POINTER(vp)], i32),
            "raftgpu_arena_destroy": ([vp], i32),
            "raftgpu_arena_info": ([vp, C.POINTER(Info)], i32),
            "raftgpu_last_error": ([vp], C.c_char_p),
            "raftgpu_group_alloc": ([vp, C.POINTER(u32)], i32),
            "raftgpu_group_alloc_range": ([vp, u32, C.POINTER(u32)], i32),
            "raftgpu_group_alloc_wide": ([vp, C.POINTER(u32)], i32),
            "raftgpu_group_free": ([vp, u32], i32),
            "raftgpu_group_set_conf": ([vp, u32, u32, u32, u32, i32, u64], i32),
            "raftgpu_group_reset": ([vp, u32, u64, u64, u64, u64], i32),
            "raftgpu_group_become_leader": ([vp, u32], i32),
            "raftgpu_group_set_log_bounds": ([vp, u32, u64, u64], i32),
            "raftgpu_group_commit_to": ([vp, u32, u64], i32),
            "raftgpu_group_get": ([vp, u32, C.POINTER(GroupState)], i32),
            "raftgpu_progress_get": ([vp, u32, u32, C.POINTER(Progress)], i32),
            "raftgpu_progress_set": ([vp, u32, u32, C.POINTER(Progress)], i32),
            "raftgpu_progress_op": ([vp, u32, u32, i32, u64, u64, u64, C.POINTER(i32)], i32),
            "raftgpu_has_quorum": ([vp, u32, u32, C.POINTER(i32)], i32),
            "raftgpu_quorum_recently_active": ([vp, u32, u32, C.POINTER(i32)], i32),
            "raftgpu_group_maybe_commit_to": ([vp, u32, u64, C.POINTER(i32)], i32),
            "raftgpu_set_group_commit": ([vp, u32, i32], i32),
            "raftgpu_assign_commit_group": ([vp, u32, u32, u64], i32),
            "raftgpu_column_write": ([vp, i32, u32, u32, u32, vp], i32),
            "raftgpu_column_read": ([vp, i32, u32, u32, u32, vp], i32),
            "raftgpu_maximal_committed_index": ([vp, u32, C.POINTER(u64), C.POINTER(i32)], i32),
            "raftgpu_maybe_commit": ([vp, u32, C.POINTER(i32), C.POINTER(u64)], i32),
            "raftgpu_recompute": ([vp, vp, u32, u32, vp, vp, vp, vp], i32),
            "raftgpu_apply_device": ([vp, vp, vp, u64, vp], i32),
            "raftgpu_apply_device_packed": ([vp, vp, vp, u64, vp], i32),
            "raftgpu_step_sorted_device": ([vp, vp, vp, u64, vp, vp, vp, vp], i32),
            "raftgpu_tile_index": ([vp, u64, u32, vp, u64], i32),
            "raftgpu_tile_groups": ([], u32),
            "raftgpu_enqueue_append_resp": ([vp, u32, vp, u64], i32),
            "raftgpu_enqueue_bulk": ([vp, vp, u64, u32], i32),
            "raftgpu_step_begin": ([vp, u32], i32),
            "raftgpu_step_begin_packed": ([vp, vp, u64, u32], i32),
            "raftgpu_pack_records": ([vp, u64, vp, u64, C.POINTER(u64)], i32),
            "raftgpu_compact_bound": ([u64], u64),
            "raftgpu_pack_compact": ([vp, u64, vp, u64, C.POINTER(u64), vp], i32),
            "raftgpu_step_begin_compact": ([vp, vp, u64, u32], i32),
            "raftgpu_step_begin_records": ([vp, vp, u64, u32], i32),
            "raftgpu_step_slot_results": ([vp, C.POINTER(vp), C.POINTER(u64)], i32),
            "raftgpu_compact_tile_index_device": ([vp, vp, vp, vp, vp, vp], i32),
            "raftgpu_step_compact_device": ([vp, vp, vp, vp, vp, vp, vp, vp, vp, u32], i32),
            "raftgpu_host_alloc": ([vp, u64, C.POINTER(vp)], i32),
            "raftgpu_host_free": ([vp, vp], i32),
            "raftgpu_step_wait": ([vp, C.POINTER(StepResult)], i32),
            "raftgpu_step": ([vp, u32, C.POINTER(StepResult)], i32),
            "raftgpu_step_results": ([vp, C.POINTER(vp), C.POINTER(vp)], i32),
            "raftgpu_step_record_results": ([vp, u32, vp, u64, C.POINTER(u64)], i32),
            "raftgpu_reset_votes": ([vp, u32], i32),
            "raftgpu_record_vote": ([vp, u32, u32, i32], i32),
            "raftgpu_tally_votes": ([vp, vp, u32, u32, vp], i32),
            "raftgpu_send_list_device": ([vp, vp, u32, u32, vp, vp, u64, vp], i32),
            "raftgpu_heartbeat_commits_device": ([vp, vp, u32, u32, vp], i32),
            "raftgpu_step_send_list": ([vp, vp, u64, C.POINTER(u64)], i32),
            "raftgpu_vote_result": ([vp, u32, C.POINTER(i32), C.POINTER(u32), C.POINTER(u32)], i32),
            "raftgpu_group_set_term": ([vp, u32, u64], i32),
            "raftgpu_control": ([vp, vp, u64, vp], i32),
            "raftgpu_arena_enable_inflights": ([vp, u32], i32),
            "raftgpu_arena_enable_leader_runs": ([vp], i32),
            "raftgpu_leader_runs_set": ([vp, vp, u64, vp], i32),
            "raftgpu_arena_enable_follower_runs": ([vp], i32),
            "raftgpu_follower_runs_set": ([vp, vp, u64, vp], i32),
            "raftgpu_follower_runs_get": ([vp, u32, u32, vp], i32),
            "raftgpu_arena_set_wire_waves": ([vp, u32], i32),
            "raftgpu_inflights_get": ([vp, u32, u32, C.POINTER(u32), C.POINTER(u32), vp, u32], i32),
            "raftgpu_heartbeat_resp_device": ([vp, vp, vp, u64, vp, vp], i32),
            "raftgpu_heartbeat_resp": ([vp, vp, u64, vp], i32),
            "raftgpu_arena_enable_read_index": ([vp, u32], i32),
            "raftgpu_read_index_request_device": ([vp, vp, vp, u64, vp, vp, u64, vp, vp], i32),
            "raftgpu_read_index_request": ([vp, vp, u64, vp, vp, u64, C.POINTER(u64)], i32),
            "raftgpu_read_index_ack_device": ([vp, vp, vp, u64, vp, u64, vp], i32),
            "raftgpu_read_index_ack": ([vp, vp, u64, vp, u64, C.POINTER(u64)], i32),
            "raftgpu_read_index_recheck": ([vp, vp, u64, vp, u64, C.POINTER(u64)], i32),
            "raftgpu_read_index_last_ctx_device": ([vp, vp, u32, u32, vp], i32),
            "raftgpu_read_index_get": ([vp, u32, C.POINTER(u32), vp, vp, vp, u32], i32),
            "raftgpu_read_index_read": ([vp, u32, u32, vp, vp, vp, vp], i32),
            "raftgpu_heartbeat_wire_device": ([vp, vp, vp, u64, vp, u64, vp, vp, u64, vp], i32),
            "raftgpu_heartbeat_wire": ([vp, vp, u64, vp, u64, vp, vp, u64, C.POINTER(u64)], i32),
            "raftgpu_heartbeat_frames_bound": ([u32], u64),
            "raftgpu_heartbeat_frames_device": ([vp, vp, u32, u32, vp, vp, vp, u64, vp, u64, vp], i32),
            "raftgpu_heartbeat_frames": ([vp, u32, u32, vp, vp, vp, u64, vp, u64, vp], i32),
            "raftgpu_append_frames_bound": ([u32], u64),
            "raftgpu_append_frames_device": ([vp, vp, u32, u32, vp, vp, vp, u64, vp, u64, vp, u64, vp], i32),
            "raftgpu_append_frames": ([vp, u32, u32, vp, vp, vp, u64, vp, u64, vp, u64, vp], i32),
            "raftgpu_follower_heartbeat_bound": ([u64], u64),
            "raftgpu_follower_heartbeat_device": ([vp, vp, vp, u64, vp, u64, vp, vp, vp, vp, vp, u64, vp, vp], i32),
            "raftgpu_follower_heartbeat": ([vp, vp, u64, vp, u64, vp, vp, vp, vp, vp, u64, vp, vp], i32),
            "raftgpu_vote_wire_device": ([vp, vp, vp, u64, vp, u64, vp, vp, vp, vp, u64, vp], i32),
            "raftgpu_vote_wire": ([vp, vp, u64, vp, u64, vp, vp, vp, vp, u64, C.POINTER(u64)], i32),
            "raftgpu_vote_request_wire_bound": ([u64], u64),
            "raftgpu_vote_request_wire_device": ([vp, vp, vp, u64, vp, u64, vp, vp, vp, vp, u64, vp, vp], i32),
            "raftgpu_vote_request_wire": ([vp, vp, u64, vp, u64, vp, vp, vp, vp, u64, vp, vp], i32),
            "raftgpu_follower_term_wire_bound": ([u64], u64),
            "raftgpu_follower_term_wire_device": ([vp, vp, vp, u64, vp, u64, vp, vp, vp, vp, u64, vp, vp], i32),
            "raftgpu_follower_term_wire": ([vp, vp, u64, vp, u64, vp, vp, vp, vp, u64, vp, vp], i32),
            "raftgpu_leader_term_wire_device": ([vp, vp, vp, u64, vp, u64, vp, vp, vp, vp, u64, vp, vp], i32),
            "raftgpu_leader_term_wire": ([vp, vp, u64, vp, u64, vp, vp, vp, vp, u64, vp, vp], i32),
            "raftgpu_leader_vote_request_wire_device": ([vp, vp, vp, u64, vp, u64, vp, vp, vp, vp, u64, vp, vp], i32),
            "raftgpu_leader_vote_request_wire": ([vp, vp, u64, vp, u64, vp, vp, vp, vp, u64, vp, vp], i32),
            "raftgpu_follower_response_wire_device": ([vp, vp, vp, u64, vp, u64, vp, vp, vp], i32),
            "raftgpu_follower_response_wire": ([vp, vp, u64, vp, u64, vp, vp, vp], i32),
            "raftgpu_follower_append_bound": ([u64], u64),
            "raftgpu_follower_append_device": ([vp, vp, vp, u64, vp, u64, vp, vp, vp, vp, u64, vp, vp], i32),
            "raftgpu_follower_append": ([vp, vp, u64, vp, u64, vp, vp, vp, vp, u64, vp, vp], i32),
            "raftgpu_follower_append_entries_device": ([vp, vp, vp, u64, vp, u64, vp, vp, vp, vp, vp, u64, vp, vp], i32),
            "raftgpu_follower_append_entries": ([vp, vp, u64, vp, u64, vp, vp, vp, vp, vp, u64, vp, vp], i32),
            "raftgpu_update_state_device": ([vp, vp, vp, u64, vp], i32),
            "raftgpu_update_state": ([vp, vp, u64, vp], i32),
            "raftgpu_wire_apply_device": ([vp, vp, vp, u64, vp, u64, vp], i32),
            "raftgpu_step_begin_wire": ([vp, C.POINTER(WireBatch), u32], i32),
            "raftgpu_step_wire_status": ([vp, C.POINTER(vp), C.POINTER(u64)], i32),
            "raftgpu_counters_read": ([vp, C.POINTER(Counters)], i32),
            "raftgpu_synchronize": ([vp], i32),
            "raftgpu_debug_read": ([vp, vp], i32),
            "raftgpu_device_alloc": ([vp, u64, C.POINTER(vp)], i32),
            "raftgpu_device_free": ([vp, vp], i32),
            "raftgpu_memcpy_h2d": ([vp, vp, vp, u64], i32),
            "raftgpu_memcpy_d2h": ([vp, vp, vp, u64], i32),
        }
        for name, (args, res) in sig.items():
            f = getattr(L, name)
            f.argtypes, f.restype = args, res
        L._signatures = sig
        _lib = L
    return _lib


_synth_lib = None


def synth_lib() -> C.CDLL:
    """libraftgpu_synth.so: the synthetic workload generator (include/raftgpu_synth.h), a
    separate library so the product .so carries no bench infrastructure."""
    global _synth_lib
    if _synth_lib is None:
        if not os.path.exists(SYNTH_LIB_PATH):
            raise RuntimeError(f"{SYNTH_LIB_PATH} is missing: run __graft_entry__.build() / make -C raft-rs_b200")
        L = C.CDLL(SYNTH_LIB_PATH)
        vp, u32, i32, u64 = C.c_void_p, C.c_uint32, C.c_int32, C.c_uint64
        L.raftgpu_synth_init.argtypes, L.raftgpu_synth_init.restype = [C.POINTER(SynthColumns), u64, u32, i32], i32
        L.raftgpu_synth_round.argtypes = [C.POINTER(SynthColumns), u64, u32, u32, vp, u64, C.POINTER(u64)]
        L.raftgpu_synth_round.restype = i32
        L.raftgpu_synth_wire_encode.argtypes = [vp, u64, vp, vp, u64, vp, C.POINTER(u64), C.POINTER(u64), vp, C.POINTER(u64)]
        L.raftgpu_synth_wire_encode.restype = i32
        L.raftgpu_synth_wire_encode_heartbeats.argtypes = [vp, u64, vp, vp, u64, vp, C.POINTER(u64), C.POINTER(u64)]
        L.raftgpu_synth_wire_encode_heartbeats.restype = i32
        L.raftgpu_synth_wire_encode_votes.argtypes = [vp, u64, vp, u64, vp, C.POINTER(u64)]
        L.raftgpu_synth_wire_encode_votes.restype = i32
        L.raftgpu_synth_wire_encode_vote_requests.argtypes = [vp, u64, vp, u64, vp, C.POINTER(u64)]
        L.raftgpu_synth_wire_encode_vote_requests.restype = i32
        _synth_lib = L
    return _synth_lib


def strerror(status: int) -> str:
    return lib().raftgpu_strerror(status).decode()


TILE_GROUPS = 256


# raftgpu_synth_vote: one vote response for raftgpu_synth_wire_encode_votes
SYNTH_VOTE_DTYPE = np.dtype([("hdr", "<u4"), ("msg_type", "<u4"), ("to", "<u8"), ("from", "<u8"), ("term", "<u8"),
                             ("commit", "<u8"), ("commit_term", "<u8"), ("reject", "<u4"), ("reserved", "<u4")])
assert SYNTH_VOTE_DTYPE.itemsize == 56


def synth_encode_votes(votes: np.ndarray):
    """raftgpu_synth_wire_encode_votes: SYNTH_VOTE_DTYPE entries -> (blob padded to 16 bytes, offsets u32[n + 1])."""
    votes = np.ascontiguousarray(votes, dtype=SYNTH_VOTE_DTYPE)
    n = len(votes)
    blob, off, nb = np.zeros(64 * n + 16, np.uint8), np.zeros(n + 1, np.uint32), C.c_uint64()
    rc = synth_lib().raftgpu_synth_wire_encode_votes(votes.ctypes.data, n, blob.ctypes.data, len(blob), off.ctypes.data,
                                                     C.byref(nb))
    if rc != OK:
        raise RaftGpuError(rc, "synth_wire_encode_votes")
    return blob[: (nb.value + 15) // 16 * 16 + 16].copy(), off


# raftgpu_synth_vote_request: one vote request for raftgpu_synth_wire_encode_vote_requests
SYNTH_VOTE_REQUEST_DTYPE = np.dtype([("hdr", "<u4"), ("msg_type", "<u4"), ("to", "<u8"), ("from", "<u8"), ("term", "<u8"),
                                     ("log_term", "<u8"), ("index", "<u8"), ("commit", "<u8"), ("commit_term", "<u8"),
                                     ("priority", "<u8"), ("context", "u1", (24,)), ("context_len", "<u4"),
                                     ("reserved", "<u4")])
assert SYNTH_VOTE_REQUEST_DTYPE.itemsize == 104


def synth_encode_vote_requests(reqs: np.ndarray):
    """raftgpu_synth_wire_encode_vote_requests: SYNTH_VOTE_REQUEST_DTYPE entries -> (blob padded to 16 bytes, offsets
    u32[n + 1])."""
    reqs = np.ascontiguousarray(reqs, dtype=SYNTH_VOTE_REQUEST_DTYPE)
    n = len(reqs)
    blob, off, nb = np.zeros(128 * n + 16, np.uint8), np.zeros(n + 1, np.uint32), C.c_uint64()
    rc = synth_lib().raftgpu_synth_wire_encode_vote_requests(reqs.ctypes.data, n, blob.ctypes.data, len(blob),
                                                             off.ctypes.data, C.byref(nb))
    if rc != OK:
        raise RaftGpuError(rc, "synth_wire_encode_vote_requests")
    return blob[: (nb.value + 15) // 16 * 16 + 16].copy(), off


def vote_request_wire_bound(n: int) -> int:
    """raftgpu_vote_request_wire_bound: response bytes enough for any n vote-request frames."""
    return int(lib().raftgpu_vote_request_wire_bound(n))


def follower_term_wire_bound(n: int) -> int:
    """raftgpu_follower_term_wire_bound: response bytes enough for any n MsgAppend / MsgHeartbeat frames."""
    return int(lib().raftgpu_follower_term_wire_bound(n))


def follower_append_bound(n: int) -> int:
    """raftgpu_follower_append_bound: response bytes enough for any n MsgAppend frames."""
    return int(lib().raftgpu_follower_append_bound(n))


def follower_heartbeat_bound(n: int) -> int:
    """raftgpu_follower_heartbeat_bound: response bytes enough for any n heartbeat frames."""
    return int(lib().raftgpu_follower_heartbeat_bound(n))


def heartbeat_frames_bound(n: int) -> int:
    """raftgpu_heartbeat_frames_bound: bytes enough for the heartbeat frames of any n group slots."""
    return int(lib().raftgpu_heartbeat_frames_bound(n))


def append_frames_bound(n: int) -> int:
    """raftgpu_append_frames_bound: bytes enough for the MsgAppend frames of any n group slots."""
    return int(lib().raftgpu_append_frames_bound(n))


def tile_groups() -> int:
    return int(lib().raftgpu_tile_groups())


def tile_index(packed: np.ndarray, n_packed: int, n_groups: int) -> np.ndarray:
    """raftgpu_tile_index: first packed record of every 256-group tile (+ the end)."""
    tg = int(lib().raftgpu_tile_groups())
    n_tiles = (n_groups + tg - 1) // tg
    out = np.zeros(n_tiles + 1, dtype=np.uint32)
    rc = lib().raftgpu_tile_index(packed.ctypes.data, n_packed, n_groups, out.ctypes.data, len(out))
    if rc != OK:
        raise RaftGpuError(rc, "raftgpu_tile_index")
    return out


# --------------------------------------------------------------------------- host columns

def new_columns(cap: int, n_groups: int | None = None):
    """Zeroed host-side SoA columns in the arena's layout ([SLOTS][cap] / [cap])."""
    c = types.SimpleNamespace(cap=int(cap), n_groups=int(cap if n_groups is None else n_groups))
    for name, (_, dt, per_peer) in COLUMNS.items():
        setattr(c, name, np.zeros((SLOTS, cap) if per_peer else cap, dtype=dt))
    c.term = np.zeros(cap, dtype=np.uint64)  # only the oracle's literal-log check reads it
    return c


def copy_columns(c):
    d = types.SimpleNamespace(cap=c.cap, n_groups=c.n_groups)
    for name in list(COLUMNS) + ["term"]:
        setattr(d, name, getattr(c, name).copy())
    return d


def make_meta(incoming, outgoing=0, learners=0, self_slot=0, group_commit=False) -> int:
    m = (incoming & 0xFF) | ((outgoing & 0xFF) << 8) | ((learners & 0xFF) << 16)
    if self_slot is not None:
        m |= ((self_slot & 7) << 24) | META_HAS_SELF
    if group_commit:
        m |= META_GROUP_COMMIT
    return m


# --------------------------------------------------------------------------- synthetic workload

class Synth:
    """Deterministic AppendResponse workload (SURVEY 8(d)); see csrc/synth.cpp."""

    def __init__(self, n_groups: int, seed: int, k_peers: int = 5, joint: bool = False,
                 cap: int | None = None):
        self.n_groups, self.seed, self.joint = n_groups, seed, joint
        self.k_union = 7 if joint else k_peers
        cap = n_groups if cap is None else cap
        self.cols = new_columns(cap, n_groups)
        self.sim_acked = np.zeros((SLOTS, cap), dtype=np.uint64)
        self.sim_last = np.zeros(cap, dtype=np.uint64)
        self.sim_flags = np.zeros((SLOTS, cap), dtype=np.uint8)
        self._sc = SynthColumns()
        self._sc.cap, self._sc.n_groups = cap, n_groups
        c = self.cols
        for name, arr in [("matched", c.matched), ("next_idx", c.next_idx),
                          ("peer_committed", c.peer_committed), ("pflags", c.pflags),
                          ("meta", c.meta), ("committed", c.committed),
                          ("term_start", c.term_start), ("last_index", c.last_index),
                          ("term", c.term), ("sim_acked", self.sim_acked),
                          ("sim_last", self.sim_last), ("sim_flags", self.sim_flags)]:
            setattr(self._sc, name, arr.ctypes.data)
        rc = synth_lib().raftgpu_synth_init(C.byref(self._sc), seed, k_peers, int(joint))
        if rc != OK:
            raise RaftGpuError(rc, "raftgpu_synth_init")
        # what an arena / the oracle is loaded with (rounds only advance the sim_* state)
        self.initial = self.cols
        self.round_no = 0
        self._buf = None

    def max_records_per_round(self) -> int:
        return self.n_groups * (2 * (self.k_union - 1) + 1)

    def next_round(self, out: np.ndarray | None = None) -> np.ndarray:
        """Returns a VIEW into a buffer that the next call overwrites (copy it to keep it):
        fresh host pages are expensive on the GPU boxes' VMs, so one buffer is reused."""
        if out is None:
            if self._buf is None:
                cap = min(self.max_records_per_round(), (7 if self.joint else 5) * self.n_groups + 64)
                self._buf = np.empty(cap, dtype=APPEND_RESP_DTYPE)
            out = self._buf
        n = C.c_uint64()
        rc = synth_lib().raftgpu_synth_round(C.byref(self._sc), self.seed, self.round_no, self.k_union,
                                       out.ctypes.data, len(out), C.byref(n))
        if rc != OK:
            raise RaftGpuError(rc, "raftgpu_synth_round")
        self.round_no += 1
        return out[: n.value]


# --------------------------------------------------------------------------- the arena

class Arena:
    """Thin owner of a raftgpu_arena*; every method is one C-ABI call."""

    def __init__(self, max_groups: int, device: int = 0, n_rings: int = 0, ring_records: int = 0):
        self._L = lib()
        self._h = C.c_void_p()
        rc = self._L.raftgpu_arena_create(device, max_groups, SLOTS, n_rings, ring_records,
                                          C.byref(self._h))
        if rc != OK:
            detail = self._L.raftgpu_last_error(None)
            self._h = C.c_void_p()
            raise RaftGpuError(rc, "raftgpu_arena_create", detail.decode() if detail else "")
        self.info = self.get_info()
        self.cap = self.info.cap

    # -- plumbing
    def _ck(self, rc, what):
        if rc != OK:
            detail = self._L.raftgpu_last_error(self._h)
            raise RaftGpuError(rc, what, detail.decode() if detail else "")

    def close(self):
        if self._h:
            self._L.raftgpu_arena_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def get_info(self) -> Info:
        i = Info()
        self._ck(self._L.raftgpu_arena_info(self._h, C.byref(i)), "arena_info")
        return i

    def debug_read(self) -> np.ndarray:
        out = np.zeros(8, dtype=np.uint64)
        self._ck(self._L.raftgpu_debug_read(self._h, out.ctypes.data), "debug_read")
        return out

    def synchronize(self):
        self._ck(self._L.raftgpu_synchronize(self._h), "synchronize")

    def counters(self) -> dict:
        c = Counters()
        self._ck(self._L.raftgpu_counters_read(self._h, C.byref(c)), "counters_read")
        return c.as_dict()

    def device_alloc(self, nbytes: int) -> int:
        p = C.c_void_p()
        self._ck(self._L.raftgpu_device_alloc(self._h, nbytes, C.byref(p)), "device_alloc")
        return p.value

    def device_free(self, ptr: int):
        self._ck(self._L.raftgpu_device_free(self._h, ptr), "device_free")

    def h2d(self, dptr: int, arr: np.ndarray):
        arr = np.ascontiguousarray(arr)
        self._ck(self._L.raftgpu_memcpy_h2d(self._h, dptr, arr.ctypes.data, arr.nbytes), "memcpy_h2d")

    def d2h(self, arr: np.ndarray, dptr: int):
        assert arr.flags.c_contiguous
        self._ck(self._L.raftgpu_memcpy_d2h(self._h, arr.ctypes.data, dptr, arr.nbytes), "memcpy_d2h")

    # -- group lifecycle
    def group_alloc(self) -> int:
        g = C.c_uint32()
        self._ck(self._L.raftgpu_group_alloc(self._h, C.byref(g)), "group_alloc")
        return g.value

    def group_alloc_wide(self) -> int:
        """A group of up to 16 peers = group slots g (even) and g + 1 (include/raftgpu.h)."""
        g = C.c_uint32()
        self._ck(self._L.raftgpu_group_alloc_wide(self._h, C.byref(g)), "group_alloc_wide")
        return g.value

    def group_alloc_range(self, n: int) -> int:
        g = C.c_uint32()
        self._ck(self._L.raftgpu_group_alloc_range(self._h, n, C.byref(g)), "group_alloc_range")
        return g.value

    def group_free(self, g):
        self._ck(self._L.raftgpu_group_free(self._h, g), "group_free")

    def group_set_conf(self, g, incoming, outgoing=0, learners=0, self_slot=0, next_idx=1):
        self._ck(self._L.raftgpu_group_set_conf(self._h, g, incoming, outgoing, learners,
                                                -1 if self_slot is None else self_slot, next_idx),
                 "group_set_conf")

    def group_reset(self, g, term_start, last_index, committed, persisted):
        self._ck(self._L.raftgpu_group_reset(self._h, g, term_start, last_index, committed, persisted),
                 "group_reset")

    def group_become_leader(self, g):
        self._ck(self._L.raftgpu_group_become_leader(self._h, g), "group_become_leader")

    def group_set_log_bounds(self, g, term_start, last_index):
        self._ck(self._L.raftgpu_group_set_log_bounds(self._h, g, term_start, last_index),
                 "group_set_log_bounds")

    def group_commit_to(self, g, to_commit) -> int:
        return self._L.raftgpu_group_commit_to(self._h, g, to_commit)

    def group_get(self, g) -> GroupState:
        s = GroupState()
        self._ck(self._L.raftgpu_group_get(self._h, g, C.byref(s)), "group_get")
        return s

    def progress_get(self, g, slot) -> Progress:
        p = Progress()
        self._ck(self._L.raftgpu_progress_get(self._h, g, slot, C.byref(p)), "progress_get")
        return p

    def progress_set(self, g, slot, p: Progress):
        self._ck(self._L.raftgpu_progress_set(self._h, g, slot, C.byref(p)), "progress_set")

    def progress_op(self, g, slot, op: int, a0=0, a1=0, a2=0) -> int:
        r = C.c_int32()
        self._ck(self._L.raftgpu_progress_op(self._h, g, slot, op, a0, a1, a2, C.byref(r)), "progress_op")
        return r.value

    def has_quorum(self, g, slot_mask: int) -> bool:
        r = C.c_int32()
        self._ck(self._L.raftgpu_has_quorum(self._h, g, slot_mask, C.byref(r)), "has_quorum")
        return bool(r.value)

    def quorum_recently_active(self, g, perspective_of_slot: int) -> bool:
        r = C.c_int32()
        self._ck(self._L.raftgpu_quorum_recently_active(self._h, g, perspective_of_slot, C.byref(r)),
                 "quorum_recently_active")
        return bool(r.value)

    def group_maybe_commit_to(self, g, max_index: int) -> bool:
        r = C.c_int32()
        self._ck(self._L.raftgpu_group_maybe_commit_to(self._h, g, max_index, C.byref(r)),
                 "group_maybe_commit_to")
        return bool(r.value)

    def set_group_commit(self, g, enable: bool):
        self._ck(self._L.raftgpu_set_group_commit(self._h, g, int(enable)), "set_group_commit")

    def assign_commit_group(self, g, slot, gid):
        self._ck(self._L.raftgpu_assign_commit_group(self._h, g, slot, gid), "assign_commit_group")

    def control(self, cmds: np.ndarray) -> np.ndarray:
        """raftgpu_control: every command of the list as its single-group call, in list order.  Returns the
        CTL_RESULT_DTYPE results (a refused command carries its status there; only the call's own failure raises)."""
        assert cmds.dtype == CTL_CMD_DTYPE and cmds.flags.c_contiguous
        res = np.zeros(len(cmds), dtype=CTL_RESULT_DTYPE)
        self._ck(self._L.raftgpu_control(self._h, cmds.ctypes.data, len(cmds), res.ctypes.data), "control")
        return res

    # -- bulk columns
    def column_write(self, col: int, slot: int, first: int, arr: np.ndarray):
        arr = np.ascontiguousarray(arr)
        self._ck(self._L.raftgpu_column_write(self._h, col, slot, first, arr.shape[0], arr.ctypes.data),
                 "column_write")

    def column_read(self, col: int, slot: int, first: int, n: int, dtype) -> np.ndarray:
        out = np.zeros(n, dtype=dtype)
        self._ck(self._L.raftgpu_column_read(self._h, col, slot, first, n, out.ctypes.data), "column_read")
        return out

    def load_columns(self, c, first: int = 0):
        """Upload host columns (groups [0, c.n_groups)) to arena groups [first, ...)."""
        n = c.n_groups
        for name, (col, dt, per_peer) in COLUMNS.items():
            arr = getattr(c, name)
            if per_peer:
                for s in range(SLOTS):
                    self.column_write(col, s, first, arr[s, :n])
            else:
                self.column_write(col, 0, first, arr[:n])

    def read_columns(self, n: int, first: int = 0):
        c = new_columns(n, n)
        for name, (col, dt, per_peer) in COLUMNS.items():
            arr = getattr(c, name)
            if per_peer:
                for s in range(SLOTS):
                    arr[s, :] = self.column_read(col, s, first, n, dt)
            else:
                arr[:] = self.column_read(col, 0, first, n, dt)
        return c

    # -- hot path
    def maximal_committed_index(self, g):
        idx, gc = C.c_uint64(), C.c_int32()
        self._ck(self._L.raftgpu_maximal_committed_index(self._h, g, C.byref(idx), C.byref(gc)),
                 "maximal_committed_index")
        return idx.value, bool(gc.value)

    def maybe_commit(self, g):
        adv, com = C.c_int32(), C.c_uint64()
        self._ck(self._L.raftgpu_maybe_commit(self._h, g, C.byref(adv), C.byref(com)), "maybe_commit")
        return bool(adv.value), com.value

    def recompute(self, first, n, stream=None, d_adv=None, d_commit=None, d_mci=None, d_gc=None):
        self._ck(self._L.raftgpu_recompute(self._h, stream, first, n, d_adv, d_commit, d_mci, d_gc),
                 "recompute")

    def apply_device(self, d_recs, n, stream=None, d_results=None):
        self._ck(self._L.raftgpu_apply_device(self._h, stream, d_recs, n, d_results), "apply_device")

    def apply_device_packed(self, d_packed, n_packed, stream=None, d_results=None):
        self._ck(self._L.raftgpu_apply_device_packed(self._h, stream, d_packed, n_packed, d_results),
                 "apply_device_packed")

    def step_sorted_device(self, d_packed, n_packed, d_tile_off, stream=None, d_results=None, d_adv=None,
                           d_commit=None):
        self._ck(self._L.raftgpu_step_sorted_device(self._h, stream, d_packed, n_packed, d_tile_off, d_results,
                                                    d_adv, d_commit), "step_sorted_device")

    def enqueue(self, recs: np.ndarray, ring: int = 0):
        assert recs.dtype == APPEND_RESP_DTYPE and recs.flags.c_contiguous
        self._ck(self._L.raftgpu_enqueue_append_resp(self._h, ring, recs.ctypes.data, len(recs)),
                 "enqueue_append_resp")

    def enqueue_bulk(self, recs: np.ndarray, sorted_by_group: bool = False):
        assert recs.dtype == APPEND_RESP_DTYPE and recs.flags.c_contiguous
        self._ck(self._L.raftgpu_enqueue_bulk(self._h, recs.ctypes.data, len(recs),
                                              BULK_SORTED if sorted_by_group else 0), "enqueue_bulk")

    def host_alloc_packed(self, n_records: int) -> np.ndarray:
        """NUMA-local pinned buffer of packed 16-byte records (u64 pairs), owned by the arena."""
        p = C.c_void_p()
        self._ck(self._L.raftgpu_host_alloc(self._h, 16 * n_records, C.byref(p)), "host_alloc")
        return np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint64)), shape=(n_records, 2))

    def pack_records(self, recs: np.ndarray, out: np.ndarray) -> int:
        assert recs.dtype == APPEND_RESP_DTYPE and recs.flags.c_contiguous and out.dtype == np.uint64
        n = C.c_uint64()
        self._ck(self._L.raftgpu_pack_records(recs.ctypes.data, len(recs), out.ctypes.data, out.shape[0],
                                              C.byref(n)), "pack_records")
        return n.value

    def step_begin_packed(self, packed: np.ndarray, n_packed: int, flags=0):
        self._ck(self._L.raftgpu_step_begin_packed(self._h, packed.ctypes.data, n_packed, flags),
                 "step_begin_packed")

    def host_alloc_bytes(self, n_bytes: int) -> np.ndarray:
        """NUMA-local pinned byte buffer owned by the arena (16-byte aligned)."""
        p = C.c_void_p()
        self._ck(self._L.raftgpu_host_alloc(self._h, n_bytes, C.byref(p)), "host_alloc")
        return np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(n_bytes,))

    def compact_tile_index_device(self, d_blob, hdr_blob: np.ndarray, d_tile_off, d_bad, stream=None):
        """hdr_blob: host bytes that start with the blob's raftgpu_compact_hdr."""
        self._ck(self._L.raftgpu_compact_tile_index_device(self._h, stream, d_blob, hdr_blob.ctypes.data, d_tile_off,
                                                           d_bad), "compact_tile_index_device")

    def step_compact_device(self, d_blob, hdr_blob: np.ndarray, d_tile_off, stream=None, d_results=None, d_adv=None,
                            d_commit=None, d_dup=None, ordered=False):
        self._ck(self._L.raftgpu_step_compact_device(self._h, stream, d_blob, hdr_blob.ctypes.data, d_tile_off,
                                                     d_results, d_adv, d_commit, d_dup, 1 if ordered else 0),
                 "step_compact_device")

    def host_free(self, buf: np.ndarray):
        self._ck(self._L.raftgpu_host_free(self._h, buf.ctypes.data), "host_free")

    def step_begin_records(self, recs: np.ndarray, flags=0):
        assert recs.dtype == APPEND_RESP_DTYPE and recs.flags.c_contiguous
        self._ck(self._L.raftgpu_step_begin_records(self._h, recs.ctypes.data, len(recs), flags), "step_begin_records")

    def step_begin_compact(self, blob: np.ndarray, n_bytes: int, flags=0):
        self._ck(self._L.raftgpu_step_begin_compact(self._h, blob.ctypes.data, n_bytes, flags),
                 "step_begin_compact")

    def step_begin(self, flags=0):
        self._ck(self._L.raftgpu_step_begin(self._h, flags), "step_begin")

    # -- Inflights on the device (SURVEY 8(f) rank 2)
    def enable_inflights(self, max_inflight: int):
        self._ck(self._L.raftgpu_arena_enable_inflights(self._h, max_inflight), "arena_enable_inflights")
        self.ins_cap = max_inflight

    def inflights_get(self, g, slot):
        """(start, count, ring u64[cap]) of one peer's window."""
        st, cnt = C.c_uint32(), C.c_uint32()
        buf = np.zeros(self.ins_cap, dtype=np.uint64)
        self._ck(self._L.raftgpu_inflights_get(self._h, g, slot, C.byref(st), C.byref(cnt), buf.ctypes.data, self.ins_cap),
                 "inflights_get")
        return st.value, cnt.value, buf

    # -- heartbeat responses / update_state (SURVEY 8(f) ranks 3 and 2)
    def heartbeat_resp(self, recs: np.ndarray) -> np.ndarray:
        """raftgpu_heartbeat_resp: REC_HEARTBEAT records -> result bytes (RES_OK | RES_SEND | RES_NO_PROGRESS)."""
        assert recs.dtype == APPEND_RESP_DTYPE and recs.flags.c_contiguous
        res = np.zeros(len(recs), dtype=np.uint8)
        self._ck(self._L.raftgpu_heartbeat_resp(self._h, recs.ctypes.data, len(recs), res.ctypes.data), "heartbeat_resp")
        return res

    # -- the leader's term runs (include/raftgpu.h)
    def enable_leader_runs(self):
        self._ck(self._L.raftgpu_arena_enable_leader_runs(self._h), "arena_enable_leader_runs")

    def set_wire_waves(self, waves: int) -> int:
        """raftgpu_arena_set_wire_waves: frames of a cell (the wire step) or group (the follower's append passes)
        decided per call.  Returns the status (RAFTGPU_ERR_INVALID for 0 or more than WIRE_WAVES_MAX)."""
        return int(self._L.raftgpu_arena_set_wire_waves(self._h, waves))

    def leader_runs_set(self, rows: np.ndarray) -> np.ndarray:
        """raftgpu_leader_runs_set: LEADER_RUNS_DTYPE rows -> the i32 status of each row (a refused row is not stored;
        only the call's own failure raises)."""
        rows = np.ascontiguousarray(rows, dtype=LEADER_RUNS_DTYPE)
        st = np.zeros(len(rows), dtype=np.int32)
        self._ck(self._L.raftgpu_leader_runs_set(self._h, rows.ctypes.data, len(rows), st.ctypes.data), "leader_runs_set")
        return st

    # -- the follower's earlier term runs (include/raftgpu.h)
    def enable_follower_runs(self):
        self._ck(self._L.raftgpu_arena_enable_follower_runs(self._h), "arena_enable_follower_runs")

    def follower_runs_set(self, rows: np.ndarray) -> np.ndarray:
        """raftgpu_follower_runs_set: FOLLOWER_RUNS_DTYPE rows -> the i32 status of each row (a refused row is not
        stored; only the call's own failure raises)."""
        rows = np.ascontiguousarray(rows, dtype=FOLLOWER_RUNS_DTYPE)
        st = np.zeros(len(rows), dtype=np.int32)
        self._ck(self._L.raftgpu_follower_runs_set(self._h, rows.ctypes.data, len(rows), st.ctypes.data),
                 "follower_runs_set")
        return st

    def follower_runs_get(self, first: int, n: int) -> np.ndarray:
        """raftgpu_follower_runs_get: the device's rows of groups [first, first + n) as FOLLOWER_RUNS_DTYPE."""
        rows = np.zeros(n, dtype=FOLLOWER_RUNS_DTYPE)
        self._ck(self._L.raftgpu_follower_runs_get(self._h, first, n, rows.ctypes.data), "follower_runs_get")
        return rows

    # -- ReadIndex, ReadOnlyOption::Safe (include/raftgpu.h)
    def enable_read_index(self, max_pending: int = 8):
        self._ck(self._L.raftgpu_arena_enable_read_index(self._h, max_pending), "arena_enable_read_index")
        self.read_max_pending = max_pending

    def read_index_request(self, reqs: np.ndarray):
        """raftgpu_read_index_request: READ_REQ_DTYPE requests in group order -> (result bytes, released reads)."""
        assert reqs.dtype == READ_REQ_DTYPE and reqs.flags.c_contiguous
        res = np.zeros(len(reqs), dtype=np.uint8)
        out = np.zeros(max(1, len(reqs)), dtype=READ_STATE_DTYPE)
        n = C.c_uint64()
        self._ck(self._L.raftgpu_read_index_request(self._h, reqs.ctypes.data, len(reqs), res.ctypes.data, out.ctypes.data,
                                                    len(reqs), C.byref(n)), "read_index_request")
        return res, out[: n.value]

    def read_index_ack(self, recs: np.ndarray) -> np.ndarray:
        """raftgpu_read_index_ack: HEARTBEAT | READ_CTX records (index = ctx id) -> released reads."""
        assert recs.dtype == APPEND_RESP_DTYPE and recs.flags.c_contiguous
        cap = min(len(recs), self.get_info().n_alloc) * self.read_max_pending
        out = np.zeros(max(1, cap), dtype=READ_STATE_DTYPE)
        n = C.c_uint64()
        self._ck(self._L.raftgpu_read_index_ack(self._h, recs.ctypes.data, len(recs), out.ctypes.data, cap, C.byref(n)),
                 "read_index_ack")
        return out[: n.value]

    def read_index_recheck(self, groups) -> np.ndarray:
        """raftgpu_read_index_recheck: post_conf_change's read tail for the listed groups -> released reads."""
        g = np.ascontiguousarray(groups, dtype=np.uint32)
        cap = len(g) * self.read_max_pending
        out = np.zeros(max(1, cap), dtype=READ_STATE_DTYPE)
        n = C.c_uint64()
        self._ck(self._L.raftgpu_read_index_recheck(self._h, g.ctypes.data, len(g), out.ctypes.data, cap, C.byref(n)),
                 "read_index_recheck")
        return out[: n.value]

    def read_index_last_ctx_device(self, first, n, d_out, stream=None):
        self._ck(self._L.raftgpu_read_index_last_ctx_device(self._h, stream, first, n, d_out), "read_index_last_ctx_device")

    def read_index_get(self, g):
        """One group's pending reads in queue order: (ctx u64[], index u64[], acks u16[])."""
        P = self.read_max_pending
        cnt = C.c_uint32()
        ctx, idx, acks = np.zeros(P, np.uint64), np.zeros(P, np.uint64), np.zeros(P, np.uint16)
        self._ck(self._L.raftgpu_read_index_get(self._h, g, C.byref(cnt), ctx.ctypes.data, idx.ctypes.data, acks.ctypes.data, P),
                 "read_index_get")
        k = cnt.value
        return ctx[:k], idx[:k], acks[:k]

    def read_index_read(self, first, n):
        """Groups [first, first + n) at once: (counts u32[n], ctx / index u64[n][P], acks u16[n][P]), queue order."""
        P = self.read_max_pending
        cnt = np.zeros(n, np.uint32)
        ctx, idx, acks = np.zeros((n, P), np.uint64), np.zeros((n, P), np.uint64), np.zeros((n, P), np.uint16)
        self._ck(self._L.raftgpu_read_index_read(self._h, first, n, cnt.ctypes.data, ctx.ctypes.data, idx.ctypes.data,
                                                 acks.ctypes.data), "read_index_read")
        return cnt, ctx, idx, acks

    def heartbeat_wire(self, batch):
        """raftgpu_heartbeat_wire: the MsgHeartbeatResponse frames of a wire batch (.bytes, .n_bytes, .offsets, .n, e.g.
        wire.WireBuffers) -> (status bytes WIRE_* << 4 | RES_*, released reads; empty without read queues)."""
        status = np.zeros(batch.n, dtype=np.uint8)
        P = getattr(self, "read_max_pending", 0)
        cap = min(batch.n, self.get_info().n_alloc) * P
        out = np.zeros(max(1, cap), dtype=READ_STATE_DTYPE)
        n = C.c_uint64()
        self._ck(self._L.raftgpu_heartbeat_wire(self._h, batch.bytes.ctypes.data, batch.n_bytes, batch.offsets.ctypes.data,
                                                batch.n, status.ctypes.data, out.ctypes.data if cap else None, cap,
                                                C.byref(n)), "heartbeat_wire")
        return status, out[: n.value]

    def heartbeat_wire_device(self, d_bytes, n_bytes, d_offsets, n, d_status, d_released=None, capacity=0, d_count=None,
                              stream=None):
        self._ck(self._L.raftgpu_heartbeat_wire_device(self._h, stream, d_bytes, n_bytes, d_offsets, n, d_status, d_released,
                                                       capacity, d_count), "heartbeat_wire_device")

    def heartbeat_frames(self, first, n, ids, select=None, bytes_out=None, offsets_out=None, bytes_capacity=None,
                         frames_capacity=None):
        """raftgpu_heartbeat_frames: bcast_heartbeat for groups [first, first + n) as MsgHeartbeat frames.  ids: u64 [9][n]
        (peer ids by slot, row 8 = the group's own id); select: u32 bitmap words from group 0, or None for all.  The
        output goes to bytes_out / offsets_out (allocated at the bound when None) with the given capacities (default:
        the arrays' sizes) -> (status, blob, offsets, totals u64[3]): status OK with the frames as views of the output
        arrays, or ERR_FULL with empty views (the totals still say what is needed); any other status raises."""
        ids = np.ascontiguousarray(ids, dtype=np.uint64)
        assert ids.shape == (SLOTS + 1, n)
        sel = None if select is None else np.ascontiguousarray(select, dtype=np.uint32)
        if bytes_out is None:
            bytes_out = np.zeros(max(16, heartbeat_frames_bound(n)), dtype=np.uint8)
        if offsets_out is None:
            offsets_out = np.zeros(SLOTS * n + 1, dtype=np.uint32)
        assert bytes_out.dtype == np.uint8 and offsets_out.dtype == np.uint32 and len(offsets_out) >= 1
        bcap = len(bytes_out) if bytes_capacity is None else bytes_capacity
        fcap = len(offsets_out) - 1 if frames_capacity is None else frames_capacity
        assert bcap <= len(bytes_out) and fcap < len(offsets_out)
        totals = np.zeros(3, dtype=np.uint64)
        rc = self._L.raftgpu_heartbeat_frames(self._h, first, n, None if sel is None else sel.ctypes.data, ids.ctypes.data,
                                              bytes_out.ctypes.data, bcap, offsets_out.ctypes.data, fcap, totals.ctypes.data)
        if rc == ERR_FULL:
            return rc, bytes_out[:0], offsets_out[:0], totals
        self._ck(rc, "heartbeat_frames")
        return rc, bytes_out[: int(totals[1])], offsets_out[: int(totals[0]) + 1], totals

    def heartbeat_frames_device(self, first, n, d_select, d_ids, d_bytes, bytes_capacity, d_offsets, frames_capacity,
                                d_totals, stream=None):
        self._ck(self._L.raftgpu_heartbeat_frames_device(self._h, stream, first, n, d_select, d_ids, d_bytes, bytes_capacity,
                                                         d_offsets, frames_capacity, d_totals), "heartbeat_frames_device")

    def append_frames(self, first, n, ids, select=None, bytes_out=None, offsets_out=None, rest_out=None,
                      bytes_capacity=None, frames_capacity=None, rest_capacity=None):
        """raftgpu_append_frames: bcast_append for groups [first, first + n) as entry-less MsgAppend frames and a rest
        list of the sends that need the log.  ids: u64 [9][n] (peer ids by slot, row 8 = the group's own id); select:
        u32 bitmap words from group 0, or None for all.  The output goes to bytes_out / offsets_out / rest_out
        (allocated at the bound when None) with the given capacities (default: the arrays' sizes) -> (status, blob,
        offsets, rest, totals u64[4]): status OK with the outputs as views of the output arrays, or ERR_FULL with empty
        views (the totals still say what is needed); any other status raises."""
        ids = np.ascontiguousarray(ids, dtype=np.uint64)
        assert ids.shape == (SLOTS + 1, n)
        sel = None if select is None else np.ascontiguousarray(select, dtype=np.uint32)
        if bytes_out is None:
            bytes_out = np.zeros(max(16, append_frames_bound(n)), dtype=np.uint8)
        if offsets_out is None:
            offsets_out = np.zeros(SLOTS * n + 1, dtype=np.uint32)
        if rest_out is None:
            rest_out = np.zeros(max(1, SLOTS * n), dtype=SEND_ENTRY_DTYPE)
        assert bytes_out.dtype == np.uint8 and offsets_out.dtype == np.uint32 and len(offsets_out) >= 1
        assert rest_out.dtype == SEND_ENTRY_DTYPE
        bcap = len(bytes_out) if bytes_capacity is None else bytes_capacity
        fcap = len(offsets_out) - 1 if frames_capacity is None else frames_capacity
        rcap = len(rest_out) if rest_capacity is None else rest_capacity
        assert bcap <= len(bytes_out) and fcap < len(offsets_out) and rcap <= len(rest_out)
        totals = np.zeros(4, dtype=np.uint64)
        rc = self._L.raftgpu_append_frames(self._h, first, n, None if sel is None else sel.ctypes.data, ids.ctypes.data,
                                           bytes_out.ctypes.data, bcap, offsets_out.ctypes.data, fcap,
                                           rest_out.ctypes.data, rcap, totals.ctypes.data)
        if rc == ERR_FULL:
            return rc, bytes_out[:0], offsets_out[:0], rest_out[:0], totals
        self._ck(rc, "append_frames")
        return rc, bytes_out[: int(totals[1])], offsets_out[: int(totals[0]) + 1], rest_out[: int(totals[2])], totals

    def append_frames_device(self, first, n, d_select, d_ids, d_bytes, bytes_capacity, d_offsets, frames_capacity,
                             d_rest, rest_capacity, d_totals, stream=None):
        self._ck(self._L.raftgpu_append_frames_device(self._h, stream, first, n, d_select, d_ids, d_bytes, bytes_capacity,
                                                      d_offsets, frames_capacity, d_rest, rest_capacity, d_totals),
                 "append_frames_device")

    def _reply(self, name, frames, tables, out_shape, bound, extra=None):
        """The host form of a reply pass: raftgpu_<name>(handle, the batch, tables, status u8[n], out u64[n][*out_shape],
        extra[n] when given, response bytes and their capacity bound(n), response offsets, totals u64[2]) -> (status, out,
        extra when given, response blob, response offsets u32[responses + 1], totals)."""
        n = frames.n
        outs = [np.zeros(n, np.uint8), np.zeros((n,) + out_shape, np.uint64)] + ([] if extra is None else [np.zeros(n, extra)])
        resp = np.zeros(max(16, bound(n)), np.uint8)
        roff, totals = np.zeros(n + 1, np.uint32), np.zeros(2, np.uint64)
        self._ck(getattr(self._L, "raftgpu_" + name)(self._h, frames.bytes.ctypes.data, frames.n_bytes,
                                                     frames.offsets.ctypes.data, n, *[t.ctypes.data for t in tables],
                                                     *[o.ctypes.data for o in outs], resp.ctypes.data, len(resp),
                                                     roff.ctypes.data, totals.ctypes.data), name)
        return (*outs, resp[: int(totals[1])], roff[: int(totals[0]) + 1], totals)

    def follower_heartbeat(self, frames, self_ids, select):
        """raftgpu_follower_heartbeat: handle_heartbeat at this arena's followers for the MsgHeartbeat frames of a wire
        batch (.bytes, .n_bytes, .offsets, .n; headers name the follower's group slot).  self_ids: u64 per group slot
        (Raft::id, the responses' `from`), select: u32 bitmap words from group 0 of the groups that are Followers; both
        cover the arena's capacity -> (status u8[n], from u64[n], response blob, response offsets u32[responses + 1],
        totals u64[2])."""
        ids = np.ascontiguousarray(self_ids, dtype=np.uint64)
        sel = np.ascontiguousarray(select, dtype=np.uint32)
        assert len(ids) >= self.cap and len(sel) * 32 >= self.cap
        return self._reply("follower_heartbeat", frames, (sel, ids), (), follower_heartbeat_bound)

    def follower_heartbeat_device(self, d_bytes, n_bytes, d_offsets, n, d_select, d_self_ids, d_status, d_from, d_resp_bytes,
                                  resp_bytes_capacity, d_resp_offsets, d_totals, stream=None):
        self._ck(self._L.raftgpu_follower_heartbeat_device(self._h, stream, d_bytes, n_bytes, d_offsets, n, d_select,
                                                           d_self_ids, d_status, d_from, d_resp_bytes, resp_bytes_capacity,
                                                           d_resp_offsets, d_totals), "follower_heartbeat_device")

    def vote_wire(self, frames, select, pre=None):
        """raftgpu_vote_wire: poll's record_vote + tally_votes for the MsgRequestVoteResponse / MsgRequestPreVoteResponse
        frames of a wire batch (.bytes, .n_bytes, .offsets, .n).  select: u32 bitmap words from group 0 of the groups that
        are PreCandidates or Candidates, pre: those that are PreCandidates (None: none); both cover the groups below the
        highest allocated one -> (status u8[n], outcomes VOTE_OUTCOME_DTYPE[k] in ascending group order)."""
        sel = np.ascontiguousarray(select, dtype=np.uint32)
        pr = None if pre is None else np.ascontiguousarray(pre, dtype=np.uint32)
        words = (self.get_info().hi + 31) // 32
        assert len(sel) >= words and (pr is None or len(pr) >= words)
        n = frames.n
        status = np.zeros(n, np.uint8)
        cap = min(n, self.get_info().n_alloc)
        out = np.zeros(max(1, cap), VOTE_OUTCOME_DTYPE)
        k = C.c_uint64()
        self._ck(self._L.raftgpu_vote_wire(self._h, frames.bytes.ctypes.data, frames.n_bytes, frames.offsets.ctypes.data, n,
                                           sel.ctypes.data, None if pr is None else pr.ctypes.data, status.ctypes.data,
                                           out.ctypes.data, cap, C.byref(k)), "vote_wire")
        return status, out[: k.value].copy()

    def vote_wire_device(self, d_bytes, n_bytes, d_offsets, n, d_select, d_pre, d_status, d_out, capacity, d_count,
                         stream=None):
        self._ck(self._L.raftgpu_vote_wire_device(self._h, stream, d_bytes, n_bytes, d_offsets, n, d_select, d_pre, d_status,
                                                  d_out, capacity, d_count), "vote_wire_device")

    def vote_request_wire(self, frames, voters):
        """raftgpu_vote_request_wire: Raft::step's term rules and the vote arm for the MsgRequestVote /
        MsgRequestPreVote frames of a wire batch (.bytes, .n_bytes, .offsets, .n; headers name the voter's group slot).
        voters: VOTER_DTYPE rows covering the groups below the highest allocated one -> (status u8[n], out u64[n][2] =
        {m.from, term after} of the applied frames, response blob, response offsets u32[responses + 1], totals u64[2])."""
        vt = np.ascontiguousarray(voters, dtype=VOTER_DTYPE)
        assert len(vt) >= self.get_info().hi
        return self._reply("vote_request_wire", frames, (vt,), (2,), vote_request_wire_bound)

    def vote_request_wire_device(self, d_bytes, n_bytes, d_offsets, n, d_voters, d_status, d_out, d_resp_bytes,
                                 resp_bytes_capacity, d_resp_offsets, d_totals, stream=None):
        self._ck(self._L.raftgpu_vote_request_wire_device(self._h, stream, d_bytes, n_bytes, d_offsets, n, d_voters, d_status,
                                                          d_out, d_resp_bytes, resp_bytes_capacity, d_resp_offsets, d_totals),
                 "vote_request_wire_device")

    def follower_term_wire(self, frames, voters):
        """raftgpu_follower_term_wire: Raft::step's term rules for the MsgAppend / MsgHeartbeat frames of a wire batch
        (.bytes, .n_bytes, .offsets, .n; headers name the follower's group slot).  voters: VOTER_DTYPE rows covering the
        groups below the highest allocated one -> (status u8[n], out u64[n][2] = {m.from, T} of the claimants, response
        blob, response offsets u32[responses + 1], totals u64[2])."""
        vt = np.ascontiguousarray(voters, dtype=VOTER_DTYPE)
        assert len(vt) >= self.get_info().hi
        return self._reply("follower_term_wire", frames, (vt,), (2,), follower_term_wire_bound)

    def follower_term_wire_device(self, d_bytes, n_bytes, d_offsets, n, d_voters, d_status, d_out, d_resp_bytes,
                                  resp_bytes_capacity, d_resp_offsets, d_totals, stream=None):
        self._ck(self._L.raftgpu_follower_term_wire_device(self._h, stream, d_bytes, n_bytes, d_offsets, n, d_voters,
                                                           d_status, d_out, d_resp_bytes, resp_bytes_capacity,
                                                           d_resp_offsets, d_totals), "follower_term_wire_device")

    def leader_term_wire(self, frames, voters):
        """raftgpu_leader_term_wire: Raft::step's term rules and the leader's drop arms for the MsgAppend,
        MsgAppendResponse, MsgRequestVoteResponse, MsgHeartbeat, MsgHeartbeatResponse and MsgRequestPreVoteResponse
        frames of a wire batch at this arena's leaders (.bytes, .n_bytes, .offsets, .n).  voters: VOTER_DTYPE rows
        covering the groups below the highest allocated one -> (status u8[n], out u64[n][2] = {leader_id, T} of the
        claimants, response blob, response offsets u32[responses + 1], totals u64[2])."""
        vt = np.ascontiguousarray(voters, dtype=VOTER_DTYPE)
        assert len(vt) >= self.get_info().hi
        return self._reply("leader_term_wire", frames, (vt,), (2,), follower_term_wire_bound)

    def leader_term_wire_device(self, d_bytes, n_bytes, d_offsets, n, d_voters, d_status, d_out, d_resp_bytes,
                                resp_bytes_capacity, d_resp_offsets, d_totals, stream=None):
        self._ck(self._L.raftgpu_leader_term_wire_device(self._h, stream, d_bytes, n_bytes, d_offsets, n, d_voters,
                                                         d_status, d_out, d_resp_bytes, resp_bytes_capacity,
                                                         d_resp_offsets, d_totals), "leader_term_wire_device")

    def leader_vote_request_wire(self, frames, voters):
        """raftgpu_leader_vote_request_wire: Raft::step's term rules and the vote arm for the MsgRequestVote /
        MsgRequestPreVote frames of a wire batch at this arena's leaders (.bytes, .n_bytes, .offsets, .n; headers name
        the leader's group slot), each group's frames after its claimant DUP.  voters: VOTER_DTYPE rows covering the
        groups below the highest allocated one -> (status u8[n], out u64[n][2] = {m.from, term after} of the OK frames,
        response blob, response offsets u32[responses + 1], totals u64[2])."""
        vt = np.ascontiguousarray(voters, dtype=VOTER_DTYPE)
        assert len(vt) >= self.get_info().hi
        return self._reply("leader_vote_request_wire", frames, (vt,), (2,), vote_request_wire_bound)

    def leader_vote_request_wire_device(self, d_bytes, n_bytes, d_offsets, n, d_voters, d_status, d_out, d_resp_bytes,
                                        resp_bytes_capacity, d_resp_offsets, d_totals, stream=None):
        self._ck(self._L.raftgpu_leader_vote_request_wire_device(self._h, stream, d_bytes, n_bytes, d_offsets, n, d_voters,
                                                                 d_status, d_out, d_resp_bytes, resp_bytes_capacity,
                                                                 d_resp_offsets, d_totals), "leader_vote_request_wire_device")

    def follower_response_wire(self, frames, voters):
        """raftgpu_follower_response_wire: Raft::step's term rules and the drop arms of step_follower and step_candidate
        for the MsgAppendResponse, MsgRequestVoteResponse, MsgHeartbeatResponse and MsgRequestPreVoteResponse frames of a
        wire batch at this arena's followers and candidates (.bytes, .n_bytes, .offsets, .n).  voters: VOTER_DTYPE rows
        covering the groups below the highest allocated one -> (status u8[n], out u64[n] = T of the claimants)."""
        vt = np.ascontiguousarray(voters, dtype=VOTER_DTYPE)
        assert len(vt) >= self.get_info().hi
        n = frames.n
        status, out = np.zeros(n, np.uint8), np.zeros(n, np.uint64)
        self._ck(self._L.raftgpu_follower_response_wire(self._h, frames.bytes.ctypes.data, frames.n_bytes,
                                                        frames.offsets.ctypes.data, n, vt.ctypes.data, status.ctypes.data,
                                                        out.ctypes.data), "follower_response_wire")
        return status, out

    def follower_response_wire_device(self, d_bytes, n_bytes, d_offsets, n, d_voters, d_status, d_out, stream=None):
        self._ck(self._L.raftgpu_follower_response_wire_device(self._h, stream, d_bytes, n_bytes, d_offsets, n, d_voters,
                                                               d_status, d_out), "follower_response_wire_device")

    def follower_append(self, frames, log):
        """raftgpu_follower_append: handle_append_entries at this arena's followers for the entry-less MsgAppend frames
        of a wire batch (.bytes, .n_bytes, .offsets, .n; headers name the follower's group slot).  log:
        FOLLOWER_LOG_DTYPE rows covering the groups below the highest allocated one -> (status u8[n], from u64[n],
        response blob, response offsets u32[responses + 1], totals u64[2])."""
        lt = np.ascontiguousarray(log, dtype=FOLLOWER_LOG_DTYPE)
        assert len(lt) >= self.get_info().hi
        return self._reply("follower_append", frames, (lt,), (), follower_append_bound)

    def follower_append_device(self, d_bytes, n_bytes, d_offsets, n, d_log, d_status, d_from, d_resp_bytes,
                               resp_bytes_capacity, d_resp_offsets, d_totals, stream=None):
        self._ck(self._L.raftgpu_follower_append_device(self._h, stream, d_bytes, n_bytes, d_offsets, n, d_log, d_status,
                                                        d_from, d_resp_bytes, resp_bytes_capacity, d_resp_offsets, d_totals),
                 "follower_append_device")

    def follower_append_entries(self, frames, log):
        """raftgpu_follower_append_entries: handle_append_entries at this arena's followers for the MsgAppend frames of
        a wire batch, entries appended at the log's tail.  log: FOLLOWER_LOG_DTYPE rows covering the groups below the
        highest allocated one, a C-contiguous array whose appended rows' runs are updated in place -> (status u8[n],
        from u64[n], appended FOLLOWER_APPENDED_DTYPE[n], response blob, response offsets u32[responses + 1], totals
        u64[2])."""
        assert log.dtype == FOLLOWER_LOG_DTYPE and log.flags.c_contiguous and len(log) >= self.get_info().hi
        return self._reply("follower_append_entries", frames, (log,), (), follower_append_bound, FOLLOWER_APPENDED_DTYPE)

    def follower_append_entries_device(self, d_bytes, n_bytes, d_offsets, n, d_log, d_status, d_from, d_appended,
                                       d_resp_bytes, resp_bytes_capacity, d_resp_offsets, d_totals, stream=None):
        self._ck(self._L.raftgpu_follower_append_entries_device(self._h, stream, d_bytes, n_bytes, d_offsets, n, d_log,
                                                                d_status, d_from, d_appended, d_resp_bytes,
                                                                resp_bytes_capacity, d_resp_offsets, d_totals),
                 "follower_append_entries_device")

    def update_state(self, entries: np.ndarray) -> np.ndarray:
        """raftgpu_update_state: send entries with next_idx = last -> result bytes."""
        assert entries.dtype == SEND_ENTRY_DTYPE and entries.flags.c_contiguous
        res = np.zeros(len(entries), dtype=np.uint8)
        self._ck(self._L.raftgpu_update_state(self._h, entries.ctypes.data, len(entries), res.ctypes.data), "update_state")
        return res

    # -- wire path (SURVEY 8(f4))
    def group_set_term(self, g, term):
        self._ck(self._L.raftgpu_group_set_term(self._h, g, term), "group_set_term")

    def step_begin_wire(self, batch, flags=0):
        """batch: anything with .bytes (u8 array), .n_bytes, .offsets (u32 array), .n, .records (24-byte records or
        None), .n_records -- e.g. wire.WireBuffers.  The arrays must stay alive and untouched until step_wait."""
        wb = WireBatch(batch.bytes.ctypes.data, batch.n_bytes, batch.offsets.ctypes.data, batch.n,
                       batch.records.ctypes.data if batch.n_records else None, batch.n_records)
        self._ck(self._L.raftgpu_step_begin_wire(self._h, C.byref(wb), flags), "step_begin_wire")

    def wire_status(self) -> np.ndarray:
        """Status bytes (RAFTGPU_WIRE_* << 4 | RAFTGPU_RES_*) of the last completed wire step (a view)."""
        p, n = C.c_void_p(), C.c_uint64()
        self._ck(self._L.raftgpu_step_wire_status(self._h, C.byref(p), C.byref(n)), "step_wire_status")
        if n.value == 0:
            return np.zeros(0, dtype=np.uint8)
        return np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(n.value,))

    def wire_apply_device(self, d_bytes, n_bytes, d_offsets, n, d_status, stream=None):
        self._ck(self._L.raftgpu_wire_apply_device(self._h, stream, d_bytes, n_bytes, d_offsets, n, d_status), "wire_apply_device")

    def step_wait(self, check: bool = True) -> StepResult:
        r = StepResult()
        rc = self._L.raftgpu_step_wait(self._h, C.byref(r))
        if check:
            self._ck(rc, "step_wait")
        r.status = rc
        return r

    def step(self, flags=0) -> StepResult:
        r = StepResult()
        self._ck(self._L.raftgpu_step(self._h, flags, C.byref(r)), "step")
        return r

    def step_results(self, n_groups: int):
        """(adv_bitmap u32[], committed u64[] | None) views into the arena's pinned results."""
        pa, pc = C.c_void_p(), C.c_void_p()
        self._ck(self._L.raftgpu_step_results(self._h, C.byref(pa), C.byref(pc)), "step_results")
        words = (n_groups + 31) // 32
        bm = np.ctypeslib.as_array(C.cast(pa, C.POINTER(C.c_uint32)), shape=(words,))
        com = np.ctypeslib.as_array(C.cast(pc, C.POINTER(C.c_uint64)), shape=(n_groups,)) if pc.value else None
        return bm, com

    def slot_results(self) -> np.ndarray:
        """Result bytes of the last zero-copy step, one per packed record / compact unit (a view)."""
        p, n = C.c_void_p(), C.c_uint64()
        self._ck(self._L.raftgpu_step_slot_results(self._h, C.byref(p), C.byref(n)), "step_slot_results")
        if n.value == 0:
            return np.zeros(0, dtype=np.uint8)
        return np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(n.value,))

    def record_results(self, ring: int = 0) -> np.ndarray:
        """Result bytes of the records enqueued on `ring` in the last step, in enqueue order."""
        n = C.c_uint64()
        self._ck(self._L.raftgpu_step_record_results(self._h, ring, None, 0, C.byref(n)),
                 "step_record_results")
        out = np.zeros(n.value, dtype=np.uint8)
        if n.value:
            self._ck(self._L.raftgpu_step_record_results(self._h, ring, out.ctypes.data, n.value,
                                                         C.byref(n)), "step_record_results")
        return out

    # -- votes
    def reset_votes(self, g):
        self._ck(self._L.raftgpu_reset_votes(self._h, g), "reset_votes")

    def record_vote(self, g, slot, vote: bool):
        self._ck(self._L.raftgpu_record_vote(self._h, g, slot, int(vote)), "record_vote")

    def send_list_device(self, first, n, d_adv, d_out, capacity, d_count, stream=None):
        self._ck(self._L.raftgpu_send_list_device(self._h, stream, first, n, d_adv, d_out, capacity, d_count),
                 "send_list_device")

    def heartbeat_commits_device(self, first, n, d_out, stream=None):
        self._ck(self._L.raftgpu_heartbeat_commits_device(self._h, stream, first, n, d_out), "heartbeat_commits_device")

    def step_send_list(self, capacity: int) -> np.ndarray:
        """Post-commit send decisions of the last completed step (raftgpu_step_send_list)."""
        out = np.zeros(capacity, dtype=SEND_ENTRY_DTYPE)
        n = C.c_uint64()
        self._ck(self._L.raftgpu_step_send_list(self._h, out.ctypes.data, capacity, C.byref(n)), "step_send_list")
        return out[: n.value]

    def tally_votes(self, first, n, d_out, stream=None):
        self._ck(self._L.raftgpu_tally_votes(self._h, stream, first, n, d_out), "tally_votes")

    def vote_result(self, g):
        r, gr, rj = C.c_int32(), C.c_uint32(), C.c_uint32()
        self._ck(self._L.raftgpu_vote_result(self._h, g, C.byref(r), C.byref(gr), C.byref(rj)),
                 "vote_result")
        return gr.value, rj.value, r.value
