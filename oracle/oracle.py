"""ctypes front-end of the CPU oracle (oracle/raft_oracle.c).

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and the
cpu_baseline / ``--impl reference`` legs of bench.py -- never by the product
path.  See oracle/raft_oracle.h for the reference file:line of every function.
"""
from __future__ import annotations

import ctypes as C
import glob
import os
import subprocess
import types

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libraft_oracle.so")

SLOTS = 8
U64_MAX = (1 << 64) - 1

VOTE_PENDING, VOTE_LOST, VOTE_WON = 0, 1, 2
VOTE_NAMES = {VOTE_PENDING: "VotePending", VOTE_LOST: "VoteLost", VOTE_WON: "VoteWon"}
STATE_PROBE, STATE_REPLICATE, STATE_SNAPSHOT = 0, 1, 2

PF_STATE_MASK, PF_PAUSED, PF_RECENT_ACTIVE, PF_INS_FULL = 0x03, 0x04, 0x08, 0x10
META_HAS_SELF, META_GROUP_COMMIT = 0x08000000, 0x10000000
REC_REJECT, REC_LOCAL, REC_EXT = 0x01, 0x02, 0x80
RES_OK, RES_OLD_PAUSED, RES_NO_PROGRESS, RES_SEND = 0x01, 0x02, 0x04, 0x08

APPEND_RESP_DTYPE = np.dtype(
    [("group", "<u4"), ("peer_slot", "u1"), ("flags", "u1"), ("reserved", "<u2"),
     ("index", "<u8"), ("commit", "<u8")]
)
assert APPEND_RESP_DTYPE.itemsize == 24

PEER_COLUMNS = ("matched", "next_idx", "peer_committed", "pending_snapshot",
                "pending_request_snapshot", "commit_group_id")
GROUP_COLUMNS = ("committed", "term_start", "last_index", "term")


def make_meta(incoming: int, outgoing: int = 0, learners: int = 0, self_slot: int | None = 0,
              group_commit: bool = False) -> int:
    m = (incoming & 0xFF) | ((outgoing & 0xFF) << 8) | ((learners & 0xFF) << 16)
    if self_slot is not None:
        m |= ((self_slot & 7) << 24) | META_HAS_SELF
    if group_commit:
        m |= META_GROUP_COMMIT
    return m


class Index(C.Structure):
    _fields_ = [("index", C.c_uint64), ("group_id", C.c_uint64)]


class AckIndexer(C.Structure):
    _fields_ = [("ids", C.POINTER(C.c_uint64)), ("idx", C.POINTER(Index)), ("n", C.c_size_t)]


class VoteMap(C.Structure):
    _fields_ = [("ids", C.POINTER(C.c_uint64)), ("vote", C.POINTER(C.c_uint8)), ("n", C.c_size_t)]


class Progress(C.Structure):
    _fields_ = [("matched", C.c_uint64), ("next_idx", C.c_uint64),
                ("pending_snapshot", C.c_uint64), ("pending_request_snapshot", C.c_uint64),
                ("commit_group_id", C.c_uint64), ("committed_index", C.c_uint64),
                ("state", C.c_uint8), ("paused", C.c_uint8), ("recent_active", C.c_uint8),
                ("ins_full", C.c_uint8), ("ins", C.c_void_p)]   # ins: optional ro_inflights*


class Inflights(C.Structure):
    """ro_inflights (inflights.rs:19-27): start, count, cap + the ring."""
    _fields_ = [("start", C.c_uint32), ("count", C.c_uint32), ("cap", C.c_uint32), ("buffer", C.POINTER(C.c_uint64))]


class RaftLog(C.Structure):
    _fields_ = [("first_index", C.c_uint64), ("dummy_term", C.c_uint64),
                ("terms", C.POINTER(C.c_uint64)), ("n", C.c_size_t), ("committed", C.c_uint64)]


class ArenaView(C.Structure):
    _fields_ = [("cap", C.c_uint32), ("n_groups", C.c_uint32)] + \
        [(n, C.POINTER(C.c_uint64)) for n in PEER_COLUMNS] + \
        [("pflags", C.POINTER(C.c_uint8)), ("meta", C.POINTER(C.c_uint32))] + \
        [(n, C.POINTER(C.c_uint64)) for n in GROUP_COLUMNS] + \
        [("ins_cap", C.c_uint32), ("ins_meta", C.POINTER(C.c_uint32)), ("ins_buf", C.POINTER(C.c_uint64))]


class WireMessage(C.Structure):
    """wo_message (wire_oracle.h): the scalar fields of eraftpb.Message."""
    _fields_ = [("msg_type", C.c_uint32), ("reject", C.c_uint32)] + \
               [(n, C.c_uint64) for n in ("to", "from_", "term", "log_term", "index", "commit", "commit_term",
                                          "request_snapshot", "reject_hint", "priority")]


def build(force: bool = False) -> str:
    """Compile oracle/libraft_oracle.so, the whole C oracle (every *.c here), with the committed Makefile
    when it is missing or older than any C source or header."""
    sources = glob.glob(os.path.join(_HERE, "*.[ch]"))
    if force or not os.path.exists(_LIB_PATH) or \
            os.path.getmtime(_LIB_PATH) < max(os.path.getmtime(f) for f in sources):
        subprocess.run(["make", "-C", _HERE, "-s"], check=True)
    return _LIB_PATH


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB_PATH)
        u64, i32, sz = C.c_uint64, C.c_int, C.c_size_t
        p64 = C.POINTER(C.c_uint64)
        L.ro_majority.restype = sz
        L.ro_majority.argtypes = [sz]
        L.ro_majority_committed_index.restype = None
        L.ro_majority_committed_index.argtypes = [p64, sz, i32, C.POINTER(AckIndexer), p64,
                                                  C.POINTER(i32)]
        L.ro_joint_committed_index.restype = None
        L.ro_joint_committed_index.argtypes = [p64, sz, p64, sz, i32, C.POINTER(AckIndexer), p64,
                                               C.POINTER(i32)]
        L.ro_majority_vote_result.restype = i32
        L.ro_majority_vote_result.argtypes = [p64, sz, C.POINTER(VoteMap)]
        L.ro_joint_vote_result.restype = i32
        L.ro_joint_vote_result.argtypes = [p64, sz, p64, sz, C.POINTER(VoteMap)]
        pp = C.POINTER(Progress)
        for name, args, res in [
            ("ro_progress_new", [pp, u64], None), ("ro_progress_reset", [pp, u64], None),
            ("ro_progress_become_probe", [pp], None), ("ro_progress_become_replicate", [pp], None),
            ("ro_progress_become_snapshot", [pp, u64], None),
            ("ro_progress_snapshot_failure", [pp], None),
            ("ro_progress_maybe_snapshot_abort", [pp], i32),
            ("ro_progress_maybe_update", [pp, u64], i32),
            ("ro_progress_update_committed", [pp, u64], None),
            ("ro_progress_optimistic_update", [pp, u64], None),
            ("ro_progress_maybe_decr_to", [pp, u64, u64, u64], i32),
            ("ro_progress_is_paused", [pp], i32), ("ro_progress_resume", [pp], None),
            ("ro_progress_pause", [pp], None), ("ro_progress_update_state", [pp, u64], i32),
        ]:
            f = getattr(L, name)
            f.argtypes, f.restype = args, res
        pl = C.POINTER(RaftLog)
        L.ro_log_last_index.argtypes, L.ro_log_last_index.restype = [pl], u64
        L.ro_log_term.argtypes, L.ro_log_term.restype = [pl, u64], u64
        L.ro_log_commit_to.argtypes, L.ro_log_commit_to.restype = [pl, u64], i32
        L.ro_log_maybe_commit.argtypes, L.ro_log_maybe_commit.restype = [pl, u64, u64], i32
        pv = C.POINTER(ArenaView)
        L.ro_arena_mci.argtypes, L.ro_arena_mci.restype = [pv, C.c_uint32, p64, C.POINTER(i32)], None
        L.ro_arena_maybe_commit.argtypes, L.ro_arena_maybe_commit.restype = [pv, C.c_uint32], i32
        L.ro_arena_maybe_commit_literal.argtypes = [pv, C.c_uint32]
        L.ro_arena_maybe_commit_literal.restype = i32
        L.ro_arena_apply.argtypes = [pv, C.c_void_p, sz, i32, C.c_void_p]
        L.ro_arena_apply.restype = None
        L.ro_arena_recompute.argtypes = [pv, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p,
                                         C.c_void_p]
        L.ro_arena_recompute.restype = u64
        L.ro_arena_vote_result.argtypes = [pv, C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32),
                                           C.POINTER(C.c_uint32)]
        L.ro_arena_vote_result.restype = i32
        L.ro_arena_send_list.argtypes = [pv, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint64]
        L.ro_arena_send_list.restype = C.c_uint64
        L.ro_arena_heartbeat_commits.argtypes = [pv, C.c_uint32, C.c_uint32, C.c_void_p]
        L.ro_arena_heartbeat_commits.restype = None
        L.ro_arena_apply_heartbeat.argtypes = [pv, C.c_void_p, sz, C.c_void_p]
        L.ro_arena_apply_heartbeat.restype = None
        L.ro_arena_update_state.argtypes = [pv, C.c_void_p, sz, C.c_void_p]
        L.ro_arena_update_state.restype = None
        L.ro_bench_recompute.argtypes = [pv, i32, i32, p64]
        L.ro_bench_recompute.restype = C.c_double
        L.ro_bench_step.argtypes = [pv, C.c_void_p, sz, i32, p64]
        L.ro_bench_step.restype = C.c_double
        L.ro_bench_step_fast.argtypes = [pv, C.c_void_p, sz, i32, p64]
        L.ro_bench_step_fast.restype = C.c_double
        pi = C.POINTER(Inflights)
        L.ro_inflights_full.argtypes, L.ro_inflights_full.restype = [pi], i32
        L.ro_inflights_add.argtypes, L.ro_inflights_add.restype = [pi, u64], i32
        L.ro_inflights_free_to.argtypes, L.ro_inflights_free_to.restype = [pi, u64], None
        L.ro_inflights_free_first_one.argtypes, L.ro_inflights_free_first_one.restype = [pi], None
        L.ro_inflights_reset.argtypes, L.ro_inflights_reset.restype = [pi], None
        L.wo_decode_message.argtypes = [C.c_void_p, sz, C.POINTER(WireMessage)]
        L.wo_decode_message.restype = i32
        L.wo_decode_batch.argtypes = [C.c_void_p, C.c_void_p, sz, C.c_uint64, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_void_p]
        L.wo_decode_batch.restype = None
        _lib = L
    return _lib


# --------------------------------------------------------------------------- quorum helpers

def _u64arr(vals):
    a = (C.c_uint64 * max(1, len(vals)))(*vals)
    return a


def _ack(lookup: dict[int, tuple[int, int]]):
    ids = list(lookup.keys())
    ida = _u64arr(ids)
    ixa = (Index * max(1, len(ids)))(*[Index(lookup[i][0], lookup[i][1]) for i in ids])
    return AckIndexer(ida, ixa, len(ids)), (ida, ixa)


def majority_committed_index(voters, lookup, use_group_commit=False):
    """MajorityConfig::committed_index (majority.rs:70-124).  lookup: id -> (index, group_id)."""
    l, keep = _ack(lookup)
    out, gc = C.c_uint64(), C.c_int()
    v = _u64arr(list(voters))
    lib().ro_majority_committed_index(v, len(voters), int(use_group_commit), C.byref(l),
                                      C.byref(out), C.byref(gc))
    return out.value, bool(gc.value)


def joint_committed_index(incoming, outgoing, lookup, use_group_commit=False):
    """JointConfig::committed_index (joint.rs:47-51)."""
    l, keep = _ack(lookup)
    out, gc = C.c_uint64(), C.c_int()
    a, b = _u64arr(list(incoming)), _u64arr(list(outgoing))
    lib().ro_joint_committed_index(a, len(incoming), b, len(outgoing), int(use_group_commit),
                                   C.byref(l), C.byref(out), C.byref(gc))
    return out.value, bool(gc.value)


def _votes(votes: dict[int, bool]):
    ids = list(votes.keys())
    ida = _u64arr(ids)
    va = (C.c_uint8 * max(1, len(ids)))(*[1 if votes[i] else 0 for i in ids])
    return VoteMap(ida, va, len(ids)), (ida, va)


def majority_vote_result(voters, votes):
    vm, keep = _votes(votes)
    return lib().ro_majority_vote_result(_u64arr(list(voters)), len(voters), C.byref(vm))


def joint_vote_result(incoming, outgoing, votes):
    vm, keep = _votes(votes)
    return lib().ro_joint_vote_result(_u64arr(list(incoming)), len(incoming),
                                      _u64arr(list(outgoing)), len(outgoing), C.byref(vm))


# --------------------------------------------------------------------------- arena helpers

def new_columns(cap: int, n_groups: int | None = None):
    """Zeroed SoA columns with the GPU arena's layout ([SLOTS][cap] / [cap])."""
    c = types.SimpleNamespace()
    c.cap = int(cap)
    c.n_groups = int(cap if n_groups is None else n_groups)
    for n in PEER_COLUMNS:
        setattr(c, n, np.zeros((SLOTS, cap), dtype=np.uint64))
    c.pflags = np.zeros((SLOTS, cap), dtype=np.uint8)
    c.meta = np.zeros(cap, dtype=np.uint32)
    for n in GROUP_COLUMNS:
        setattr(c, n, np.zeros(cap, dtype=np.uint64))
    return c


def copy_columns(c):
    d = types.SimpleNamespace(cap=c.cap, n_groups=c.n_groups)
    for n in PEER_COLUMNS + ("pflags", "meta") + GROUP_COLUMNS:
        setattr(d, n, getattr(c, n).copy())
    if getattr(c, "ins_cap", 0):
        d.ins_cap, d.ins_meta, d.ins_buf = c.ins_cap, c.ins_meta.copy(), c.ins_buf.copy()
    return d


def view(c) -> ArenaView:
    v = ArenaView()
    v.cap, v.n_groups = c.cap, c.n_groups
    for n in PEER_COLUMNS + GROUP_COLUMNS:
        arr = getattr(c, n)
        assert arr.dtype == np.uint64 and arr.flags.c_contiguous
        setattr(v, n, arr.ctypes.data_as(C.POINTER(C.c_uint64)))
    assert c.pflags.dtype == np.uint8 and c.pflags.flags.c_contiguous
    assert c.meta.dtype == np.uint32 and c.meta.flags.c_contiguous
    v.pflags = c.pflags.ctypes.data_as(C.POINTER(C.c_uint8))
    v.meta = c.meta.ctypes.data_as(C.POINTER(C.c_uint32))
    ins_cap = int(getattr(c, "ins_cap", 0))
    v.ins_cap = ins_cap
    if ins_cap:    # the Inflights windows are modelled (enable_inflights)
        assert c.ins_meta.dtype == np.uint32 and c.ins_meta.shape == (SLOTS, c.cap) and c.ins_meta.flags.c_contiguous
        assert c.ins_buf.dtype == np.uint64 and c.ins_buf.shape == (SLOTS, c.cap, ins_cap) and c.ins_buf.flags.c_contiguous
        v.ins_meta = c.ins_meta.ctypes.data_as(C.POINTER(C.c_uint32))
        v.ins_buf = c.ins_buf.ctypes.data_as(C.POINTER(C.c_uint64))
    return v


def enable_inflights(c, ins_cap: int):
    """Model the per-peer Inflights windows (inflights.rs) of these columns: empty rings of `ins_cap` entries."""
    c.ins_cap = int(ins_cap)
    c.ins_meta = np.zeros((SLOTS, c.cap), dtype=np.uint32)
    c.ins_buf = np.zeros((SLOTS, c.cap, ins_cap), dtype=np.uint64)
    return c


def arena_mci(c, g: int):
    out, gc = C.c_uint64(), C.c_int()
    v = view(c)
    lib().ro_arena_mci(C.byref(v), g, C.byref(out), C.byref(gc))
    return out.value, bool(gc.value)


def arena_apply(c, recs: np.ndarray, mode: int = 0, want_results: bool = True):
    """Apply records in arrival order.  mode 0 = batched, 1 = per-message maybe_commit."""
    assert recs.dtype == APPEND_RESP_DTYPE and recs.flags.c_contiguous
    res = np.zeros(len(recs), dtype=np.uint8) if want_results else None
    v = view(c)
    lib().ro_arena_apply(C.byref(v), recs.ctypes.data, len(recs), mode,
                         res.ctypes.data if res is not None else None)
    return res


def arena_recompute(c, first: int = 0, n: int | None = None, want_mci: bool = False):
    n = c.n_groups - first if n is None else n
    bitmap = np.zeros((c.cap + 31) // 32, dtype=np.uint32)
    mci = np.zeros(c.cap, dtype=np.uint64) if want_mci else None
    gc = np.zeros(c.cap, dtype=np.uint8) if want_mci else None
    v = view(c)
    adv = lib().ro_arena_recompute(C.byref(v), first, n, bitmap.ctypes.data,
                                   mci.ctypes.data if want_mci else None,
                                   gc.ctypes.data if want_mci else None)
    return adv, bitmap, mci, gc


def arena_maybe_commit(c, g: int, literal: bool = False) -> bool:
    v = view(c)
    f = lib().ro_arena_maybe_commit_literal if literal else lib().ro_arena_maybe_commit
    return bool(f(C.byref(v), g))


def arena_vote_result(c, votes: np.ndarray, g: int):
    assert votes.dtype == np.uint8 and votes.shape == (SLOTS, c.cap)
    gr, rj = C.c_uint32(), C.c_uint32()
    v = view(c)
    r = lib().ro_arena_vote_result(C.byref(v), votes.ctypes.data, g, C.byref(gr), C.byref(rj))
    return gr.value, rj.value, r


SEND_ENTRY_DTYPE = np.dtype([("group", "<u4"), ("peer_slot", "u1"), ("flags", "u1"), ("reserved", "<u2"),
                             ("next_idx", "<u8")])


def arena_send_list(c, adv_bitmap=None, first: int = 0, n: int | None = None):
    """bcast_append over the advanced groups (raft.rs:857-865, 780-788): entries in (group, slot) order."""
    n = c.n_groups - first if n is None else n
    v = view(c)
    bm = None if adv_bitmap is None else np.ascontiguousarray(adv_bitmap, dtype=np.uint32)
    need = lib().ro_arena_send_list(C.byref(v), first, n, None if bm is None else bm.ctypes.data, None, 0)
    out = np.zeros(need, dtype=SEND_ENTRY_DTYPE)
    got = lib().ro_arena_send_list(C.byref(v), first, n, None if bm is None else bm.ctypes.data, out.ctypes.data, need)
    assert got == need
    return out


def arena_apply_heartbeat(c, recs: np.ndarray) -> np.ndarray:
    """handle_heartbeat_response (raft.rs:1777-1819) for every REC_HEARTBEAT record, in order."""
    assert recs.dtype == APPEND_RESP_DTYPE and recs.flags.c_contiguous
    res = np.zeros(len(recs), dtype=np.uint8)
    v = view(c)
    lib().ro_arena_apply_heartbeat(C.byref(v), recs.ctypes.data, len(recs), res.ctypes.data)
    return res


def arena_update_state(c, entries: np.ndarray) -> np.ndarray:
    """Progress::update_state(last) for every {group, peer_slot, next_idx = last} entry (16-byte send entries)."""
    assert entries.dtype.itemsize == 16 and entries.flags.c_contiguous
    res = np.zeros(len(entries), dtype=np.uint8)
    v = view(c)
    lib().ro_arena_update_state(C.byref(v), entries.ctypes.data, len(entries), res.ctypes.data)
    return res


def arena_heartbeat_commits(c, first: int = 0, n: int | None = None) -> np.ndarray:
    """send_heartbeat's commit = min(matched, committed) per peer (raft.rs:838-840); [SLOTS][n]."""
    n = c.n_groups - first if n is None else n
    out = np.zeros((SLOTS, n), dtype=np.uint64)
    v = view(c)
    lib().ro_arena_heartbeat_commits(C.byref(v), first, n, out.ctypes.data)
    return out


def bench_recompute(c, n_threads: int, iters: int):
    adv = C.c_uint64()
    v = view(c)
    secs = lib().ro_bench_recompute(C.byref(v), n_threads, iters, C.byref(adv))
    return secs, adv.value


def bench_step(c, recs: np.ndarray, n_threads: int, fast: bool = False):
    adv = C.c_uint64()
    v = view(c)
    f = lib().ro_bench_step_fast if fast else lib().ro_bench_step
    secs = f(C.byref(v), recs.ctypes.data, len(recs), n_threads, C.byref(adv))
    return secs, adv.value


# --------------------------------------------------------------------------- wire decode (SURVEY 8(f4))

WIRE_OK, WIRE_SKIP_TYPE, WIRE_TERM, WIRE_NEEDS_LOG, WIRE_MALFORMED, WIRE_DUP = range(6)


def wire_decode_message(raw: bytes):
    """wo_decode_message: dict of the scalar fields, or None when the bytes are not a protobuf message."""
    m = WireMessage()
    buf = (C.c_uint8 * max(1, len(raw))).from_buffer_copy(raw or b"\0")
    if not lib().wo_decode_message(buf, len(raw), C.byref(m)):
        return None
    return {"msg_type": m.msg_type, "reject": m.reject, "to": m.to, "from": m.from_, "term": m.term,
            "log_term": m.log_term, "index": m.index, "commit": m.commit, "commit_term": m.commit_term,
            "request_snapshot": m.request_snapshot, "reject_hint": m.reject_hint, "priority": m.priority}


def wire_n_bytes(blob: np.ndarray, n_bytes: int | None) -> int:
    """A wire batch's length: n_bytes, at most len(blob) (the oracles read no byte past the blob)."""
    n_bytes = len(blob) if n_bytes is None else int(n_bytes)
    assert 0 <= n_bytes <= len(blob)
    return n_bytes


def wire_decode_batch(blob: np.ndarray, offsets: np.ndarray, n_groups: int, group_term: np.ndarray | None = None,
                      n_bytes: int | None = None):
    """wo_decode_batch -> (status u8[n], records (24-byte dtype)[n], hint u64[n], request_snapshot u64[n]).  n_bytes:
    the batch's length (default len(blob)); a frame that ends past it is WIRE_MALFORMED."""
    n = len(offsets) - 1
    rec_dtype = np.dtype([("group", "<u4"), ("peer_slot", "u1"), ("flags", "u1"), ("reserved", "<u2"),
                          ("index", "<u8"), ("commit", "<u8")])
    status = np.zeros(n, dtype=np.uint8)
    recs = np.zeros(n, dtype=rec_dtype)
    hint = np.zeros(n, dtype=np.uint64)
    snap = np.zeros(n, dtype=np.uint64)
    blob = np.ascontiguousarray(blob, dtype=np.uint8)
    offsets = np.ascontiguousarray(offsets, dtype=np.uint32)
    gt = None if group_term is None else np.ascontiguousarray(group_term, dtype=np.uint64)
    lib().wo_decode_batch(blob.ctypes.data, offsets.ctypes.data, n, wire_n_bytes(blob, n_bytes),
                          None if gt is None else gt.ctypes.data, n_groups, status.ctypes.data, recs.ctypes.data,
                          hint.ctypes.data, snap.ctypes.data)
    return status, recs, hint, snap
